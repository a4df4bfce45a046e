"""Neural-network model base class — the drop-in for reference ``src/nn_skeleton.py``.

Same constructor (`ModelSkeleton(mc)`), same layer-constructor methods with the
same argument meaning (`_conv_layer`, `_conv_bn_layer`, `_pooling_layer`), same
graph attributes (`image_input`, `preds`, `det_boxes`, `det_probs`, `det_class`,
`model_params`, `model_size_counter`, `flop_counter`, `activation_counter`) and the
same `filter_prediction(boxes, probs, cls_idx)`.  Instead of building a TF-1.0
graph, each constructor records the layer into a `libsqdet_b200` engine plan
(C ABI, `include/sqdet_b200.h`); the arithmetic runs in hand-written sm_90a
kernels.  There is no TensorFlow and no CPU fallback.

What replaces `sess.run([model.det_boxes, model.det_probs, model.det_class],
feed_dict={model.image_input: images})` (reference src/demo.py:193-195):
  * `Session().run(fetches, feed_dict)`           — same call shape, or
  * `model.detect(images)`                         — direct,
  * `model.detect_filtered(images)`                — detect + filter_prediction on
    every image in one GPU pass (what demo.py:193-199 / eval.py:75-87 do in two
    steps with a Python loop).
Training-only graph pieces (loss / train / viz graphs, `_fc_layer`, the input
FIFO queue; nn_skeleton.py:285-372,589-694) are out of scope of this engine.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import SqdetError  # noqa: F401
from .frames import ORDERS, PIXEL_FORMATS, frame_count, order_code, pack_frames


class GraphTensor:
  """Opaque handle to a tensor of the engine plan (stands in for a tf.Tensor)."""

  def __init__(self, model, name, tid=None, shape=None, fetch=None):
    self.model = model
    self.name = name
    self.id = tid
    self.shape = shape            # (B, H, W, C) for activations
    self.fetch = fetch            # 'det_boxes' | 'det_probs' | 'det_class' | None

  def get_shape(self):
    return self.shape

  def __repr__(self):
    return 'GraphTensor(%r, shape=%r)' % (self.name, self.shape)


class GraphParam:
  """Handle to one model parameter (stands in for a tf.Variable in
  `model.model_params`, which the reference hands to tf.train.Saver)."""

  def __init__(self, model, name, shape):
    self.model = model
    self.name = name
    self.shape = tuple(shape)

  def __repr__(self):
    return 'GraphParam(%r, shape=%r)' % (self.name, self.shape)


class Session:
  """Minimal stand-in for tf.Session so reference-style callers keep reading
  `sess.run(fetches, feed_dict={model.image_input: images})`."""

  def __init__(self, *args, **kwargs):
    pass

  def __enter__(self):
    return self

  def __exit__(self, *exc):
    return False

  def run(self, fetches, feed_dict=None):
    single = isinstance(fetches, GraphTensor)
    flist = [fetches] if single else list(fetches)
    if not flist:
      return []
    model = flist[0].model
    out = model.run(flist, feed_dict or {})
    return out[0] if single else out


class ModelSkeleton:
  """Base class of NN detection models (reference nn_skeleton.py:72)."""

  def __init__(self, mc, gpu_id=0, math_mode=None):
    self.mc = mc
    self.gpu_id = int(gpu_id)
    # dropout keep probability (nn_skeleton.py:78); inference => identity
    self.keep_prob = 0.5 if mc.IS_TRAINING else 1.0
    if mc.IS_TRAINING:
      raise NotImplementedError(
          'squeezedet_b200 is an inference engine: mc.IS_TRAINING must be False')
    if math_mode is None:
      math_mode = getattr(mc, 'MATH_MODE', _lib.MATH_TF32X3_TC)
    self.math_mode = int(math_mode)
    cfg = _lib.Config(
        batch_size=int(mc.BATCH_SIZE), image_height=int(mc.IMAGE_HEIGHT),
        image_width=int(mc.IMAGE_WIDTH), classes=int(mc.CLASSES),
        anchors_per_grid=int(mc.ANCHOR_PER_GRID),
        top_n_detection=int(mc.TOP_N_DETECTION),
        prob_thresh=float(mc.PROB_THRESH), nms_thresh=float(mc.NMS_THRESH),
        exp_thresh=float(mc.EXP_THRESH),
        batch_norm_epsilon=float(mc.BATCH_NORM_EPSILON),
        math_mode=self.math_mode, max_dets=int(getattr(mc, 'MAX_DETS', 0)))
    self._lib = _lib.load()
    handle = C.c_void_p()
    _lib.check(self._lib.sqdet_create(C.byref(cfg), self.gpu_id, C.byref(handle)))
    self._engine = handle
    self._finalized = False
    self._tensors = {}

    # image batch input [B, H, W, 3] fp32 (BGR, mean-subtracted)  (nn_skeleton.py:81-84)
    self.image_input = self.ph_image_input = GraphTensor(
        self, 'image_input', 0,
        (mc.BATCH_SIZE, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, 3))
    self._tensors['image_input'] = self.image_input

    self.model_params = []           # GraphParam list, reference order
    self.model_size_counter = []     # (layer_name, parameter count)
    self.flop_counter = []           # (layer_name, flops)
    self.activation_counter = [('input', mc.IMAGE_WIDTH * mc.IMAGE_HEIGHT * 3)]
    self.preds = None
    self.det_boxes = self.det_probs = self.det_class = None

  # -------------------------------------------------------------------------------------
  def __del__(self):
    try:
      if getattr(self, '_engine', None):
        self._lib.sqdet_destroy(self._engine)
        self._engine = None
    except Exception:
      pass

  def _add_forward_graph(self):
    """NN architecture specification."""
    raise NotImplementedError

  def _new_tensor(self, name, tid):
    shape = (C.c_int64 * 4)()
    buf = C.create_string_buffer(256)
    _lib.check(self._lib.sqdet_tensor_info(self._engine, tid, buf, 256, shape))
    t = GraphTensor(self, buf.value.decode(), tid, tuple(int(s) for s in shape))
    self._tensors[t.name] = t
    return t

  def _count(self, layer_name, channels, filters, size, out_shape, relu):
    # parameter / flop / activation counters, nn_skeleton.py:549-561
    self.model_size_counter.append(
        (layer_name, (1 + size * size * int(channels)) * filters))
    num_flops = (1 + 2 * int(channels) * size * size) * filters * out_shape[1] * out_shape[2]
    if relu:
      num_flops += 2 * filters * out_shape[1] * out_shape[2]
    self.flop_counter.append((layer_name, num_flops))
    self.activation_counter.append(
        (layer_name, out_shape[1] * out_shape[2] * out_shape[3]))

  # ---- layer constructors -----------------------------------------------------------
  def _conv_layer(self, layer_name, inputs, filters, size, stride, padding='SAME',
                  freeze=False, xavier=False, relu=True, stddev=0.001):
    """Convolutional layer: relu?(conv2d(inputs) + biases)  (nn_skeleton.py:471-563).
    `freeze`, `xavier`, `stddev` only affect training/initialisation and are
    accepted for signature compatibility."""
    out = C.c_int()
    _lib.check(self._lib.sqdet_add_conv(
        self._engine, layer_name.encode(), inputs.id, int(filters), int(size),
        int(stride), _lib.pad_code(padding), int(bool(relu)), C.byref(out)))
    t = self._new_tensor(layer_name, out.value)
    channels = inputs.shape[3]
    self.model_params += [
        GraphParam(self, layer_name + '/kernels', (size, size, channels, filters)),
        GraphParam(self, layer_name + '/biases', (filters,))]
    self._count(layer_name, channels, filters, size, t.shape, relu)
    return t

  def _conv_bn_layer(self, inputs, conv_param_name, bn_param_name, scale_param_name,
                     filters, size, stride, padding='SAME', freeze=False, relu=True,
                     conv_with_bias=False, stddev=0.001):
    """Convolution + frozen BatchNorm + [relu]  (nn_skeleton.py:374-468).
    Variables live under scope `conv_param_name`: kernels, [biases], gamma, beta,
    mean, var (the Caffe bn_/scale_ names only matter when importing a .pkl)."""
    if padding.upper() != 'SAME':
      raise ValueError('_conv_bn_layer is only used with SAME padding')
    out = C.c_int()
    _lib.check(self._lib.sqdet_add_conv_bn(
        self._engine, conv_param_name.encode(), inputs.id, int(filters), int(size),
        int(stride), int(bool(relu)), int(bool(conv_with_bias)), C.byref(out)))
    t = self._new_tensor(conv_param_name, out.value)
    channels = inputs.shape[3]
    names = ['kernels'] + (['biases'] if conv_with_bias else []) + \
        ['gamma', 'beta', 'mean', 'var']
    for n in names:
      shp = (size, size, channels, filters) if n == 'kernels' else (filters,)
      self.model_params.append(GraphParam(self, conv_param_name + '/' + n, shp))
    self._count(conv_param_name, channels, filters, size, t.shape, relu)
    return t

  def _pooling_layer(self, layer_name, inputs, size, stride, padding='SAME'):
    """Max pooling (nn_skeleton.py:565-586)."""
    out = C.c_int()
    _lib.check(self._lib.sqdet_add_pool(
        self._engine, layer_name.encode(), inputs.id, int(size), int(stride),
        _lib.pad_code(padding), C.byref(out)))
    t = self._new_tensor(layer_name, out.value)
    self.activation_counter.append((layer_name, int(np.prod(t.shape[1:]))))
    return t

  def _fused_fire(self, layer_name, inputs, s1x1, e1x1, e3x3):
    """squeeze1x1 -> (expand1x1 || expand3x3) -> concat as ONE plan op so the engine
    can run the expand pair as a single fused tensor-core kernel
    (reference: three _conv_layer calls + tf.concat, squeezeDet.py:96-106)."""
    out = C.c_int()
    _lib.check(self._lib.sqdet_add_fire(
        self._engine, layer_name.encode(), inputs.id, int(s1x1), int(e1x1),
        int(e3x3), C.byref(out)))
    t = self._new_tensor(layer_name, out.value)
    cin = inputs.shape[3]
    sq_shape = t.shape[:3] + (s1x1,)
    for sub, ch, flt, sz in (('/squeeze1x1', cin, s1x1, 1),
                             ('/expand1x1', s1x1, e1x1, 1),
                             ('/expand3x3', s1x1, e3x3, 3)):
      nm = layer_name + sub
      self.model_params += [GraphParam(self, nm + '/kernels', (sz, sz, ch, flt)),
                            GraphParam(self, nm + '/biases', (flt,))]
      self._count(nm, ch, flt, sz, (sq_shape if sub == '/squeeze1x1'
                                    else t.shape[:3] + (flt,)), True)
    return t

  def _add_relu(self, name, a, b):
    """tf.nn.relu(a + b) of a residual unit (resnet50_convDet.py:55)."""
    out = C.c_int()
    _lib.check(self._lib.sqdet_add_add_relu(self._engine, name.encode(), a.id, b.id,
                                            C.byref(out)))
    return self._new_tensor(name, out.value)

  def _dropout(self, inputs, keep_prob, name=None):
    """tf.nn.dropout with keep_prob == 1.0 at inference: the identity."""
    assert keep_prob == 1.0
    return inputs

  # ---- interpretation graph ---------------------------------------------------------
  def _add_interpretation_graph(self):
    """Interpret NN output (nn_skeleton.py:142-283): declares `preds`/ANCHOR_BOX to
    the engine, freezes the plan and exposes det_boxes / det_probs / det_class."""
    mc = self.mc
    anchors = np.ascontiguousarray(np.asarray(mc.ANCHOR_BOX, dtype=np.float64))
    if anchors.ndim != 2 or anchors.shape[1] != 4:
      raise ValueError('mc.ANCHOR_BOX must be [ANCHORS, 4]')
    _lib.check(self._lib.sqdet_set_preds(
        self._engine, self.preds.id, anchors.ctypes.data, anchors.shape[0]))
    _lib.check(self._lib.sqdet_finalize(self._engine))
    self._finalized = True
    means = np.ascontiguousarray(np.asarray(mc.BGR_MEANS, dtype=np.float64).reshape(3))
    _lib.check(self._lib.sqdet_set_bgr_means(self._engine, means.ctypes.data))
    B, A = mc.BATCH_SIZE, anchors.shape[0]
    self.det_boxes = GraphTensor(self, 'bbox', None, (B, A, 4), 'det_boxes')
    self.det_probs = GraphTensor(self, 'score', None, (B, A), 'det_probs')
    self.det_class = GraphTensor(self, 'class_idx', None, (B, A), 'det_class')
    md = C.c_int32()
    _lib.check(self._lib.sqdet_results_dev(self._engine, None, None, None, None, None,
                                           C.byref(md)))
    self.max_dets = int(md.value)

  def _add_loss_graph(self):
    raise NotImplementedError('training graph: out of scope of the inference engine')

  _add_train_graph = _add_viz_graph = _add_loss_graph

  # ---- parameters -------------------------------------------------------------------
  def param_names(self):
    return [p.name for p in self.model_params]

  def set_param(self, name, value):
    arr = np.ascontiguousarray(np.asarray(value, dtype=np.float32))
    shape = (C.c_int64 * max(arr.ndim, 1))(*arr.shape)
    _lib.check(self._lib.sqdet_set_param(self._engine, name.encode(), arr.ctypes.data,
                                         shape, arr.ndim))

  def load_weights(self, weights, strict=True):
    """`weights`: mapping reference-variable-name -> ndarray (e.g. an .npz).  Stands
    in for tf.train.Saver(model.model_params).restore (demo.py:181-184)."""
    names = self.param_names()
    missing = [n for n in names if n not in weights]
    if strict and missing:
      raise KeyError('missing parameters: %s' % missing[:5])
    for n in names:
      if n in weights:
        self.set_param(n, weights[n])
    return missing

  # ---- execution ----------------------------------------------------------------------
  def _images_array(self, images, dtype=np.float32):
    mc = self.mc
    arr = np.asarray(images, dtype=dtype)
    want = (mc.BATCH_SIZE, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, 3)
    if arr.shape != want:
      # TF raises ValueError on a feed-shape mismatch against the static placeholder
      raise ValueError('Cannot feed value of shape %r for image_input, which has '
                       'shape %r' % (arr.shape, want))
    return np.ascontiguousarray(arr)

  def detect(self, images, want_dets=False):
    """images [B,H,W,3] float -> (det_boxes [B,A,4] f32, det_probs [B,A] f32,
    det_class [B,A] i64) [+ (dets, counts) when want_dets]."""
    if not self._finalized:
      raise SqdetError(-4, 'model graph is not finalized')
    arr = self._images_array(images)
    B, A = self.det_probs.shape
    boxes = np.empty((B, A, 4), np.float32)
    probs = np.empty((B, A), np.float32)
    cls = np.empty((B, A), np.int64)
    dets = np.empty((B, self.max_dets), _lib.DET_DTYPE) if want_dets else None
    counts = np.empty((B,), np.int32) if want_dets else None
    _lib.check(self._lib.sqdet_detect(
        self._engine, arr.ctypes.data, boxes.ctypes.data, probs.ctypes.data,
        cls.ctypes.data, dets.ctypes.data if want_dets else None,
        counts.ctypes.data if want_dets else None, None))
    if want_dets:
      return boxes, probs, cls, dets, counts
    return boxes, probs, cls

  def detect_records(self, images):
    """images -> (dets [B,max_dets] structured, counts [B]) — only the filtered
    records cross PCIe (the end-to-end fast path)."""
    arr = self._images_array(images)
    B = self.mc.BATCH_SIZE
    dets = np.empty((B, self.max_dets), _lib.DET_DTYPE)
    counts = np.empty((B,), np.int32)
    _lib.check(self._lib.sqdet_detect(self._engine, arr.ctypes.data, None, None, None,
                                      dets.ctypes.data, counts.ctypes.data, None))
    return dets, counts

  # pipelined host path: copy of batch i+1 overlaps the compute of batch i (depth 2)
  def submit(self, images_ptr, dets_ptr, counts_ptr, img_type=_lib.IMG_F32):
    """Enqueue one batch (raw host pointers, ideally pinned; must stay valid until the
    matching wait()).  img_type: _lib.IMG_F32 (feed_dict semantics) or _lib.IMG_U8 (uint8
    BGR as cv2 returns it; `- mc.BGR_MEANS` happens on the GPU, demo.py:187-190)."""
    _lib.check(self._lib.sqdet_submit(self._engine, images_ptr, int(img_type), dets_ptr,
                                      counts_ptr))

  def wait(self):
    _lib.check(self._lib.sqdet_wait(self._engine))

  def detect_u8(self, images_u8):
    """uint8 BGR images [B,H,W,3] (already at mc.IMAGE_WIDTH x IMAGE_HEIGHT) ->
    (dets, counts): the demo.py:187-199 loop body from `im - mc.BGR_MEANS` on, on the GPU."""
    B = self.mc.BATCH_SIZE
    arr = self._images_array(images_u8, np.uint8)
    dets = np.empty((B, self.max_dets), _lib.DET_DTYPE)
    counts = np.empty((B,), np.int32)
    self.submit(arr.ctypes.data, dets.ctypes.data, counts.ctypes.data, _lib.IMG_U8)
    self.wait()
    return dets, counts

  # ---- variable-size uint8 frames: pre-processing on the GPU (demo.py:187-190 / imdb.py:85-97) ----
  def submit_frames(self, frames, dets_ptr, counts_ptr, order='demo', rescale=False):
    """frames: list of n uint8 BGR arrays [h_i, w_i, 3] as cv2.imread returns them,
    1 <= n <= mc.BATCH_SIZE.  The engine resizes (cv2 float32 INTER_LINEAR) to
    (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT) and subtracts mc.BGR_MEANS in the reference order ('demo':
    resize then subtract, demo.py:187-190; 'eval': subtract then resize, imdb.py:85-97).
    rescale=True: boxes are divided by each frame's (x_scale, y_scale) BEFORE filter_prediction,
    like eval.py:80-87, in this submission only; set_box_scale's table does not apply.
    dets_ptr / counts_ptr receive n rows (sqdet_submit_frames_n: a short batch runs the kernels
    planned for BATCH_SIZE, so image i's records equal those of a full batch).  Same wait() contract as submit(); the frame arrays must stay alive until then."""
    n = frame_count(frames, self.mc.BATCH_SIZE)
    arrs = []
    for f in frames:
      a = np.ascontiguousarray(np.asarray(f, dtype=np.uint8))
      if a.ndim != 3 or a.shape[2] != 3:
        raise ValueError('a frame must be uint8 [h, w, 3], got %r' % (a.shape,))
      arrs.append(a)
    ptrs = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
    hs = (C.c_int32 * n)(*[a.shape[0] for a in arrs])
    ws = (C.c_int32 * n)(*[a.shape[1] for a in arrs])
    code = ORDERS[order]
    self._frames_alive = arrs
    _lib.check(self._lib.sqdet_submit_frames_n(self._engine, n, ptrs, hs, ws, code,
                                               int(bool(rescale)), dets_ptr, counts_ptr))

  def detect_frames(self, frames, order='demo', rescale=False):
    """Synchronous convenience over submit_frames: n frames -> (dets [n,max_dets], counts [n])."""
    n = len(frames)
    dets = np.empty((n, self.max_dets), _lib.DET_DTYPE)
    counts = np.empty((n,), np.int32)
    self.submit_frames(frames, dets.ctypes.data, counts.ctypes.data, order, rescale)
    self.wait()
    return dets, counts

  def set_box_scale(self, scales):
    """eval.py:83-84 for host-resized inputs: `scales` = B (x_scale, y_scale) pairs, or None to
    switch the rescale off.  Later forwards of already-resized images (detect, detect_records,
    submit, forward_device) divide det_boxes by them before the filter; submit_frames does not."""
    if scales is None:
      _lib.check(self._lib.sqdet_set_box_scale(self._engine, None))
      return
    arr = np.ascontiguousarray(np.asarray(scales, dtype=np.float32).reshape(-1))
    if arr.size != 2 * self.mc.BATCH_SIZE:
      raise ValueError('need BATCH_SIZE (x_scale, y_scale) pairs')
    _lib.check(self._lib.sqdet_set_box_scale(self._engine, arr.ctypes.data))

  # ---- multi-GPU: the one all-gather of the filtered records (shard.py drives this) ------------
  def comm_init(self, nranks, rank, unique_id, in_forward=True):
    """ncclCommInitRank on this engine's device; `unique_id` = the 128 bytes rank 0 obtained
    from _lib.comm_unique_id() and shared through any host channel.  in_forward=True makes
    every forward end with the all-gather (captured in its CUDA graph)."""
    buf = (C.c_char * 128).from_buffer_copy(bytes(unique_id))
    _lib.check(self._lib.sqdet_comm_init(self._engine, int(nranks), int(rank), buf))
    if in_forward:
      _lib.check(self._lib.sqdet_set_gather_in_forward(self._engine, 1))

  def set_gather_in_forward(self, on):
    _lib.check(self._lib.sqdet_set_gather_in_forward(self._engine, int(bool(on))))

  def allgather(self, stream=None):
    _lib.check(self._lib.sqdet_allgather(self._engine, None, stream))

  def gathered_device(self):
    """(device pointer, bytes per rank, nranks) of the all-gather receive buffer."""
    p, nb, nr = C.c_void_p(), C.c_int64(), C.c_int32()
    _lib.check(self._lib.sqdet_gathered_dev(self._engine, C.byref(p), C.byref(nb), C.byref(nr)))
    return p.value, int(nb.value), int(nr.value)

  def read_gathered(self):
    """Host copy of the receive buffer as [nranks, bytes_per_rank] uint8 (synchronous)."""
    ptr, nb, nr = self.gathered_device()
    out = np.empty((nr, nb), np.uint8)
    _lib.check(self._lib.sqdet_stream_sync(self.gpu_id, self.engine_stream()))
    _lib.check(self._lib.sqdet_memcpy_d2h(out.ctypes.data, ptr, out.nbytes, None))
    _lib.check(self._lib.sqdet_stream_sync(self.gpu_id, None))
    return out

  def comm_destroy(self):
    _lib.check(self._lib.sqdet_comm_destroy(self._engine))

  def engine_stream(self):
    return self._lib.sqdet_engine_stream(self._engine)

  @staticmethod
  def records_to_lists(dets, count):
    """One image's records -> the reference's filter_prediction return triple."""
    if count < 0:
      raise SqdetError(-6, 'more boxes above PROB_THRESH than the record capacity')
    d = dets[:count]
    boxes = [np.array([r['cx'], r['cy'], r['w'], r['h']], dtype=np.float32) for r in d]
    probs = [np.float32(r['prob']) for r in d]
    cls = [int(r['cls']) for r in d]
    return boxes, probs, cls

  def detect_filtered(self, images):
    """detect + filter_prediction for every image: list of (final_boxes,
    final_probs, final_cls_idx) per image (demo.py:193-199 in one GPU pass)."""
    dets, counts = self.detect_records(images)
    return [self.records_to_lists(dets[i], int(counts[i])) for i in range(len(counts))]

  def run(self, fetches, feed_dict):
    """sess.run equivalent for fetches among det_boxes/det_probs/det_class/preds/any
    activation handle."""
    if self.image_input not in feed_dict and self.ph_image_input not in feed_dict:
      raise ValueError('feed_dict must feed model.image_input')
    images = feed_dict[self.image_input]
    boxes, probs, cls = self.detect(images)
    table = {'det_boxes': boxes, 'det_probs': probs, 'det_class': cls}
    out = []
    for f in fetches:
      if f.fetch is not None:
        out.append(table[f.fetch])
      else:
        out.append(self.read_tensor(f))
    return out

  def read_tensor(self, t):
    """Fetch an activation of the last forward (debug / layer-wise parity)."""
    if isinstance(t, str):
      t = self._tensors[t]
    out = np.empty(t.shape, np.float32)
    _lib.check(self._lib.sqdet_read_tensor(self._engine, t.id, out.ctypes.data))
    return out

  # device-resident path (no host copies; used by bench / multi-GPU runner)
  def forward_device(self, images_dev_ptr, stream=None, n=None):
    """Forward of the device images at `images_dev_ptr`: all BATCH_SIZE of them, or only the
    first n (1 <= n <= BATCH_SIZE; sqdet_forward_n), in which case the buffer needs to hold just
    those n images and result rows [n, BATCH_SIZE) are left untouched (counts set to 0)."""
    if n is None:
      _lib.check(self._lib.sqdet_forward(self._engine, images_dev_ptr, stream))
    else:
      _lib.check(self._lib.sqdet_forward_n(self._engine, images_dev_ptr, int(n), stream))

  def forward_device_u8(self, images_dev_ptr, stream=None, n=None):
    """forward_device of uint8 BGR images [n, H, W, 3] at `images_dev_ptr` (any byte alignment),
    as cv2.imread / cv2.resize leave them; the engine subtracts mc.BGR_MEANS (demo.py:190).  The
    results are bitwise those of forward_device on the converted fp32 images (sqdet_forward_u8)."""
    n = self.mc.BATCH_SIZE if n is None else int(n)
    _lib.check(self._lib.sqdet_forward_u8(self._engine, images_dev_ptr, n, stream))

  def forward_device_frames(self, frames, order='demo', rescale=False, stream=None):
    """Forward of 1..BATCH_SIZE uint8 BGR frames of any size already on this engine's device:
    CUDA tensors [h, w, 3] with stride(2) == 1 and stride(1) == 3; the row stride is free, so a
    crop view such as frame[500:-205, 239:-439] passes without a copy.  The engine resizes them
    to (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT) and subtracts mc.BGR_MEANS in `order` ('demo' or
    'eval', as submit_frames) in one launch into image_input, then runs the forward on `stream`
    (forward_device_frames_fmt with 'bgr': sqdet_forward_frames with SQDET_FMT_BGR, which is
    sqdet_forward_frames_u8).  rescale=True divides the boxes by each frame's scales before the
    filter, in this call only.  Asynchronous: read the results through results_device()."""
    self.forward_device_frames_fmt(frames, 'bgr', None, order=order, rescale=rescale,
                                   stream=stream)

  def forward_device_frames_nv12(self, frames, crops=None, order='demo', rescale=False,
                                 stream=None):
    """forward_device_frames of NV12 frames already on this engine's device, as a hardware video
    decoder writes them.  Each frame is a uint8 CUDA tensor [3H/2, W] (the luma plane's H rows
    stacked on the chroma plane's H/2 rows of interleaved U,V bytes, the layout cv2 uses) or a
    pair (luma [H, W], chroma [H/2, W]); H and W even, rows may be strided, columns must be
    adjacent.  crops: None, or per frame None (the whole frame) or (x, y, w, h) inside it, at any
    origin.  The engine converts each crop exactly as cv2.cvtColor(nv12, COLOR_YUV2BGR_NV12)
    [y:y+h, x:x+w] (BT.601 limited range), then resizes and subtracts the means as
    forward_device_frames, bit for bit, in one launch into image_input, without writing a BGR
    frame (sqdet_forward_frames_nv12).  rescale=True scales the boxes back to each crop.
    Asynchronous: read the results through results_device()."""
    return self.forward_device_frames_fmt(frames, 'nv12', crops=crops, order=order,
                                          rescale=rescale, stream=stream)

  def forward_device_frames_fmt(self, frames, fmt, crops=None, order='demo', rescale=False,
                                stream=None):
    """forward_device_frames of frames in pixel format `fmt` already on this engine's device.
    Each frame is made of uint8 CUDA tensors whose rows may be strided and whose bytes within a
    row are adjacent:
      'bgr', 'rgb'    [h, w, 3] with strides (row, 3, 1);
      'bgra', 'rgba'  [h, w, 4] with strides (row, 4, 1) (capture surfaces; alpha is never read);
      'rgb_planar'    [3, h, w] with strides (plane, row, 1), as torchvision.io.decode_jpeg(...,
                      device='cuda') returns it (or a frame of list(batch) of [n, 3, h, w]), or an
                      (r, g, b) tuple of [h, w] planes;
      'nv12'          as forward_device_frames_nv12;
      'i420'          a tight [3h/2, w] tensor (Y's rows, then U's and V's bytes, as cv2 lays it
                      out) or a (y [h, w], u [h/2, w/2], v [h/2, w/2]) tuple at any pitches;
                      h and w even.
    crops: None, or per frame None (the whole frame) or (x, y, w, h) inside it, at any origin.  The
    engine converts each crop to BGR exactly as cv2.cvtColor does (COLOR_RGB2BGR, _BGRA2BGR,
    _RGBA2BGR, _YUV2BGR_NV12, _YUV2BGR_I420), then resizes and subtracts the means as
    forward_device_frames, bit for bit, in one launch into image_input, without writing a BGR
    frame (sqdet_forward_frames).  rescale=True scales the boxes back to each crop.
    Asynchronous: read the results through results_device()."""
    frames = list(frames)
    n = frame_count(frames, self.mc.BATCH_SIZE)
    code = order_code(order)
    planes, pitches, hs, ws, rects = pack_frames(frames, fmt, crops, self.gpu_id)
    _lib.check(self._lib.sqdet_forward_frames(
        self._engine, n, PIXEL_FORMATS.index(fmt), planes, pitches, hs, ws, rects, code,
        int(bool(rescale)), stream))

  def forward_device_tiles(self, frames, fmt, tiles, order='demo', stream=None):
    """Detection over whole frames as overlapping tiles (sqdet_forward_tiles).  frames: as
    forward_device_frames_fmt takes them, in pixel format `fmt`; tiles: 1..BATCH_SIZE tuples
    (frame_index, x, y, w, h), each a non-empty rectangle inside its frame (utils.util.tile_grid
    makes a covering grid; a whole-frame "overview" tile may be added), every frame with at least
    one tile.  Tile k runs as row k of forward_device_frames_fmt over the tiles as crops with
    rescale=True, then each frame's detections, shifted into frame pixels, are merged by one
    top-N and NMS on the GPU.  Asynchronous: read the merged records through
    tile_results_device() (record 'anchor' = p * A + anchor of the frame's p-th tile) and the
    per-tile rows through results_device()."""
    code = order_code(order)
    frames, tiles = list(frames), [tuple(int(v) for v in tile) for tile in tiles]
    B, n, t = self.mc.BATCH_SIZE, len(frames), len(tiles)
    if not 1 <= t <= B:
      raise ValueError('need 1 to %d tiles, got %d' % (B, t))
    if not 1 <= n <= t:
      raise ValueError('need 1 to %d frames (at most one per tile), got %d' % (t, n))
    planes, pitches, hs, ws, _ = pack_frames(frames, fmt, None, self.gpu_id)
    flat = []
    for k, tile in enumerate(tiles):
      if len(tile) != 5:
        raise ValueError('tile %d: need (frame_index, x, y, w, h), got %r' % (k, tile))
      f, x, y, w, h = tile
      if not 0 <= f < n:
        raise ValueError('tile %d: frame index %d outside [0, %d)' % (k, f, n))
      if w < 1 or h < 1 or x < 0 or y < 0 or x + w > ws[f] or y + h > hs[f]:
        raise ValueError('tile %d: %r is not a non-empty rectangle inside frame %d (%dx%d)'
                         % (k, tile, f, ws[f], hs[f]))
      flat.extend(tile)
    missing = sorted(set(range(n)) - {tile[0] for tile in tiles})
    if missing:
      raise ValueError('frame %d has no tile' % missing[0])
    _lib.check(self._lib.sqdet_forward_tiles(
        self._engine, n, PIXEL_FORMATS.index(fmt), planes, pitches, hs, ws, t,
        (C.c_int32 * (5 * t))(*flat), code, stream))

  def tile_results_device(self):
    """Device pointers of forward_device_tiles' merged results: {'dets': [B, max_dets] records,
    'counts': [B] int32, 'max_dets': int}.  Valid until the next forward_device_tiles."""
    d, c, md = C.c_void_p(), C.c_void_p(), C.c_int32()
    _lib.check(self._lib.sqdet_tile_results_dev(self._engine, C.byref(d), C.byref(c),
                                                C.byref(md)))
    return {'dets': d.value, 'counts': c.value, 'max_dets': int(md.value)}

  def tile_results(self, n, stream=None):
    """Host copies (dets [n, max_dets], counts [n]) of the merged results of the first n frames,
    after `stream` (the one forward_device_tiles ran on) has finished."""
    res = self.tile_results_device()
    dets = np.empty((n, res['max_dets']), _lib.DET_DTYPE)
    counts = np.empty((n,), np.int32)
    _lib.check(self._lib.sqdet_stream_sync(self.gpu_id, stream))
    _lib.check(self._lib.sqdet_memcpy_d2h(dets.ctypes.data, res['dets'], dets.nbytes, None))
    _lib.check(self._lib.sqdet_memcpy_d2h(counts.ctypes.data, res['counts'], counts.nbytes, None))
    _lib.check(self._lib.sqdet_stream_sync(self.gpu_id, None))
    return dets, counts

  def draw_detections_device(self, frames, fmt, which='tiles', crops=None, cdict=None,
                             stream=None):
    """Draws the last forward's detections onto `frames` in place, in device memory, exactly as
    demo.draw_detections + utils.viz.draw_box draw them with cv2 on a uint8 BGR image
    (sqdet_draw_dets): boxes and 'CLASS: (PROB)' labels of the records above mc.PLOT_PROB_THRESH,
    FONT_HERSHEY_SIMPLEX at 0.3, colours looked up as draw_box does (the label's class name in
    `cdict`, default utils.viz.CLASS_COLORS, else (0, 255, 0)).  frames and crops: as
    forward_device_frames_fmt takes them, in pixel format `fmt`.  which='tiles' draws frame f's
    merged records of forward_device_tiles (frame pixels: no crops); which='frames' draws image i's
    records of forward_device_frames_fmt with rescale=True on its crop.  RGB and RGBA frames get
    the colours in their own channel order (alpha untouched); NV12 and I420 frames get each
    colour's (Y, U, V) on the boxes' pixels and the chroma samples around them.  Asynchronous on
    `stream`: run it on the stream the forward ran on."""
    from .utils.viz import CLASS_COLORS
    if which not in ('tiles', 'frames'):
      raise ValueError("which must be 'tiles' or 'frames', got %r" % (which,))
    frames = list(frames)
    n = frame_count(frames, self.mc.BATCH_SIZE)
    planes, pitches, hs, ws, rects = pack_frames(frames, fmt, crops, self.gpu_id)
    res = self.tile_results_device() if which == 'tiles' else self.results_device()
    cdict = CLASS_COLORS if cdict is None else cdict
    names = list(self.mc.CLASS_NAMES)
    bgr = []
    for name in names:
      key = name.split(':')[0]                    # draw_box's label.split(':')[0]
      bgr.extend(int(v) for v in (cdict[key] if cdict and key in cdict else (0, 255, 0)))
    enc = [s.encode('ascii') for s in names]
    style = _lib.DrawStyle(len(names), (C.c_char_p * len(enc))(*enc),
                           (C.c_uint8 * len(bgr))(*bgr), float(self.mc.PLOT_PROB_THRESH), 0.3)
    _lib.check(self._lib.sqdet_draw_dets(
        n, PIXEL_FORMATS.index(fmt), planes, pitches, hs, ws, rects, res['dets'], res['counts'],
        res['max_dets'], C.byref(style), stream))

  def forward_profiled(self, images_dev_ptr, stream=None):
    n = self._lib.sqdet_num_ops(self._engine)
    ms = np.zeros(n, np.float32)
    _lib.check(self._lib.sqdet_forward_profiled(self._engine, images_dev_ptr, stream,
                                                ms.ctypes.data))
    return list(zip(self.op_table(), ms.tolist()))

  def op_table(self):
    """[(name, flops, params, min_bytes)] per plan op (+ the two post-proc ops)."""
    rows = []
    for i in range(self._lib.sqdet_num_ops(self._engine)):
      buf = C.create_string_buffer(256)
      fl, pa, by = C.c_int64(), C.c_int64(), C.c_int64()
      _lib.check(self._lib.sqdet_op_info(self._engine, i, buf, 256, C.byref(fl),
                                         C.byref(pa), C.byref(by)))
      rows.append((buf.value.decode(), fl.value, pa.value, by.value))
    return rows

  def op_k_splits(self):
    """{op name: S} for the ops whose K the plan splits over a cluster of S > 1 CTAs."""
    out = {}
    for i, (name, _, _, _) in enumerate(self.op_table()):
      s = self._lib.sqdet_op_k_split(self._engine, i)
      if s < 0:
        _lib.check(s)
      if s > 1:
        out[name] = s
    return out

  def results_device(self):
    """Device pointers of the last forward's results: dict of ints + max_dets."""
    ptrs = [C.c_void_p() for _ in range(5)]
    md = C.c_int32()
    _lib.check(self._lib.sqdet_results_dev(self._engine, *[C.byref(p) for p in ptrs],
                                           C.byref(md)))
    keys = ('det_boxes', 'det_probs', 'det_class', 'dets', 'counts')
    out = {k: p.value for k, p in zip(keys, ptrs)}
    out['max_dets'] = int(md.value)
    return out

  def launches_per_forward(self):
    return self._lib.sqdet_launches_per_forward(self._engine)

  # ---- filter_prediction ---------------------------------------------------------------
  def filter_prediction(self, boxes, probs, cls_idx):
    """Filter bounding box predictions with probability threshold and non-maximum
    suppression (nn_skeleton.py:696-734) — same arguments and return triple, computed
    by the GPU filter kernel through `sqdet_topk_nms`.

    Args:
      boxes: array of [cx, cy, w, h].   probs: array of probabilities.
      cls_idx: array of class indices.
    Returns:
      final_boxes (list of ndarray(4)), final_probs (list of float32),
      final_cls_idx (list of int).
    """
    mc = self.mc
    boxes = np.ascontiguousarray(np.asarray(boxes, dtype=np.float32)).reshape(-1, 4)
    probs = np.ascontiguousarray(np.asarray(probs, dtype=np.float32)).reshape(-1)
    cls_idx = np.ascontiguousarray(np.asarray(cls_idx, dtype=np.int64)).reshape(-1)
    n = len(probs)
    if n == 0:
      return [], [], []
    topn = 0 < mc.TOP_N_DETECTION < n
    cap = int(mc.TOP_N_DETECTION) if topn else min(n, 1024)
    # one pooled, grow-only scratch allocation instead of five cudaMalloc/cudaFree pairs per call
    pool = _lib.scratch_pool(self.gpu_id)
    p_boxes, p_probs, p_cls, p_dets, p_cnt = pool.carve(
        boxes.nbytes, probs.nbytes, cls_idx.nbytes, cap * _lib.DET_DTYPE.itemsize, 4)
    pool.upload(p_boxes, boxes)
    pool.upload(p_probs, probs)
    pool.upload(p_cls, cls_idx)
    _lib.check(self._lib.sqdet_topk_nms(
        p_boxes, p_probs, p_cls, 1, n, int(mc.CLASSES), int(mc.TOP_N_DETECTION),
        float(mc.PROB_THRESH), float(mc.NMS_THRESH), p_dets, p_cnt, cap, None))
    dets = pool.download(p_dets, _lib.DET_DTYPE, (cap,))
    count = int(pool.download(p_cnt, np.int32, (1,))[0])
    return self.records_to_lists(dets, count)
