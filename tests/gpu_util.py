"""Helpers shared by the tests: engines and forwards, the fp64 oracles and their per-element
bound, and stage-isolated calls of the C ABI."""
import ctypes as C

import numpy as np
import pytest

import oracle
from oracle import preproc
from oracle import tiles as oracle_tiles
from oracle.torch_port import TorchForward
from squeezedet_b200 import _lib
from squeezedet_b200 import config as cfg
from squeezedet_b200._lib import DeviceBuffer
from squeezedet_b200.nets import SqueezeDet, SqueezeDetPlus, VGG16ConvDet, ResNet50ConvDet
from squeezedet_b200.nets.squeezeDet import FireNetBase
from squeezedet_b200.utils import synth

NETS = {
    'squeezeDet': (SqueezeDet, cfg.kitti_squeezeDet_config),
    'squeezeDet+': (SqueezeDetPlus, cfg.kitti_squeezeDetPlus_config),
    'vgg16': (VGG16ConvDet, cfg.kitti_vgg16_config),
    'resnet50': (ResNet50ConvDet, cfg.kitti_res50_config),
}
MODES = [_lib.MATH_FP32_SIMT, _lib.MATH_TF32X3_TC]

# Tolerances (BASELINE.json north_star): scores and box coordinates within 1e-4 relative;
# class ids / kept-box indices exact wherever the oracle's own margin exceeds fp noise.
TOL = 1e-4

ERR_NOT_FOUND = -5          # SQDET_ERR_NOT_FOUND: tensor fused into its consumer
POST_LAUNCHES = 2           # interpret + filter (sqdet_launches_per_forward)
FIRE_TILE_H, FIRE_TILE_W = 8, 16
# The engine runs a fire as one kernel when the squeeze is <= 16 wide and the grid holds at least
# 4 tiles per SM.  H100 SXM has 132 SMs, H100 PCIe 114: sizes below stay on one side of the rule
# on both.
ONE_KERNEL_MIN_TILES = 4 * 132
PAIR_MAX_TILES = 4 * 114


def fire_tiles(batch, h, w):
  return batch * -(-h // FIRE_TILE_H) * -(-w // FIRE_TILE_W)


# ---- engines -------------------------------------------------------------------------------------
def make_mc(net, width, height, batch):
  mc = NETS[net][1]()
  mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = width, height, batch
  rows = oracle.layer_table(net, height, width)
  mc.GRID_H, mc.GRID_W = rows[-1][2][0], rows[-1][2][1]
  mc.ANCHOR_BOX = cfg.set_anchors(mc)
  mc.ANCHORS = len(mc.ANCHOR_BOX)
  return mc


def make_net(net, width, height, batch, device, math_mode=None, seed=0):
  """(model, weights): benchmark net `net` with synthetic weights `seed` loaded.  The weight table
  of synth.model_param_specs(model) is the one of oracle.param_specs(net)."""
  model = NETS[net][0](make_mc(net, width, height, batch), device, math_mode=math_mode)
  weights = synth.synthetic_weights(synth.model_param_specs(model), seed=seed)
  model.load_weights(weights)
  return model, weights


class TableNet(FireNetBase):
  """FireNetBase over any BODY.  Conv rows named in `bn_convs` become _conv_bn_layer (conv +
  bias + frozen BN + ReLU, ResNet-50's first layer)."""

  def __init__(self, mc, body, bn_convs=(), gpu_id=0, math_mode=None):
    self.BODY = tuple(body)
    self.bn_convs = set(bn_convs)
    FireNetBase.__init__(self, mc, gpu_id, math_mode)

  def _conv_layer(self, layer_name, inputs, filters, size, stride, padding='SAME', **kw):
    if layer_name in self.bn_convs:
      return self._conv_bn_layer(inputs, layer_name, 'bn_' + layer_name, 'scale_' + layer_name,
                                 filters, size, stride, padding, relu=True, conv_with_bias=True)
    return FireNetBase._conv_layer(self, layer_name, inputs, filters, size, stride, padding, **kw)


def body_grid(body, height, width):
  """(H, W) of the body's last tensor (= the ConvDet head's grid)."""
  h, w = height, width
  for row in body:
    if row[0] in ('conv', 'pool'):
      k, s, pad = row[-3:]
      h = oracle.conv_geometry(h, k, s, pad)[0]
      w = oracle.conv_geometry(w, k, s, pad)[0]
  return h, w


def build(body, batch, height, width, math_mode, device, bn_convs=()):
  """(mc, model, weights) of a TableNet over `body` with synthetic weights."""
  mc = cfg.kitti_squeezeDet_config()
  mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = width, height, batch
  mc.GRID_H, mc.GRID_W = body_grid(body, height, width)
  mc.ANCHOR_BOX = cfg.set_anchors(mc)
  mc.ANCHORS = len(mc.ANCHOR_BOX)
  model = TableNet(mc, body, bn_convs, device, math_mode=math_mode)
  weights = synth.synthetic_weights(synth.model_param_specs(model), seed=7)
  model.load_weights(weights)
  return mc, model, weights


def engine_tensor(model, name):
  """Handle of any engine tensor by name, including ones the Python net does not register
  (a fire's squeeze output)."""
  lib = model._lib
  buf = C.create_string_buffer(256)
  for tid in range(lib.sqdet_num_tensors(model._engine)):
    _lib.check(lib.sqdet_tensor_info(model._engine, tid, buf, 256, None))
    if buf.value.decode() == name:
      return model._new_tensor(name, tid)
  raise KeyError(name)


def read_tensors(model, names):
  return {nm: model.read_tensor(engine_tensor(model, nm)) for nm in names}


def assert_fused_away(model, name):
  with pytest.raises(_lib.SqdetError) as exc:
    model.read_tensor(engine_tensor(model, name))
  assert exc.value.code == ERR_NOT_FOUND, exc.value


def forward_n(model, images, n=None, stream=None):
  """forward_device of the first n images (all with n = None) from a device buffer that holds
  just those images, then a sync of `stream` (None: the legacy stream, never graph-captured)."""
  x = images if n is None else images[:n]
  buf = DeviceBuffer.from_numpy(np.ascontiguousarray(x, np.float32), model.gpu_id)
  model.forward_device(buf.ptr, stream, n)
  _lib.check(model._lib.sqdet_stream_sync(model.gpu_id, stream))
  buf.free()


def assert_rows_equal(got, full, n, *what):
  """Rows [0, n) of each array of an n-image forward bitwise those of the full forward."""
  for key, want in full.items():
    assert got[key][:n].tobytes() == want[:n].tobytes(), (key, n) + what


RESULTS = (('det_boxes', np.float32, 4), ('det_probs', np.float32, None),
           ('det_class', np.int64, None))


def fetch_results(model, device):
  """Every device result buffer of the engine, all B rows."""
  B, A = model.det_probs.shape
  res = model.results_device()
  lib = model._lib
  out = {}
  for key, dtype, last in RESULTS:
    out[key] = np.empty((B, A, last) if last else (B, A), dtype)
  out['dets'] = np.empty((B, res['max_dets']), _lib.DET_DTYPE)
  out['counts'] = np.empty((B,), np.int32)
  _lib.check(lib.sqdet_stream_sync(device, None))
  for key, arr in out.items():
    _lib.check(lib.sqdet_memcpy_d2h(arr.ctypes.data, res[key], arr.nbytes, None))
  _lib.check(lib.sqdet_stream_sync(device, None))
  return out


# ---- the per-element fp64 bound ------------------------------------------------------------------
# Forward-error bar in units of sum |products|, for K products per output: fp32 round-to-nearest
# accumulation random-walks to ~ sqrt(K) * 2^-24 (measured 2.7e-6 at K = 2304 on all-positive
# operands with the FFMA kernel); the 3xTF32 path drops terms of 2^-21 per product.  One bar for
# both math modes:
def adv_tol(K):
  return 1.2e-7 * np.sqrt(K)


def bound_ratio(got, want64, bar):
  """|got - want64| / bar per element: 0 where the error is 0, inf where got is NaN or a non-zero
  error meets a zero bar."""
  err = np.abs(np.asarray(got, np.float64) - want64)
  with np.errstate(divide='ignore', invalid='ignore'):
    ratio = np.where(err > 0, err / bar, 0.0)
  ratio[np.isnan(err)] = np.inf
  return ratio


def assert_within_bound(got, want64, bar, K, what):
  """|got - want64| < adv_tol(K) * bar everywhere; a failure names the worst element."""
  ratio = bound_ratio(got, want64, bar)
  worst = np.unravel_index(np.argmax(ratio), ratio.shape)
  assert ratio[worst] < adv_tol(K), (what, 'element', tuple(int(i) for i in worst),
                                     float(ratio[worst]), adv_tol(K))


def conv_oracle(x, w, b=None, stride=1, padding='SAME', relu=False, scale=None, shift=None):
  """(fp64 conv, its bar): relu?(conv(x, w) + b) [* scale + shift], and |x| (*) |w| + |b|
  [* |scale| + |shift|], the scale that bounds any fp32 summation of the products.  ReLU is
  1-Lipschitz, so it leaves the bar as it is."""
  want = oracle.conv2d(x, w, b, stride, padding, False, np.float64)
  bar = oracle.conv2d(np.abs(x), np.abs(w), None if b is None else np.abs(b), stride, padding,
                      False, np.float64)
  if scale is not None:
    want, bar = want * scale + shift, bar * np.abs(scale) + np.abs(shift)
  if relu:
    want = np.maximum(want, 0)
  return want, bar


def fire_oracle(x, ws, bs, w1, b1, w3, b3, dtype):
  q = oracle.conv2d(x, ws, bs, 1, 'SAME', True, dtype)
  a = oracle.conv2d(q, w1, b1, 1, 'SAME', True, dtype)
  b = oracle.conv2d(q, w3, b3, 1, 'SAME', True, dtype)
  return np.concatenate([a, b], axis=3)


def fire_error_bound(x, ws, w1, w3, q64):
  """Per-element scale of the error of squeeze -> ReLU -> expand in any fp32 summation order:
  the expand's own rounding, tol * (|q| (*) |w_e|), plus the squeeze's error carried through the
  expand, tol * ((|x| (*) |w_s|) (*) |w_e|); ReLU is 1-Lipschitz, so it cannot amplify the
  squeeze error."""
  def conv(a, w):
    return oracle.conv2d(a, w, None, 1, 'SAME', False, np.float64)
  sx = conv(np.abs(x), np.abs(ws))
  return np.concatenate([conv(np.abs(q64), np.abs(w1)) + conv(sx, np.abs(w1)),
                         conv(np.abs(q64), np.abs(w3)) + conv(sx, np.abs(w3))], axis=3)


# ---- detections ----------------------------------------------------------------------------------
def assert_boxes_close(got, ref32, ref64):
  """Box coordinates: within 1e-4 relative of the fp32 reference, plus the reference's OWN
  fp32 uncertainty (|ref32 - ref64|, x4) — boxes that clip from ~4000 px wide pre-clip values
  carry ~1e-3 px of fp32 rounding in any implementation — plus 4e-3 px absolute (3e-6 of the
  image width)."""
  got = np.asarray(got, np.float64)
  tol = TOL * np.abs(ref32) + 4.0 * np.abs(np.asarray(ref32, np.float64) - ref64) + 4e-3
  bad = np.abs(got - ref32) > tol
  assert not bad.any(), (int(bad.sum()), float(np.abs(got - ref32)[bad].max()))


def make_png(path, h, w, seed):
  """A frame with structure (rectangles on noise) so detections spread over the image."""
  import cv2
  rng = np.random.default_rng(seed)
  im = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
  for _ in range(12):
    y0, x0 = int(rng.integers(0, h - 40)), int(rng.integers(0, w - 80))
    im[y0:y0 + int(rng.integers(20, 120)), x0:x0 + int(rng.integers(40, 300))] = \
        rng.integers(0, 256, 3, dtype=np.uint8)
  assert cv2.imwrite(path, im)
  return im


def make_kitti(root):
  """A KITTI tree under `root` of three full-size frames, each with one label: (data directory,
  image ids, {id: frame})."""
  data = root / 'KITTI'
  (data / 'training' / 'image_2').mkdir(parents=True)
  (data / 'training' / 'label_2').mkdir(parents=True)
  (data / 'ImageSets').mkdir()
  ids, frames = [], {}
  for k, (h, w) in enumerate([(375, 1242), (370, 1224), (376, 1241)]):
    idx = '%06d' % k
    ids.append(idx)
    frames[idx] = make_png(str(data / 'training' / 'image_2' / (idx + '.png')), h, w, seed=20 + k)
    (data / 'training' / 'label_2' / (idx + '.txt')).write_text(
        'Car 0.00 0 -1.57 100.00 120.00 300.00 250.00 1.5 1.6 3.9 1.0 1.7 10.0 -1.5\n')
  (data / 'ImageSets' / 'val.txt').write_text('\n'.join(ids) + '\n')
  return data, ids, frames


def oracle_pipeline(net, mc, weights, frame_u8, order, rescale):
  """The reference pipeline on one frame: oracle pre-processing (pinned to cv2) -> torch-CPU
  forward -> interpret_output -> [rescale ALL boxes, eval.py:83-84] -> filter_prediction.
  Returns the filtered (boxes, probs, classes) and whether the top-66 scores hold a near tie."""
  fed = preproc.preprocess(frame_u8, mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BGR_MEANS, order)
  preds = TorchForward(net, weights)(fed[None])
  boxes, probs, cls = oracle.interpret_output(preds, mc.ANCHOR_BOX, mc.CLASSES,
                                              mc.ANCHOR_PER_GRID, mc.IMAGE_WIDTH,
                                              mc.IMAGE_HEIGHT, mc.EXP_THRESH)
  boxes, probs, cls = boxes[0].copy(), probs[0], cls[0]
  if rescale:
    # eval.py:72-74,83-84 (scales are Python floats; numpy divides the float32 array in float32)
    x_scale = mc.IMAGE_WIDTH / float(frame_u8.shape[1])
    y_scale = mc.IMAGE_HEIGHT / float(frame_u8.shape[0])
    boxes[:, 0::2] /= x_scale
    boxes[:, 1::2] /= y_scale
  fb, fp, fc, src = oracle.filter_prediction(boxes, probs, cls, mc.CLASSES, mc.TOP_N_DETECTION,
                                             mc.PROB_THRESH, mc.NMS_THRESH)
  order66 = np.argsort(-probs.astype(np.float64), kind='stable')[:66]
  top = probs[order66].astype(np.float64)
  gap = np.abs(top[:, None] - top[None, :]) <= 10 * TOL * top[:, None]
  np.fill_diagonal(gap, False)
  return fb, fp, fc, bool(gap.any())


# ---- stage-isolated calls ------------------------------------------------------------------------
def conv2d_gpu(x, w, b=None, stride=1, padding='SAME', relu=True, scale=None, shift=None,
               y_cstride=None, y_coff=0, math_mode=0, device=0, y_init=None):
  lib = _lib.load()
  B, H, W, Cin = x.shape
  k, _, _, Cout = w.shape
  Ho = oracle.conv_geometry(H, k, stride, padding)[0]
  Wo = oracle.conv_geometry(W, k, stride, padding)[0]
  cs = y_cstride or Cout
  dx = DeviceBuffer.from_numpy(x.astype(np.float32), device)
  dw = DeviceBuffer.from_numpy(w.astype(np.float32), device)
  db = DeviceBuffer.from_numpy(b.astype(np.float32), device) if b is not None else None
  dsc = DeviceBuffer.from_numpy(scale.astype(np.float32), device) if scale is not None else None
  dsh = DeviceBuffer.from_numpy(shift.astype(np.float32), device) if shift is not None else None
  y0 = y_init if y_init is not None else np.full((B, Ho, Wo, cs), np.nan, np.float32)
  dy = DeviceBuffer.from_numpy(y0, device)
  _lib.check(lib.sqdet_conv2d(dx.ptr, dw.ptr, db.ptr if db else None, dsc.ptr if dsc else None,
                              dsh.ptr if dsh else None, dy.ptr, B, H, W, Cin, Cout, k, stride,
                              _lib.pad_code(padding), int(relu), cs, y_coff, math_mode, None))
  _lib.check(lib.sqdet_stream_sync(device, None))
  return dy.to_numpy(np.float32, (B, Ho, Wo, cs))


def maxpool_gpu(x, k, stride, padding, device=0, offset=0):
  """sqdet_maxpool_nhwc; `offset` > 0 places x and y that many floats into larger buffers (an
  offset of 1 leaves both pointers 4 bytes past 16-byte alignment)."""
  lib = _lib.load()
  B, H, W, Cc = x.shape
  Ho = oracle.conv_geometry(H, k, stride, padding)[0]
  Wo = oracle.conv_geometry(W, k, stride, padding)[0]
  n_out = B * Ho * Wo * Cc
  dx = DeviceBuffer.from_numpy(np.concatenate([np.zeros(offset, np.float32),
                                               x.astype(np.float32).ravel()]), device)
  dy = DeviceBuffer.from_numpy(np.full(offset + n_out, np.nan, np.float32), device)
  _lib.check(lib.sqdet_maxpool_nhwc(dx.ptr + 4 * offset, dy.ptr + 4 * offset, B, H, W, Cc, k,
                                    stride, _lib.pad_code(padding), None))
  y = dy.to_numpy(np.float32, (offset + n_out,))
  assert np.isnan(y[:offset]).all()
  return y[offset:].reshape(B, Ho, Wo, Cc)


def interpret_gpu(preds, anchors_f64, K, classes, img_w, img_h, exp_thresh=1.0, device=0):
  lib = _lib.load()
  B, gh, gw, _ = preds.shape
  A = gh * gw * K
  dp = DeviceBuffer.from_numpy(preds.astype(np.float32), device)
  da = DeviceBuffer.from_numpy(np.asarray(anchors_f64, np.float64).astype(np.float32), device)
  db = DeviceBuffer(B * A * 16, device)
  dpr = DeviceBuffer(B * A * 4, device)
  dc = DeviceBuffer(B * A * 8, device)
  _lib.check(lib.sqdet_interpret(dp.ptr, da.ptr, db.ptr, dpr.ptr, dc.ptr, B, gh, gw, K, classes,
                                 img_w, img_h, C.c_float(exp_thresh), None))
  return (db.to_numpy(np.float32, (B, A, 4)), dpr.to_numpy(np.float32, (B, A)),
          dc.to_numpy(np.int64, (B, A)))


def topk_nms_gpu(boxes, probs, cls, classes, top_n, prob_thresh, nms_thresh, max_dets=None,
                 device=0):
  """boxes [B,A,4] probs [B,A] cls [B,A] -> (dets [B,max_dets], counts [B])."""
  lib = _lib.load()
  boxes = np.ascontiguousarray(boxes, np.float32)
  B, A = probs.shape
  if max_dets is None:
    max_dets = top_n if 0 < top_n < A else min(A, 1024)
  db = DeviceBuffer.from_numpy(boxes, device)
  dp = DeviceBuffer.from_numpy(np.ascontiguousarray(probs, np.float32), device)
  dc = DeviceBuffer.from_numpy(np.ascontiguousarray(cls, np.int64), device)
  dd = DeviceBuffer(B * max_dets * 28, device)
  dn = DeviceBuffer(B * 4, device)
  _lib.check(lib.sqdet_topk_nms(db.ptr, dp.ptr, dc.ptr, B, A, classes, top_n,
                                C.c_float(prob_thresh), C.c_float(nms_thresh), dd.ptr, dn.ptr,
                                max_dets, None))
  return dd.to_numpy(_lib.DET_DTYPE, (B, max_dets)), dn.to_numpy(np.int32, (B,))


# ---- tiles of whole frames -----------------------------------------------------------------------
def assert_merge_matches_oracle(dets, counts, rows, tiles, n, mc):
  """The merged records of frames [0, n) bitwise those of oracle.tiles.merge_tiles on `rows`."""
  want = oracle_tiles.merge_tiles(rows['det_boxes'], rows['det_probs'], rows['det_class'], tiles,
                                  n, mc.CLASSES, mc.TOP_N_DETECTION, mc.PROB_THRESH, mc.NMS_THRESH)
  for f, (fb, fp, fc, src) in enumerate(want):
    k = int(counts[f])
    assert k == len(src), (f, k, len(src))
    d = dets[f]
    assert d['anchor'][:k].tolist() == src, f
    assert d['cls'][:k].tolist() == list(fc), f
    assert np.asarray(fp, np.float32).tobytes() == d['prob'][:k].tobytes(), f
    got_b = np.stack([d['cx'][:k], d['cy'][:k], d['w'][:k], d['h'][:k]], -1)
    assert np.asarray(fb, np.float32).reshape(-1, 4).tobytes() == got_b.tobytes(), f
    assert_padding(d, k, f)
  return want


def assert_padding(records, k, what):
  """Records [k, max_dets) are padding: anchor and class -1, every float +0.0."""
  pad = records[k:]
  assert (pad['anchor'] == -1).all() and (pad['cls'] == -1).all(), what
  for key in ('prob', 'cx', 'cy', 'w', 'h'):
    assert not pad[key].copy().view(np.uint32).any(), (what, key)


def merge_gpu_rc(boxes, probs, cls, tiles, n, classes, top_n, prob_thresh, nms_thresh, max_dets,
                 device):
  """(return code, dets [n, max_dets], counts [n]) of sqdet_merge_tiles on host rows, tile k =
  tiles[k] = (frame, x, y); the output buffers start as 0x77 bytes and counts 12345."""
  lib = _lib.load()
  t, A = probs.shape
  db = DeviceBuffer.from_numpy(np.ascontiguousarray(boxes, np.float32), device)
  dp = DeviceBuffer.from_numpy(np.ascontiguousarray(probs, np.float32), device)
  dc = DeviceBuffer.from_numpy(np.ascontiguousarray(cls, np.int64), device)
  dd = DeviceBuffer.from_numpy(np.full(n * max_dets * 28, 0x77, np.uint8), device)
  dn = DeviceBuffer.from_numpy(np.full(n, 12345, np.int32), device)
  fr = (C.c_int32 * t)(*[tl[0] for tl in tiles])
  xy = (C.c_int32 * (2 * t))(*[v for tl in tiles for v in tl[1:3]])
  rc = lib.sqdet_merge_tiles(db.ptr, dp.ptr, dc.ptr, A, t, fr, xy, n, classes, top_n,
                             C.c_float(prob_thresh), C.c_float(nms_thresh), dd.ptr, dn.ptr,
                             max_dets, None)
  return rc, dd.to_numpy(_lib.DET_DTYPE, (n, max_dets)), dn.to_numpy(np.int32, (n,))


def merge_gpu(boxes, probs, cls, tiles, n, classes, top_n, prob_thresh, nms_thresh, max_dets,
              device):
  rc, dets, counts = merge_gpu_rc(boxes, probs, cls, tiles, n, classes, top_n, prob_thresh,
                                  nms_thresh, max_dets, device)
  _lib.check(rc)
  return dets, counts


def adversarial_rows(t, A, classes, rng):
  """Tile rows with probabilities tied within and across tiles, +-0, NaN, classes out of range,
  and pairs that meet across tiles at IoU exactly float32(0.4) once the offsets are added."""
  boxes = np.stack([rng.integers(1, 60, (t, A)) + 0.5, rng.integers(1, 30, (t, A)) + 0.5,
                    rng.integers(2, 20, (t, A)).astype(float),
                    rng.integers(2, 20, (t, A)).astype(float)], -1).astype(np.float32)
  probs = rng.choice(np.float32([0.9, 0.5, 0.25, 0.125, 0.0, -0.0, np.nan, 0.75]),
                     (t, A)).astype(np.float32)
  cls = rng.integers(0, classes, (t, A)).astype(np.int64)
  cls[rng.random((t, A)) < 0.05] = -1
  cls[rng.random((t, A)) < 0.05] = classes + 2
  # tile k's anchor 0 at x = 10.5, tile k+1's anchor 1 at 3.5 + 10 (offset): 7-wide boxes 3 apart,
  # IoU 4/10 exactly; top score so the pair survives the top-N cut
  for k in range(0, t - 1, 2):
    boxes[k, 0] = (10.5, 8.5, 7, 7)
    boxes[k + 1, 1] = (3.5, 8.5, 7, 7)
    probs[k, 0], probs[k + 1, 1] = 0.9, 0.9
    cls[k, 0] = cls[k + 1, 1] = 1
  return boxes, probs, cls


def rel_err(got, want):
  """max |got-want| / max|want| — the per-tensor relative error used for activations."""
  want = np.asarray(want, np.float64)
  return float(np.abs(np.asarray(got, np.float64) - want).max() / max(np.abs(want).max(), 1e-30))


def preprocess_gpu(img_u8, width, height, bgr_means, order, device=0):
  """sqdet_preprocess_u8 on one uint8 [H0, W0, 3] image -> float32 [height, width, 3]."""
  lib = _lib.load()
  img = np.ascontiguousarray(img_u8, np.uint8)
  h0, w0 = img.shape[:2]
  src = DeviceBuffer.from_numpy(img, device)
  dst = DeviceBuffer(height * width * 3 * 4, device)
  means = np.ascontiguousarray(np.asarray(bgr_means, np.float64).reshape(3))
  code = {'demo': 0, 'eval': 1}[order]
  _lib.check(lib.sqdet_preprocess_u8(src.ptr, h0, w0, dst.ptr, height, width, means.ctypes.data,
                                     code, None))
  return dst.to_numpy(np.float32, (height, width, 3))


def class_margin(preds64, anchors_per_grid, classes):
  """Relative top-2 margin of the per-anchor class probabilities, from fp64 oracle preds
  [B,Hg,Wg,K*(C+5)]: (p_top1 - p_top2) / p_top1 (the sigmoid confidence is a common factor).
  An argmax may legitimately differ from the oracle's only where this is below fp noise."""
  p = np.asarray(preds64, np.float64)
  B = p.shape[0]
  K, C = anchors_per_grid, classes
  logits = p[..., :K * C].reshape(B, -1, C)
  z = logits - logits.max(axis=2, keepdims=True)
  e = np.exp(z)
  pr = e / e.sum(axis=2, keepdims=True)
  top = np.sort(pr, axis=2)
  if C == 1:
    return np.ones(pr.shape[:2])
  return (top[..., -1] - top[..., -2]) / top[..., -1]


def assert_classes_match(got_cls, want_cls, preds64, anchors_per_grid, classes, tol):
  """north_star: class ids bit-exact.  A mismatch is tolerated ONLY where the fp64 oracle's
  own top-2 class margin is below 10*tol (a near tie that fp32 rounding may order either way);
  returns the number of such near-tie mismatches."""
  mism = np.asarray(got_cls) != np.asarray(want_cls)
  if not mism.any():
    return 0
  margin = class_margin(preds64, anchors_per_grid, classes)
  bad = mism & (margin >= 10 * tol)
  assert not bad.any(), ('class id differs outside a near tie', int(bad.sum()),
                         float(margin[bad].max()))
  return int(mism.sum())


def fire_gpu(x, wsq, bsq, we1, be1, we3, be3, math_mode=1, device=0):
  """sqdet_fire on host arrays: x [B,H,W,Cin], HWIO kernels -> y [B,H,W,E1+E3]."""
  lib = _lib.load()
  B, H, W, Cin = x.shape
  S, E1, E3 = wsq.shape[3], we1.shape[3], we3.shape[3]
  bufs = [DeviceBuffer.from_numpy(np.ascontiguousarray(a, np.float32), device)
          for a in (x, wsq, bsq, we1, be1, we3, be3)]
  y0 = np.full((B, H, W, E1 + E3), np.nan, np.float32)
  dy = DeviceBuffer.from_numpy(y0, device)
  _lib.check(lib.sqdet_fire(*[b.ptr for b in bufs], dy.ptr, B, H, W, Cin, S, E1, E3,
                            int(math_mode), None))
  _lib.check(lib.sqdet_stream_sync(device, None))
  return dy.to_numpy(np.float32, y0.shape)


# ---- JPEG encoder tests ------------------------------------------------------------------------
def content(kind, h, w, c, rng):
  """uint8 [h, w, c] test content: noise, gradients, flat, 0/255 checkerboards of pixels (the
  largest AC coefficients, ZRL at low quality) or of 8x8 blocks (DC differences of category 11),
  or isolated dots on flat grey."""
  if kind == 'noise':
    return rng.integers(0, 256, (h, w, c), dtype=np.uint8)
  y, x = np.mgrid[:h, :w]
  if kind == 'grad':
    return ((y[..., None] * 3 + x[..., None] * 5 + np.arange(c) * 40) % 256).astype(np.uint8)
  if kind == 'flat':
    return np.full((h, w, c), 77, np.uint8)
  if kind in ('check', 'blocks'):     # 0/255 per pixel, or per 8x8 block (DC category 11)
    cell = (y + x) % 2 if kind == 'check' else (y // 8 + x // 8) % 2
    return np.repeat((cell * 255).astype(np.uint8)[..., None], c, axis=2)
  img = np.full((h, w, c), 128, np.uint8)
  img[(y % 8 == 7) & (x % 8 == 7)] = 255
  return img


class Frame:
  """One frame in `fmt` (an h x w image; 4:2:0 formats need even sizes) on the device, with rows
  `pad` bytes longer than tight and starting `off` bytes into their allocation, and its BGR image
  as cv2.cvtColor makes it."""

  def __init__(self, fmt, h, w, rng, device, kind='noise', pad=0, off=0):
    import cv2
    import torch
    self.fmt = fmt
    if fmt in ('bgr', 'rgb', 'bgra', 'rgba'):
      c = 4 if fmt in ('bgra', 'rgba') else 3
      host = content(kind, h, w, c, rng)
      code = {'bgr': None, 'rgb': cv2.COLOR_RGB2BGR, 'bgra': cv2.COLOR_BGRA2BGR,
              'rgba': cv2.COLOR_RGBA2BGR}[fmt]
      self.bgr = host if code is None else cv2.cvtColor(host, code)
      self.dev = self._pitched(host.reshape(h, w * c), pad, off, device).unflatten(1, (w, c))
    elif fmt == 'rgb_planar':
      host = content(kind, h, w, 3, rng)
      self.bgr = cv2.cvtColor(host, cv2.COLOR_RGB2BGR)
      self.dev = tuple(self._pitched(np.ascontiguousarray(host[..., i]), pad, off, device)
                       for i in range(3))
    else:
      host = content(kind, h * 3 // 2, w, 1, rng)[..., 0]
      code = cv2.COLOR_YUV2BGR_NV12 if fmt == 'nv12' else cv2.COLOR_YUV2BGR_I420
      self.bgr = cv2.cvtColor(host, code)
      if fmt == 'nv12':
        self.dev = (self._pitched(host[:h], pad, off, device),
                    self._pitched(host[h:], pad, off, device))
      else:
        self.dev = torch.from_numpy(host).to(device)

  @staticmethod
  def _pitched(a, pad, off, device):
    import torch
    rows, cols = a.shape
    buf = torch.zeros(off + rows * (cols + pad), dtype=torch.uint8, device=device)
    t = buf[off:].view(rows, cols + pad)[:, :cols]
    t.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    return t


def want(frame, crop, quality):
  """cv2.imencode's file of `frame`'s BGR image cropped to (x, y, w, h) at `quality`."""
  import cv2
  x, y, w, h = crop
  return cv2.imencode('.jpg', np.ascontiguousarray(frame.bgr[y:y + h, x:x + w]),
                      [cv2.IMWRITE_JPEG_QUALITY, quality])[1].tobytes()


def raw_encode(frames, cap, quality=95, stream=None):
  """sqdet_encode_jpeg of BGR device frames at capacity cap -> (data, lengths, scratch)."""
  import torch
  lib = _lib.load()
  n = len(frames)
  planes = (C.c_void_p * (3 * n))(*sum([[f.data_ptr(), None, None] for f in frames], []))
  hs = (C.c_int32 * n)(*[f.shape[0] for f in frames])
  ws = (C.c_int32 * n)(*[f.shape[1] for f in frames])
  sb = lib.sqdet_jpeg_scratch_bytes(n, hs, ws, None)
  dev = frames[0].device
  data = torch.zeros((n, cap), dtype=torch.uint8, device=dev)
  lengths = torch.zeros((n,), dtype=torch.int64, device=dev)
  scratch = torch.empty((sb,), dtype=torch.uint8, device=dev)
  _lib.check(lib.sqdet_encode_jpeg(n, 0, planes, None, hs, ws, None, quality, data.data_ptr(), cap,
                                   lengths.data_ptr(), scratch.data_ptr(), sb, stream))
  return data, lengths, scratch
