"""Kernel branches outside the convolution tables, each against a plain reference:
  * filter_kernel at its capacity edges (registers vs L2 for the top-n scores, the 1024-record
    threshold branch, max_dets, class ids outside [0, classes)), bit-exact against
    oracle.filter_prediction;
  * add_relu_kernel's float4 body, tail and unaligned paths, including an add+ReLU whose operand
    is the image input and therefore reads the caller's images buffer;
  * sqdet_conv2d argument validation, the same in both math modes.
tests/test_host_logic.py restates each branch predicate and checks that the tables below reach
every branch."""
import numpy as np
import pytest

import oracle
from squeezedet_b200 import _lib
from squeezedet_b200 import config as cfg
from squeezedet_b200.nn_skeleton import ModelSkeleton
from squeezedet_b200.utils import synth
from gpu_util import fetch_results, make_net, topk_nms_gpu

pytestmark = pytest.mark.gpu
ERR_INVALID_ARG = -1
PROB_THRESH, NMS_THRESH, CLASSES = 0.005, 0.4, 3

# ---- filter_prediction capacity edges -----------------------------------------------------------
FILTER_CASES = [
    # A, top_n, candidates above PROB_THRESH (threshold branch) or None, max_dets (None: the
    # helper's default), quantised scores, class ids drawn from [0, CLASSES] (CLASSES is invalid)
    # top-n branch around the 24 scores per thread that stay in registers (A <= 24576)
    (24576, 64, None, None, False, False), (24576, 64, None, None, True, False),
    (24577, 64, None, None, False, False), (24577, 64, None, None, True, False),
    (43200, 64, None, None, False, True), (43200, 64, None, None, True, False),
    (43200, 1024, None, None, True, True),
    # top_n from 1 to the 1024-record limit, and A - 1
    (16848, 1, None, None, False, False), (16848, 64, None, None, True, True),
    (16848, 513, None, None, False, False), (16848, 1024, None, None, True, False),
    (300, 299, None, None, True, True),
    # threshold branch at its capacity: min(1024, max_dets) records kept, one more overflows
    (3000, 0, 1024, 1024, False, False), (3000, 0, 1025, 1024, False, False),
    (3000, 0, 100, 100, True, True), (3000, 0, 101, 100, False, False),
]


def filter_inputs(A, top_n, n_above, quantised, bad_cls, seed):
  rng = np.random.default_rng(seed)
  boxes = np.stack([rng.uniform(0, 1242, A), rng.uniform(0, 375, A), rng.uniform(4, 60, A),
                    rng.uniform(4, 40, A)], 1).astype(np.float32)
  if n_above is None:
    probs = rng.uniform(0, 1, A)
    if quantised:                  # few distinct values: long tie runs across the radix threshold
      probs = np.round(probs * 4) / 4
  else:
    probs = rng.uniform(0, 0.004, A)
    above = rng.permutation(A)[:n_above]
    probs[above] = np.round(rng.uniform(0.5, 1, n_above) * 8) / 8 if quantised else \
        rng.uniform(0.5, 1, n_above)
  cls = rng.integers(0, CLASSES + (1 if bad_cls else 0), A).astype(np.int64)
  return boxes, probs.astype(np.float32), cls


def check_filter(dets, count, boxes, probs, cls, top_n, max_dets):
  """The record layout the GPU filter writes against oracle.filter_prediction, bit-exact."""
  fb, fp, fc, src = oracle.filter_prediction(boxes, probs, cls, CLASSES, top_n, PROB_THRESH,
                                             NMS_THRESH)
  if not 0 < top_n < len(probs) and (probs > PROB_THRESH).sum() > min(1024, max_dets):
    assert count == -1                        # reported, not truncated
    assert np.all(dets['anchor'] == -1)
    return
  n = len(src)
  assert count == n, (count, n)
  d = dets[:n]
  assert d['anchor'].tolist() == src
  assert d['cls'].tolist() == fc
  assert all(0 <= c < CLASSES for c in fc)
  assert np.array_equal(d['prob'], np.asarray(fp, np.float32).reshape(n))
  got = np.stack([d['cx'], d['cy'], d['w'], d['h']], 1)
  assert np.array_equal(got, np.asarray(fb, np.float32).reshape(n, 4))
  assert np.all(dets[n:]['anchor'] == -1)


@pytest.mark.parametrize('case', FILTER_CASES)
def test_filter_capacity_edges(case, gpu_device):
  A, top_n, n_above, max_dets, quantised, bad_cls = case
  boxes, probs, cls = filter_inputs(A, top_n, n_above, quantised, bad_cls, seed=A + top_n)
  dets, counts = topk_nms_gpu(boxes[None], probs[None], cls[None], CLASSES, top_n, PROB_THRESH,
                              NMS_THRESH, max_dets=max_dets)
  check_filter(dets[0], int(counts[0]), boxes, probs, cls, top_n, dets.shape[1])


def test_full_squeezedet_1600x480_uncached_filter(gpu_device):
  """SqueezeDet at 1600x480 has 27000 anchors, past the 24576 whose scores the filter keeps in
  registers: the GPU filter on the engine's own det tensors equals the oracle's on them."""
  model, _ = make_net('squeezeDet', 1600, 480, 1, gpu_device, seed=0)
  mc = model.mc
  assert mc.ANCHORS == 27000
  images = synth.synthetic_images(1, 480, 1600, seed=77)
  boxes, probs, cls, dets, counts = model.detect(images, want_dets=True)
  assert 0 < mc.TOP_N_DETECTION < mc.ANCHORS
  fb, fp, fc, src = oracle.filter_prediction(boxes[0], probs[0], cls[0], mc.CLASSES,
                                             mc.TOP_N_DETECTION, mc.PROB_THRESH, mc.NMS_THRESH)
  n = int(counts[0])
  assert n == len(src) > 0
  assert dets[0]['anchor'][:n].tolist() == src
  assert dets[0]['cls'][:n].tolist() == fc
  assert np.array_equal(dets[0]['prob'][:n], np.asarray(fp, np.float32))


# ---- add+ReLU: image operand, float4 body, tail, unaligned --------------------------------------
class AddReluNet(ModelSkeleton):
  """body 'image': mix = conv1x1(image, 3 -> 3), res = relu(image + mix);
  body 'conv':  conv1 = conv3x3(image, 8), mix = conv1x1(conv1, 8 -> 8), res = relu(conv1 + mix);
  then conv2 (3x3, 32) and the 72-channel ConvDet head."""

  def __init__(self, mc, body, gpu_id=0, math_mode=None):
    ModelSkeleton.__init__(self, mc, gpu_id, math_mode)
    x = self.image_input
    if body == 'conv':
      x = self._conv_layer('conv1', x, filters=8, size=3, stride=1)
    mix = self._conv_layer('mix', x, filters=x.shape[3], size=1, stride=1, relu=False)
    res = self._add_relu('res', x, mix)
    y = self._conv_layer('conv2', res, filters=32, size=3, stride=1)
    self.preds = self._conv_layer('conv12', y, filters=mc.ANCHOR_PER_GRID * (mc.CLASSES + 5),
                                  size=3, stride=1, relu=False)
    self._add_interpretation_graph()


ADD_RELU_CASES = [
    # body, B, H, W, images offset in floats inside the caller's buffer (None: detect(), which
    # runs on the engine's own input buffer)
    ('image', 1, 9, 15, None),     # n = 405: float4 body + tail
    ('conv', 2, 8, 12, None),      # 8-channel conv operands, n = 1536: float4 body only
    ('image', 2, 9, 15, 0),        # caller's images, 16-byte aligned: float4 body + tail
    ('image', 2, 9, 15, 1),        # caller's images one float past alignment: scalar path
]
ADD_RELU_CHANNELS = {'image': 3, 'conv': 8}


def small_mc(batch, height, width):
  mc = cfg.kitti_squeezeDet_config()
  mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = width, height, batch
  mc.GRID_H, mc.GRID_W = height, width
  mc.ANCHOR_BOX = cfg.set_anchors(mc)
  mc.ANCHORS = len(mc.ANCHOR_BOX)
  return mc


def activations(model):
  return {n: model.read_tensor(n) for n in ('mix', 'res', 'conv2', 'conv12')}


def check_add_relu(model, body, images):
  """res == max(x + mix, 0) in float32, with x the images fed (body 'image') or conv1."""
  x = images if body == 'image' else model.read_tensor('conv1')
  mix = model.read_tensor('mix')
  want = np.maximum(np.asarray(x, np.float32) + mix, np.float32(0))
  assert np.array_equal(model.read_tensor('res'), want)


@pytest.mark.parametrize('case', ADD_RELU_CASES)
def test_add_relu_paths(case, gpu_device):
  body, B, H, W, offset = case
  model = AddReluNet(small_mc(B, H, W), body, gpu_device)
  model.load_weights(synth.synthetic_weights(synth.model_param_specs(model), seed=5))
  images = synth.synthetic_images(B, H, W, seed=6)
  if offset is None:
    model.detect(images)
    check_add_relu(model, body, images)
    return
  # the engine's own input tensor holds other images, so an operand read from it would show
  model.detect(synth.synthetic_images(B, H, W, seed=7))

  def forward_at(off):
    """forward_device on the images `off` floats into a larger buffer."""
    flat = np.concatenate([np.zeros(off, np.float32), images.ravel(), np.zeros(3, np.float32)])
    buf = _lib.DeviceBuffer.from_numpy(flat, gpu_device)
    model.forward_device(buf.ptr + 4 * off)
    _lib.check(model._lib.sqdet_stream_sync(gpu_device, None))
    buf.free()
    check_add_relu(model, body, images)
    return fetch_results(model, gpu_device), activations(model)

  want_res, want_act = forward_at(0)
  if offset:
    # nothing requires 16-byte aligned images: the offset forward is bitwise the aligned one
    got_res, got_act = forward_at(offset)
    for key in want_res:
      assert got_res[key].tobytes() == want_res[key].tobytes(), key
    for key in want_act:
      assert got_act[key].tobytes() == want_act[key].tobytes(), key


# ---- conv argument validation -------------------------------------------------------------------
BAD_EPILOGUES = [
    # y_cstride, y_coff, scale given, shift given (Cout = 72)
    (72, 1, False, False), (80, -1, False, False), (71, 0, False, False), (72, 0, True, False),
    (72, 0, False, True)]


@pytest.mark.parametrize('entry', ['conv2d_simt', 'conv2d_tc'])
@pytest.mark.parametrize('bad', BAD_EPILOGUES)
def test_conv_rejects_bad_epilogue(entry, bad, gpu_device):
  """A channel window outside [0, y_cstride) or an unpaired scale / shift is refused with
  SQDET_ERR_INVALID_ARG in every math mode, before anything is written.  y sits 256 floats into a
  sentinel-filled buffer, so a kernel that ran anyway would write inside the allocation."""
  cs, coff, has_scale, has_shift = bad
  lib = _lib.load()
  B, H, W, Cin, Cout, pad = 1, 12, 20, 32, 72, 256
  rng = np.random.default_rng(3)
  dx = _lib.DeviceBuffer.from_numpy(rng.normal(size=(B, H, W, Cin)).astype(np.float32), gpu_device)
  dw = _lib.DeviceBuffer.from_numpy(rng.normal(size=(3, 3, Cin, Cout)).astype(np.float32),
                                    gpu_device)
  vec = [_lib.DeviceBuffer.from_numpy(rng.normal(size=Cout).astype(np.float32), gpu_device)
         for _ in range(3)]
  sentinel = np.full(2 * pad + B * H * W * cs, 7.0, np.float32)
  dy = _lib.DeviceBuffer.from_numpy(sentinel, gpu_device)
  sc = vec[1].ptr if has_scale else None
  sh = vec[2].ptr if has_shift else None
  y = dy.ptr + 4 * pad
  mode = _lib.MATH_FP32_SIMT if entry == 'conv2d_simt' else _lib.MATH_TF32X3_TC
  rc = lib.sqdet_conv2d(dx.ptr, dw.ptr, vec[0].ptr, sc, sh, y, B, H, W, Cin, Cout, 3, 1, 0, 1, cs,
                        coff, mode, None)
  assert rc == ERR_INVALID_ARG, (rc, lib.sqdet_last_error())
  _lib.check(lib.sqdet_stream_sync(gpu_device, None))
  assert dy.to_numpy(np.float32, sentinel.shape).tobytes() == sentinel.tobytes()
