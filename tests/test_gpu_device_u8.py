"""sqdet_forward_u8: uint8 BGR batches already in device memory.  Every check is bitwise against
sqdet_forward_n on float32(float64(u8) - BGR_MEANS): det_boxes, det_probs, det_class, the records,
the counts and every materialised activation.  Where a fused conv+pool first layer is the only
reader of the image tensor, that kernel reads the bytes itself and tensor 0 is left alone;
elsewhere one launch converts the batch into tensor 0 first."""
import ctypes as C

import numpy as np
import pytest

from gpu_util import (ERR_NOT_FOUND, MODES, build, engine_tensor, fetch_results, forward_n,
                      make_net)
from squeezedet_b200 import _lib
from squeezedet_b200 import config as cfg
from squeezedet_b200._lib import DeviceBuffer
from squeezedet_b200.nn_skeleton import ModelSkeleton
from squeezedet_b200.utils import synth

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_STATE = -1, -4


def converted(u8, means):
  return (u8.astype(np.float64) - np.asarray(means, np.float64).reshape(3)).astype(np.float32)


def random_u8(shape, seed):
  return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def activations(model):
  """Every materialised tensor but the image input, by name."""
  lib = model._lib
  buf = C.create_string_buffer(256)
  out = {}
  for tid in range(1, lib.sqdet_num_tensors(model._engine)):
    _lib.check(lib.sqdet_tensor_info(model._engine, tid, buf, 256, None))
    name = buf.value.decode()
    try:
      out[name] = model.read_tensor(engine_tensor(model, name))
    except _lib.SqdetError as exc:
      assert exc.code == ERR_NOT_FOUND, exc
  return out


def snapshot(model):
  out = {'result/' + k: v for k, v in fetch_results(model, model.gpu_id).items()}
  out.update(activations(model))
  return out


def assert_same(got, want, what, n=None):
  assert got.keys() == want.keys()
  for key in want:
    g, w = (got[key], want[key]) if n is None else (got[key][:n], want[key][:n])
    assert g.tobytes() == w.tobytes(), (key,) + what


def u8_buffer(u8, offset, device):
  """A device buffer holding u8 `offset` bytes in, with sentinels before and after."""
  flat = np.concatenate([np.full(offset, 0xA5, np.uint8), u8.ravel(), np.full(7, 0x5A, np.uint8)])
  return DeviceBuffer.from_numpy(flat, device)


def forward_u8(model, u8, offset=0, n=None, stream=None):
  buf = u8_buffer(u8 if n is None else u8[:n], offset, model.gpu_id)
  model.forward_device_u8(buf.ptr + offset, stream, n)
  _lib.check(model._lib.sqdet_stream_sync(model.gpu_id, stream))
  buf.free()


def reference(model, u8, n=None, stream=None):
  """snapshot after sqdet_forward_n on the converted images."""
  forward_n(model, converted(u8, model.mc.BGR_MEANS), n, stream)
  return snapshot(model)


def image_input(model):
  return model.read_tensor('image_input')


# ---- the fused kernel: all four instances, padding, BN, ragged pooled tiles, both math modes -----
KERNEL_ROWS = [
    # Cout, k, conv padding, pool padding, BN, H, W.  64 channels -> 256 threads, 96 -> 384.
    (64, 3, 'SAME', 'SAME', False, 37, 75),     # conv pads (1, 1) both ways; a row is 225 bytes
    (96, 3, 'SAME', 'VALID', False, 41, 130),   # conv pads rows (1, 1), columns (0, 1)
    (64, 3, 'VALID', 'SAME', False, 5, 6),      # a single pooled pixel
    (96, 3, 'VALID', 'VALID', False, 64, 263),
    (64, 7, 'SAME', 'VALID', True, 45, 99),     # ResNet-50's conv1 + pool1: pads (3, 3)
    (96, 7, 'VALID', 'VALID', False, 20, 50),   # less than one 4 x 16 pooled tile
    (64, 7, 'SAME', 'SAME', False, 32, 258),    # pads (2, 3)
    (96, 7, 'VALID', 'SAME', False, 77, 141),
]
KERNEL_BATCH = 3


@pytest.mark.parametrize('math_mode', MODES)
@pytest.mark.parametrize('row', KERNEL_ROWS, ids=lambda r: '%dc-k%d-%s-%s%s-%dx%d' % (
    r[0], r[1], r[2], r[3], '-bn' if r[4] else '', r[5], r[6]))
def test_fused_first_layer(row, math_mode, gpu_device):
  cout, k, cpad, ppad, bn, height, width = row
  body = [('conv', 'conv1', cout, k, 2, cpad), ('pool', 'pool1', 3, 2, ppad)]
  B = KERNEL_BATCH
  mc, model, _ = build(body, B, height, width, math_mode, gpu_device, ('conv1',) if bn else ())
  feed = synth.synthetic_images(B, height, width, seed=3)
  model.detect(feed)
  u8 = random_u8((B, height, width, 3), seed=height * width + cout)
  want = reference(model, u8)
  for offset in (0, 3):
    forward_u8(model, u8, offset)
    assert_same(snapshot(model), want, ('offset', offset))
  # the kernel read the bytes: tensor 0 still holds the detect() feed
  assert image_input(model).tobytes() == feed.tobytes()


# ---- the four benchmark nets at full size -------------------------------------------------------
FULL_NETS = ['squeezeDet', 'squeezeDet+', 'resnet50', 'vgg16']


@pytest.mark.parametrize('net', FULL_NETS)
def test_full_size_nets(net, gpu_device):
  """B = 3 at 1242x375: image 1 starts 2 mod 4 bytes after image 0, rows alternate between 0 and 2
  mod 4.  The pointer is also moved 1, 2 and 3 bytes into a larger buffer; the forwards run on
  the engine's stream, so through captured graphs."""
  model, _ = make_net(net, 1242, 375, 3, gpu_device)
  mc = model.mc
  feed = synth.synthetic_images(3, 375, 1242, seed=4)
  model.detect(feed)
  stream = model.engine_stream()
  u8 = random_u8((3, 375, 1242, 3), seed=len(net))
  want = reference(model, u8, stream=stream)
  conv = converted(u8, mc.BGR_MEANS)
  for offset in (0, 1, 2, 3):
    forward_u8(model, u8, offset, stream=stream)
    assert_same(snapshot(model), want, (net, 'offset', offset))
    # VGG16's conv1_1 runs on tensor cores in gather mode: that net converts into tensor 0
    assert image_input(model).tobytes() == (conv if net == 'vgg16' else feed).tobytes()


# ---- partial batches, graph cache, means ----------------------------------------------------------
def squeezedet_small(batch, device):
  return build([('conv', 'conv1', 64, 3, 2, 'SAME'), ('pool', 'pool1', 3, 2, 'SAME'),
                ('fire', 'fire2', 16, 64, 64)], batch, 47, 133, _lib.MATH_TF32X3_TC, device)[1]


@pytest.mark.parametrize('fused', [True, False], ids=['fused', 'converted'])
def test_partial_batches(fused, gpu_device):
  """n < B: rows [0, n) bitwise those of the full batch, counts[n:] = 0, on both paths."""
  B = 4
  if fused:
    model = squeezedet_small(B, gpu_device)
  else:
    model = build([('conv', 'conv1', 32, 3, 1, 'SAME'), ('pool', 'pool1', 3, 2, 'SAME')], B, 23,
                  61, _lib.MATH_TF32X3_TC, gpu_device)[1]
  stream = model.engine_stream()
  u8 = random_u8((B, model.mc.IMAGE_HEIGHT, model.mc.IMAGE_WIDTH, 3), seed=9)
  forward_u8(model, u8, 1, stream=stream)
  full = snapshot(model)
  assert_same(full, reference(model, u8, stream=stream), ('full',))
  for n in (1, 3):
    forward_u8(model, u8, 2, n=n, stream=stream)
    got = snapshot(model)
    assert_same(got, full, ('n', n), n)
    assert not got['result/counts'][n:].any()


def test_graph_cache_keys_the_input_type(gpu_device):
  """One device address fed first fp32 images, then uint8 ones, on the same stream: the second
  forward must not replay the first one's graph."""
  model = squeezedet_small(2, gpu_device)
  mc = model.mc
  stream = model.engine_stream()
  shape = (2, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, 3)
  u8 = random_u8(shape, seed=12)
  want = reference(model, u8)
  images = synth.synthetic_images(2, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, seed=13)
  buf = DeviceBuffer.from_numpy(images, gpu_device)
  for _ in range(2):
    model.forward_device(buf.ptr, stream)
  _lib.check(model._lib.sqdet_stream_sync(gpu_device, stream))
  _lib.check(model._lib.sqdet_memcpy_h2d(buf.ptr, u8.ctypes.data, u8.nbytes, None))
  _lib.check(model._lib.sqdet_stream_sync(gpu_device, None))
  model.forward_device_u8(buf.ptr, stream)
  _lib.check(model._lib.sqdet_stream_sync(gpu_device, stream))
  assert_same(snapshot(model), want, ('fp32 then uint8 at one address',))
  buf.free()


@pytest.mark.parametrize('fused', [True, False], ids=['fused', 'converted'])
def test_means_change_between_replays(fused, gpu_device):
  """sqdet_set_bgr_means between two graph-replayed uint8 forwards of one buffer on one stream
  is followed by the second forward."""
  if fused:
    model = squeezedet_small(2, gpu_device)
  else:
    model = build([('conv', 'conv1', 32, 3, 1, 'SAME'), ('pool', 'pool1', 3, 2, 'SAME')], 2, 23,
                  61, _lib.MATH_TF32X3_TC, gpu_device)[1]
  mc = model.mc
  stream = model.engine_stream()
  u8 = random_u8((2, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, 3), seed=14)
  buf = u8_buffer(u8, 0, gpu_device)
  results = []
  for means in (mc.BGR_MEANS, np.array([[[90.5, 101.25, 140.0]]])):
    m = np.ascontiguousarray(np.asarray(means, np.float64).reshape(3))
    _lib.check(model._lib.sqdet_set_bgr_means(model._engine, m.ctypes.data))
    for _ in range(2):                   # capture, then replay
      model.forward_device_u8(buf.ptr, stream)
    _lib.check(model._lib.sqdet_stream_sync(gpu_device, stream))
    got = snapshot(model)
    forward_n(model, converted(u8, m))
    assert_same(got, snapshot(model), ('means', tuple(m)))
    results.append(got)
  assert results[0]['result/det_probs'].tobytes() != results[1]['result/det_probs'].tobytes()
  buf.free()


# ---- which path the plan picks, seen through tensor 0 -------------------------------------------
class ImageAddReluNet(ModelSkeleton):
  """res = relu(image + conv1x1(image)): the image is read by two ops."""

  def __init__(self, mc, gpu_id=0, math_mode=None):
    ModelSkeleton.__init__(self, mc, gpu_id, math_mode)
    x = self.image_input
    mix = self._conv_layer('mix', x, filters=3, size=1, stride=1, relu=False)
    res = self._add_relu('res', x, mix)
    self.preds = self._conv_layer('conv12', res, filters=mc.ANCHOR_PER_GRID * (mc.CLASSES + 5),
                                  size=3, stride=1, relu=False)
    self._add_interpretation_graph()


def add_relu_net(batch, height, width, device):
  mc = cfg.kitti_squeezeDet_config()
  mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = width, height, batch
  mc.GRID_H, mc.GRID_W = height, width
  mc.ANCHOR_BOX = cfg.set_anchors(mc)
  mc.ANCHORS = len(mc.ANCHOR_BOX)
  model = ImageAddReluNet(mc, device)
  model.load_weights(synth.synthetic_weights(synth.model_param_specs(model), seed=5))
  return model


PATH_CASES = {
    # name: (builds the model on a device, image tensor holds the converted batch)
    'conv+pool': (lambda d: squeezedet_small(2, d), False),
    'conv without pool': (lambda d: build([('conv', 'conv1', 16, 3, 2, 'SAME')], 2, 19, 45,
                                          _lib.MATH_FP32_SIMT, d)[1], True),
    'vgg16 conv1_1': (lambda d: build([('conv', 'conv1_1', 64, 3, 1, 'SAME'),
                                       ('pool', 'pool1', 2, 2, 'SAME')], 2, 19, 45,
                                      _lib.MATH_TF32X3_TC, d)[1], True),
    'image add+relu': (lambda d: add_relu_net(2, 9, 15, d), True),
}


@pytest.mark.parametrize('case', sorted(PATH_CASES))
def test_path_choice(case, gpu_device):
  make, converts = PATH_CASES[case]
  model = make(gpu_device)
  mc = model.mc
  B, H, W = mc.BATCH_SIZE, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH
  feed = synth.synthetic_images(B, H, W, seed=8)
  model.detect(feed)
  u8 = random_u8((B, H, W, 3), seed=15)
  want = reference(model, u8)
  base = model.launches_per_forward()
  for offset in (0, 1):                  # word loads, then the byte-wise conversion
    forward_u8(model, u8, offset)
    assert_same(snapshot(model), want, (case, offset))
    held = converted(u8, mc.BGR_MEANS) if converts else feed
    assert image_input(model).tobytes() == held.tobytes(), case
  assert model.launches_per_forward() == base


TAIL_CASES = [(1, 9, 29), (1, 10, 31), (1, 11, 25), (3, 7, 13)]   # B * H * W % 4 = 1, 2, 3, 1


@pytest.mark.parametrize('B,H,W', TAIL_CASES)
def test_converted_tail(B, H, W, gpu_device):
  """The converted path at pixel counts that are not a multiple of 4: tensor 0 holds
  float32(float64(u8) - BGR_MEANS) bit for bit, and the records equal those of the fp32 feed."""
  mc, model, _ = build([('conv', 'conv1', 16, 3, 1, 'SAME')], B, H, W, _lib.MATH_TF32X3_TC,
                       gpu_device)
  u8 = random_u8((B, H, W, 3), seed=B * H * W)
  forward_u8(model, u8)
  got = fetch_results(model, gpu_device)
  feed = converted(u8, mc.BGR_MEANS)
  assert image_input(model).tobytes() == feed.tobytes()
  dets, counts = model.detect_records(feed)
  assert np.array_equal(counts, got['counts']) and counts.min() >= 0
  assert dets.tobytes() == got['dets'].tobytes()


# ---- pipelined submissions (sqdet_submit) take the same path ----------------------------------
def test_submit_u8_fused_leaves_tensor0(gpu_device):
  """On a fused plan a uint8 submission runs no conversion: after sqdet_detect of fp32 images A,
  submissions of other bytes B (one per slot) leave A in tensor 0, and their records equal those
  of the fp32 feed of B."""
  model = squeezedet_small(2, gpu_device)
  mc = model.mc
  shape = (2, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, 3)
  u8 = random_u8(shape, seed=18)
  want_dets, want_counts = model.detect_records(converted(u8, mc.BGR_MEANS))
  feed = synth.synthetic_images(2, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, seed=19)
  model.detect(feed)
  for slot in (0, 1):
    dets, counts = model.detect_u8(u8)
    assert np.array_equal(counts, want_counts) and dets.tobytes() == want_dets.tobytes(), slot
    assert image_input(model).tobytes() == feed.tobytes(), slot


def test_submit_mixed_types_converted(gpu_device):
  """On a plan that converts into tensor 0, four submissions with two in flight, fp32 in slot 0
  and uint8 in slot 1: every submission's records equal its synchronous run's."""
  B, H, W = 2, 96, 320
  mc, model, _ = build([('conv', 'conv1', 32, 3, 1, 'SAME'), ('pool', 'pool1', 3, 2, 'SAME')], B,
                       H, W, _lib.MATH_TF32X3_TC, gpu_device)
  srcs = [synth.synthetic_images(B, H, W, seed=20 + i) if i % 2 == 0 else
          random_u8((B, H, W, 3), seed=20 + i) for i in range(4)]
  want = [model.detect_records(x if i % 2 == 0 else converted(x, mc.BGR_MEANS))
          for i, x in enumerate(srcs)]
  outs = [(np.empty((B, model.max_dets), _lib.DET_DTYPE), np.empty((B,), np.int32)) for _ in srcs]
  for i, x in enumerate(srcs):
    model.submit(x.ctypes.data, outs[i][0].ctypes.data, outs[i][1].ctypes.data,
                 _lib.IMG_F32 if i % 2 == 0 else _lib.IMG_U8)
    if i >= 1:
      model.wait()
  model.wait()
  for i, ((d, c), (wd, wc)) in enumerate(zip(outs, want)):
    assert np.array_equal(c, wc) and wc.min() >= 0 and d.tobytes() == wd.tobytes(), i


# ---- refused calls write nothing ------------------------------------------------------------------
def test_errors_before_device_work(gpu_device):
  model = squeezedet_small(2, gpu_device)
  mc = model.mc
  lib = model._lib
  feed = synth.synthetic_images(2, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, seed=16)
  model.detect(feed)
  before = snapshot(model)
  u8 = random_u8((2, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, 3), seed=17)
  buf = u8_buffer(u8, 0, gpu_device)
  for eng, ptr, n, code in [(None, buf.ptr, 1, ERR_INVALID_ARG),
                            (model._engine, None, 1, ERR_INVALID_ARG),
                            (model._engine, buf.ptr, 0, ERR_INVALID_ARG),
                            (model._engine, buf.ptr, 3, ERR_INVALID_ARG),
                            (model._engine, buf.ptr, -1, ERR_INVALID_ARG)]:
    assert lib.sqdet_forward_u8(eng, ptr, n, model.engine_stream()) == code, (eng, ptr, n)
  assert b'n must be' in lib.sqdet_last_error()
  _lib.check(lib.sqdet_stream_sync(gpu_device, model.engine_stream()))
  assert_same(snapshot(model), before, ('after refused calls',))
  assert image_input(model).tobytes() == feed.tobytes()
  # an engine not yet finalized
  h = C.c_void_p()
  conf = _lib.Config(batch_size=1, image_height=8, image_width=8, classes=3, anchors_per_grid=9,
                     top_n_detection=64, prob_thresh=0.005, nms_thresh=0.4, exp_thresh=1.0,
                     batch_norm_epsilon=1e-5, math_mode=0, max_dets=0)
  _lib.check(lib.sqdet_create(C.byref(conf), gpu_device, C.byref(h)))
  assert lib.sqdet_forward_u8(h, buf.ptr, 1, None) == ERR_STATE
  assert b'finalize' in lib.sqdet_last_error()
  lib.sqdet_destroy(h)
  buf.free()
