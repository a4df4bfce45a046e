"""Stage-isolated GPU parity tests (call through the C ABI; oracle = numpy
restatement / committed reference fixtures)."""
import numpy as np
import pytest

import oracle
from squeezedet_b200 import _lib
from gpu_util import (conv2d_gpu, maxpool_gpu, interpret_gpu, topk_nms_gpu, preprocess_gpu, rel_err)

pytestmark = pytest.mark.gpu

# fp32 tolerance for one conv layer vs the fp64 oracle, relative to the tensor's max
CONV_RTOL = 2e-5

CONV_CASES = [
    # B, H, W, Cin, Cout, k, stride, padding
    (2, 37, 50, 3, 64, 3, 2, 'SAME'),      # conv1 (SqueezeDet) shape class
    (1, 41, 53, 3, 96, 7, 2, 'VALID'),     # conv1 (SqueezeDet+)
    (2, 24, 31, 64, 16, 1, 1, 'SAME'),     # squeeze
    (2, 24, 31, 16, 64, 3, 1, 'SAME'),     # expand3x3, Cin=16
    (1, 13, 29, 48, 192, 3, 1, 'SAME'),    # fire6 expand (Cin=48)
    (1, 12, 20, 96, 384, 1, 1, 'SAME'),    # fire10 expand1x1
    (1, 12, 20, 256, 72, 3, 1, 'SAME'),    # ConvDet head (N=72), split-K over filter rows (8 K chunks)
    (1, 12, 20, 384, 72, 3, 1, 'SAME'),    # ConvDet head, split-K over input-channel ranges (12 K chunks)
    (1, 17, 23, 64, 128, 1, 2, 'SAME'),    # ResNet strided 1x1
    (1, 20, 20, 32, 32, 3, 1, 'SAME'),
    # first-layer gather mode (3x3 over 3 channels): every stride / padding / alignment class
    (1, 33, 65, 3, 64, 3, 2, 'VALID'),     # odd row pitch: patch rows start 4-, 8-, 12-byte misaligned
    (2, 34, 70, 3, 64, 3, 2, 'SAME'),      # even dims: zero padding only at the bottom / right
    (2, 13, 29, 3, 64, 3, 1, 'SAME'),      # VGG conv1_1 shape class (pad 1 on all sides)
    (1, 48, 100, 3, 96, 3, 1, 'VALID'),
    (1, 64, 96, 64, 64, 1, 1, 'SAME'),     # flat 1x1 tiling, 48 whole tiles
    (3, 11, 13, 32, 48, 1, 1, 'SAME'),     # flat 1x1 tiling, ragged last tile
    # gather mode with 16- and 32-wide output tiles (conv_tc_kernel<16|32, 32, true>)
    (2, 19, 35, 3, 16, 3, 1, 'SAME'),
    (1, 21, 40, 3, 16, 3, 2, 'VALID'),
    (1, 22, 37, 3, 32, 3, 2, 'SAME'),
    (2, 17, 30, 3, 32, 3, 1, 'VALID'),
    # Cin % 32 == 16 with a 16-wide output tile: KC = 16, NT = 16 (conv_tc_kernel<16, 16, false>)
    (2, 14, 23, 16, 16, 3, 1, 'SAME'),
    (1, 13, 29, 48, 16, 1, 1, 'SAME'),
    # one-pixel-high / -wide images under a 3x3 window: every tap but the centre row / column pads
    (2, 1, 37, 32, 64, 3, 1, 'SAME'),
    (1, 29, 1, 16, 32, 3, 1, 'SAME'),
    (1, 1, 40, 3, 16, 3, 1, 'SAME'),
    # M = B * Ho * Wo around one 128-pixel tile: 1, 127, 128, 129
    (1, 1, 1, 64, 64, 3, 1, 'SAME'),
    (1, 1, 127, 32, 48, 1, 1, 'SAME'),
    (2, 8, 8, 16, 32, 3, 1, 'SAME'),
    (1, 3, 43, 48, 64, 3, 1, 'SAME'),
    # ragged last output-channel chunk with NT = 64: 100 = 64 + 36 (not a multiple of 8),
    # 200 = 3 * 64 + 8
    (1, 9, 15, 64, 100, 3, 1, 'SAME'),
    (1, 10, 13, 32, 200, 1, 1, 'SAME'),
    # the 32-chunk launch limit: 2048 = 32 chunks of 64 runs on wgmma, 2049 is declined and
    # runs on the SIMT kernel
    (1, 3, 5, 32, 2048, 1, 1, 'SAME'),
    (1, 3, 5, 32, 2049, 1, 1, 'SAME'),
    # the 72-wide ConvDet head tile (one conv of 65..72 channels, Cin % 32 == 0): ragged and odd
    # channel counts inside the tile, a 1x1 on it, and both sides of its 64 / 65 and 72 / 73 edges
    (1, 12, 20, 64, 65, 3, 1, 'SAME'),
    (2, 11, 17, 32, 69, 3, 1, 'SAME'),
    (1, 13, 21, 96, 71, 3, 1, 'SAME'),
    (1, 16, 24, 128, 72, 1, 1, 'SAME'),
    (1, 12, 20, 48, 72, 3, 1, 'SAME'),     # Cin % 32 == 16: KC = 16, so the 64-wide tile
    (1, 12, 20, 64, 73, 3, 1, 'SAME'),     # one channel past the 72 tile
    (1, 96, 200, 32, 72, 3, 1, 'SAME'),    # 150 pixel tiles: more CTAs than SMs
]


@pytest.mark.parametrize('math_mode', [_lib.MATH_FP32_SIMT, _lib.MATH_TF32X3_TC])
@pytest.mark.parametrize('case', CONV_CASES)
def test_conv2d_vs_oracle(case, math_mode, gpu_device):
  B, H, W, Cin, Cout, k, stride, padding = case
  rng = np.random.default_rng(hash(case) % (2 ** 31))
  x = rng.normal(size=(B, H, W, Cin)).astype(np.float32)
  w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(np.float32)
  b = rng.normal(size=(Cout,)).astype(np.float32)
  want = oracle.conv2d(x, w, b, stride, padding, apply_relu=True, dtype=np.float64)
  got = conv2d_gpu(x, w, b, stride, padding, relu=True, math_mode=math_mode)
  assert got.shape == want.shape
  assert rel_err(got, want) < CONV_RTOL
  # the fp32 oracle itself must be within the same distance of fp64 (sanity of the bar)
  assert rel_err(oracle.conv2d(x, w, b, stride, padding, True, np.float32), want) < CONV_RTOL


def check_affine_and_channel_window(math_mode, Cin, Cout, y_cstride, y_coff):
  rng = np.random.default_rng(11)
  x = rng.normal(size=(1, 15, 18, Cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, Cin, Cout)) / np.sqrt(9 * Cin)).astype(np.float32)
  b = rng.normal(size=(Cout,)).astype(np.float32)
  sc = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
  sh = rng.normal(size=Cout).astype(np.float32)
  want = oracle.conv2d(x, w, b, 1, 'SAME', False, np.float64) * sc + sh
  y0 = np.full((1, 15, 18, y_cstride), 7.0, np.float32)
  got = conv2d_gpu(x, w, b, 1, 'SAME', relu=False, scale=sc, shift=sh, y_cstride=y_cstride,
                   y_coff=y_coff, math_mode=math_mode, y_init=y0)
  assert rel_err(got[..., y_coff:y_coff + Cout], want) < CONV_RTOL
  assert np.all(got[..., :y_coff] == 7.0) and np.all(got[..., y_coff + Cout:] == 7.0)  # untouched


@pytest.mark.parametrize('math_mode', [_lib.MATH_FP32_SIMT, _lib.MATH_TF32X3_TC])
def test_conv2d_no_relu_affine_and_channel_window(math_mode, gpu_device):
  """BN-style scale/shift epilogue, no ReLU, and a strided channel window (fire concat)."""
  check_affine_and_channel_window(math_mode, 32, 48, 80, 16)


@pytest.mark.parametrize('math_mode', [_lib.MATH_FP32_SIMT, _lib.MATH_TF32X3_TC])
def test_conv2d_affine_and_channel_window_on_72_tile(math_mode, gpu_device):
  """The same epilogue on the 72-wide head tile: 72 channels at offset 8 of 88."""
  check_affine_and_channel_window(math_mode, 64, 72, 88, 8)


MAXPOOL_CASES = [
    # stride 2 with 2x2 / 3x3 windows (maxpool_s2_vec4_kernel), C % 4 != 0 (scalar kernel)
    ((2, 47, 61, 64), 3, 2, 'SAME'), ((1, 47, 62, 128), 3, 2, 'SAME'),
    ((1, 45, 61, 96), 3, 2, 'VALID'), ((2, 31, 37, 64), 2, 2, 'SAME'),
    ((1, 9, 11, 6), 3, 2, 'SAME'),
    # every other window / stride: the generic maxpool_vec4_kernel
    ((2, 23, 37, 64), 2, 1, 'SAME'), ((1, 23, 37, 32), 2, 1, 'VALID'),
    ((2, 19, 29, 64), 3, 1, 'SAME'), ((1, 19, 29, 16), 3, 1, 'VALID'),
    ((1, 31, 44, 64), 3, 3, 'SAME'), ((2, 13, 17, 32), 1, 1, 'SAME'),
    # 5.1 M float4 outputs: more than the grid cap of 16 waves of 8 CTAs per SM, so grid-strided
    ((2, 200, 200, 256), 2, 1, 'SAME'),
]
# C % 4 == 0 with x and y one float past 16-byte alignment: the scalar kernel
MAXPOOL_MISALIGNED_CASES = [((2, 31, 37, 64), 3, 2, 'SAME', 1), ((1, 23, 37, 32), 2, 1, 'VALID', 1)]


@pytest.mark.parametrize('shape,k,stride,padding', MAXPOOL_CASES)
def test_maxpool_exact(shape, k, stride, padding, gpu_device):
  rng = np.random.default_rng(5)
  x = (rng.normal(size=shape) - 2.0).astype(np.float32)
  assert np.array_equal(maxpool_gpu(x, k, stride, padding), oracle.max_pool(x, k, stride, padding))


@pytest.mark.parametrize('shape,k,stride,padding,offset', MAXPOOL_MISALIGNED_CASES)
def test_maxpool_exact_misaligned(shape, k, stride, padding, offset, gpu_device):
  rng = np.random.default_rng(6)
  x = (rng.normal(size=shape) - 2.0).astype(np.float32)
  assert np.array_equal(maxpool_gpu(x, k, stride, padding, offset=offset),
                        oracle.max_pool(x, k, stride, padding))


@pytest.mark.parametrize('classes,K,gh,gw', [(3, 9, 24, 78), (20, 9, 5, 7), (3, 9, 22, 76),
                                             (3, 1, 24, 78), (3, 5, 13, 41), (1, 9, 11, 37)])
def test_interpret_vs_oracle(classes, K, gh, gw, gpu_device):
  rng = np.random.default_rng(classes)
  B, W, H = 2, 1242, 375
  preds = (rng.normal(size=(B, gh, gw, K * (classes + 5))) * 1.5).astype(np.float32)
  preds[0, 0, 0, K * classes + K + 2] = 3.0         # dw above EXP_THRESH -> linear tail
  preds[0, 0, 1, K * classes + K + 3] = -40.0
  anchors = oracle.set_anchors(W, H, gh, gw, oracle.postproc.ANCHOR_SHAPES_SQUEEZE[:K])
  wb, wp, wc = oracle.interpret_output(preds, anchors, classes, K, W, H, 1.0)
  gb, gp, gc = interpret_gpu(preds, anchors, K, classes, W, H, 1.0)
  # bar (BASELINE.json): coordinates and scores within 1e-4 relative; 1e-3 px absolute covers
  # 1-ulp expf differences on 4000-px-wide boxes that cancel down to small clipped values
  np.testing.assert_allclose(gb, wb, rtol=1e-4, atol=1e-3)
  np.testing.assert_allclose(gp, wp, rtol=1e-5, atol=1e-9)
  # class ids: exact wherever the oracle's own top-2 margin exceeds fp noise
  b64, p64, c64 = oracle.interpret_output(preds, anchors, classes, K, W, H, 1.0, np.float64)
  assert gc.dtype == np.int64
  mism = gc != wc
  assert mism.mean() < 1e-4
  assert np.array_equal(gc, c64) or mism.sum() <= 2


def _check_case(c, dets, count):
  n = len(c['out_cls'])
  assert count == n, (c['name'], count, n)
  d = dets[:n]
  assert d['cls'].tolist() == c['out_cls'].tolist(), c['name']
  got_boxes = np.stack([d['cx'], d['cy'], d['w'], d['h']], 1) if n else np.zeros((0, 4), np.float32)
  assert np.array_equal(got_boxes, c['out_boxes']), c['name']            # bit-exact
  assert np.array_equal(d['prob'], c['out_probs']), c['name']
  for a, bx in zip(d['anchor'], got_boxes):                               # kept-box indices
    assert np.array_equal(c['boxes'][a], bx)
  assert np.all(dets[n:]['anchor'] == -1)


def test_topk_nms_bit_exact_vs_reference_fixtures(postproc_kat, gpu_device):
  for c in postproc_kat['cases']:
    dets, counts = topk_nms_gpu(c['boxes'][None], c['probs'][None], c['cls'][None], c['classes'],
                                c['top_n'], c['prob_thresh'], c['nms_thresh'])
    _check_case(c, dets[0], int(counts[0]))


def test_topk_nms_batched_equals_per_image(postproc_kat, gpu_device):
  cs = [c for c in postproc_kat['cases'] if c['n'] == 200 and c['top_n'] == 64]
  assert len(cs) == 2
  boxes = np.stack([c['boxes'] for c in cs])
  probs = np.stack([c['probs'] for c in cs])
  cls = np.stack([c['cls'] for c in cs])
  dets, counts = topk_nms_gpu(boxes, probs, cls, 3, 64, 0.005, 0.4)
  for i, c in enumerate(cs):
    _check_case(c, dets[i], int(counts[i]))


def test_topk_nms_ties_use_documented_rule(gpu_device):
  """All 16848 scores identical (the reference's own-init degenerate case): the engine's
  documented tie rule is (prob desc, anchor asc) -> anchors 0..63 are the candidates."""
  A = 16848
  rng = np.random.default_rng(1)
  boxes = np.stack([rng.uniform(0, 1242, A), rng.uniform(0, 375, A), rng.uniform(4, 60, A),
                    rng.uniform(4, 40, A)], 1).astype(np.float32)
  probs = np.full(A, 1.0 / 6.0, np.float32)
  cls = rng.integers(0, 3, A).astype(np.int64)
  dets, counts = topk_nms_gpu(boxes[None], probs[None], cls[None], 3, 64, 0.005, 0.4)
  fb, fp, fc, src = oracle.filter_prediction(boxes, probs, cls, 3, 64, 0.005, 0.4)
  assert int(counts[0]) == len(src)
  assert dets[0]['anchor'][:len(src)].tolist() == src
  assert max(src) < 64


def test_topk_nms_threshold_overflow_flag(gpu_device):
  A = 3000
  rng = np.random.default_rng(2)
  boxes = np.abs(rng.normal(size=(1, A, 4))).astype(np.float32) + 1
  probs = rng.uniform(0.5, 1, (1, A)).astype(np.float32)
  cls = np.zeros((1, A), np.int64)
  dets, counts = topk_nms_gpu(boxes, probs, cls, 3, 0, 0.005, 0.4, max_dets=1024)
  assert int(counts[0]) == -1          # > 1024 boxes above PROB_THRESH: reported, not truncated


def test_util_nms_gpu_matches_reference_keep(postproc_kat, gpu_device):
  from squeezedet_b200.utils import util
  for c in postproc_kat['cases']:
    if 0 < len(c['nms_keep']) <= 512:
      assert util.nms(c['boxes'], c['probs'], c['nms_thresh']) == c['nms_keep'].tolist(), c['name']


@pytest.mark.parametrize('order', ['demo', 'eval'])
@pytest.mark.parametrize('h0,w0,h,w', [(370, 1224, 375, 1242), (375, 1242, 375, 1242),
                                       (720, 1280, 375, 1242), (37, 41, 19, 23), (5, 7, 31, 3)])
def test_preprocess_u8_resize_meansub(h0, w0, h, w, order, gpu_device):
  """f-1: uint8 -> float32, cv2 INTER_LINEAR resize, mean subtraction in the reference's two
  orders.  The kernel restates oracle/preproc.py operation for operation (the oracle is pinned to
  cv2 within 3 float32 ulp of the pixel range, tests/test_oracle_preproc.py)."""
  from oracle import preproc
  means = np.array([103.939, 116.779, 123.68])
  rng = np.random.default_rng(h0 + 3 * w)
  img = rng.integers(0, 256, (h0, w0, 3), dtype=np.uint8)
  want = preproc.preprocess(img, w, h, means, order)
  got = preprocess_gpu(img, w, h, means, order)
  assert got.shape == want.shape
  ulp = float(np.spacing(np.float32(255.0)))
  assert np.abs(got - want).max() <= 2 * ulp, float(np.abs(got - want).max())
  cv2 = pytest.importorskip('cv2')
  x = img.astype(np.float32)
  if order == 'demo':
    ref = (cv2.resize(x, (w, h)) - means.reshape(1, 1, 3)).astype(np.float32)
  else:
    x -= means.reshape(1, 1, 3)
    ref = cv2.resize(x, (w, h))
  assert np.abs(got - ref).max() <= 4 * ulp
