"""sqdet_fire: the fire module as ONE stage-isolated call (reference src/nets/squeezeDet.py:81-106,
src/nets/squeezeDetPlus.py:81-106), over every fire shape of SqueezeDet and SqueezeDet+, both
math modes, vs the numpy oracle (fp64 truth, fp32 reference semantics)."""
import numpy as np
import pytest

import oracle
from squeezedet_b200 import _lib
from gpu_util import adv_tol, bound_ratio, fire_error_bound, fire_gpu, fire_oracle, rel_err

pytestmark = pytest.mark.gpu

# (Cin, s1x1, e1x1, e3x3): squeezeDet.py:46-71 and squeezeDetPlus.py:46-73
SQUEEZEDET_FIRES = [(64, 16, 64, 64), (128, 16, 64, 64), (128, 32, 128, 128), (256, 32, 128, 128),
                    (256, 48, 192, 192), (384, 48, 192, 192), (384, 64, 256, 256),
                    (512, 64, 256, 256), (512, 96, 384, 384), (768, 96, 384, 384)]
SQUEEZEDET_PLUS_FIRES = [(96, 96, 64, 64), (128, 96, 64, 64), (128, 192, 128, 128),
                         (256, 192, 128, 128), (256, 288, 192, 192), (384, 288, 192, 192),
                         (384, 384, 256, 256), (512, 384, 256, 256)]   # fire9-11 repeat the last
# spatial cases: ragged tiles on both axes, a single-tile image, a batch > 1
SPATIAL = [(2, 19, 37), (1, 8, 16), (1, 24, 78)]
FIRE_RTOL = 3e-5      # two stacked convs vs fp64, relative to the tensor's max


def make_case(shape, spatial, seed):
  Cin, S, E1, E3 = shape
  B, H, W = spatial
  rng = np.random.default_rng(seed)
  x = np.maximum(rng.normal(size=(B, H, W, Cin)), 0).astype(np.float32)   # post-ReLU input
  ws = (rng.normal(size=(1, 1, Cin, S)) * np.sqrt(2.0 / Cin)).astype(np.float32)
  w1 = (rng.normal(size=(1, 1, S, E1)) * np.sqrt(2.0 / S)).astype(np.float32)
  w3 = (rng.normal(size=(3, 3, S, E3)) * np.sqrt(2.0 / (9 * S))).astype(np.float32)
  bs, b1, b3 = [rng.normal(0, 0.3, size=(n,)).astype(np.float32) for n in (S, E1, E3)]
  return x, ws, bs, w1, b1, w3, b3


@pytest.mark.parametrize('math_mode', [_lib.MATH_FP32_SIMT, _lib.MATH_TF32X3_TC])
@pytest.mark.parametrize('shape', SQUEEZEDET_FIRES + SQUEEZEDET_PLUS_FIRES)
def test_fire_vs_oracle(shape, math_mode, gpu_device):
  spatial = SPATIAL[(shape[0] + shape[1]) % 2]          # alternate the two ragged cases
  args = make_case(shape, spatial, seed=shape[0] * 7 + shape[1])
  want64 = fire_oracle(*args, dtype=np.float64)
  want32 = fire_oracle(*args, dtype=np.float32)
  got = fire_gpu(*args, math_mode=math_mode, device=gpu_device)
  assert got.shape == want64.shape and not np.isnan(got).any()
  assert rel_err(got, want64) < FIRE_RTOL, rel_err(got, want64)
  assert rel_err(got, want32) < 1e-4
  assert rel_err(want32, want64) < FIRE_RTOL          # sanity of the bar
  r = fire_bound_ratio(args, got, want64)
  assert r < 1.0, r


# Shapes the shipped nets never produce, chosen to reach both fire_tc_kernel<KCI> instantiations
# (KCI = 16 for Cin % 32 == 16, else 32) and the planner's edges (conv_tc.cu, tc_fire_plan):
#   S = 16 (one kernel) and S = 32, 48, 64 (squeeze and expands as three sqdet_conv2d launches),
#   E1 != E3, expand widths that are not multiples of 64 or of 8,
#   16 expand chunks of 64 (the one-kernel limit) and 17 (sqdet_fire falls back to separate
#   launches).
TINY_IMAGES = ((1, 1), (1, 17), (9, 1), (8, 16), (9, 17))
FIRE_EDGE_CASES = [
    # (Cin, S, E1, E3), (B, H, W)
    *[((cin, s, 64, 64), (2, 11, 21)) for cin in (16, 48, 80, 112) for s in (16, 32, 48, 64)],
    ((64, 16, 40, 88), (2, 13, 19)),
    ((96, 32, 24, 200), (1, 10, 33)),
    ((48, 48, 40, 88), (2, 9, 17)),
    ((128, 64, 40, 88), (2, 9, 17)),
    ((64, 16, 512, 512), (1, 9, 18)),
    ((64, 16, 576, 512), (1, 9, 18)),
    # tiny images: 1x1, one row, one column, one exact 8x16 tile, one pixel past it on both axes
    *[((48, 32, 40, 88), (3, h, w)) for h, w in TINY_IMAGES],
    *[((64, 48, 64, 64), (3, h, w)) for h, w in ((1, 1), (8, 16), (9, 17))],
    *[((cin, 16, 40, 88), (3, h, w)) for cin in (48, 64) for h, w in TINY_IMAGES],
]


def fire_bound_ratio(args, got, want64):
  """max |got - want64| / gpu_util.fire_error_bound, in units of the bar adv_tol(K) with K the
  longer of the two convs' sums; must stay below 1."""
  x, ws, bs, w1, b1, w3, b3 = args
  q64 = oracle.conv2d(x, ws, bs, 1, 'SAME', True, np.float64)
  ratio = bound_ratio(got, want64, fire_error_bound(x, ws, w1, w3, q64))
  return float(ratio.max()) / adv_tol(max(x.shape[3], 9 * ws.shape[3]))


@pytest.mark.parametrize('math_mode', [_lib.MATH_FP32_SIMT, _lib.MATH_TF32X3_TC])
@pytest.mark.parametrize('shape,spatial', FIRE_EDGE_CASES)
def test_fire_edge_shapes_vs_oracle(shape, spatial, math_mode, gpu_device):
  """Every one-kernel fire variant and the planner's edges, against fp64 with the per-tensor
  bar of test_fire_vs_oracle and the per-element bound of fire_error_bound; the same call twice
  is bit-identical."""
  Cin, S, E1, E3 = shape
  args = make_case(shape, spatial, seed=Cin * 131 + S * 7 + E1 + E3 + sum(spatial))
  want64 = fire_oracle(*args, dtype=np.float64)
  want32 = fire_oracle(*args, dtype=np.float32)
  got = fire_gpu(*args, math_mode=math_mode, device=gpu_device)
  assert got.shape == want64.shape and not np.isnan(got).any()
  assert rel_err(got, want64) < FIRE_RTOL, rel_err(got, want64)
  assert rel_err(got, want32) < 1e-4
  r = fire_bound_ratio(args, got, want64)
  assert r < 1.0, r
  again = fire_gpu(*args, math_mode=math_mode, device=gpu_device)
  assert np.array_equal(got, again)            # deterministic: fixed summation order


@pytest.mark.parametrize('shape', [SQUEEZEDET_FIRES[0], SQUEEZEDET_FIRES[3], SQUEEZEDET_FIRES[9]])
def test_fire_full_grid_and_border_padding(shape, gpu_device):
  """A full 24x78 grid (3 x 5 tiles, ragged right edge) and a bias-dominated squeeze: SAME
  padding of the 3x3 expand pads the POST-ReLU squeeze output with zeros, so a fused kernel must
  force halo pixels outside the image to 0 rather than relu(bias)."""
  x, ws, bs, w1, b1, w3, b3 = make_case(shape, SPATIAL[2], seed=99)
  bs = np.abs(bs) + 1.0                                # relu(0*w + bias) = bias > 0 at the halo
  want = fire_oracle(x, ws, bs, w1, b1, w3, b3, np.float64)
  got = fire_gpu(x, ws, bs, w1, b1, w3, b3, math_mode=_lib.MATH_TF32X3_TC, device=gpu_device)
  assert rel_err(got, want) < FIRE_RTOL, rel_err(got, want)
  # border rows / columns carry the padding effect: check them on their own scale
  for sl in (np.s_[:, 0], np.s_[:, -1], np.s_[:, :, 0], np.s_[:, :, -1]):
    assert rel_err(got[sl], want[sl]) < FIRE_RTOL


@pytest.mark.parametrize('shape,spatial', [
    (SQUEEZEDET_FIRES[0], (2, 94, 160)),     # S=16
    (SQUEEZEDET_FIRES[3], (8, 24, 78)),      # S=32
    (SQUEEZEDET_FIRES[5], (8, 24, 78)),      # S=48
    (SQUEEZEDET_FIRES[7], (8, 24, 78)),      # S=64
])
def test_fire_persistent_grid_many_items(shape, spatial, gpu_device):
  """Grids of many more tiles than SMs, at every squeeze width: deterministic and within the bar."""
  args = make_case(shape, spatial, seed=5 + shape[1])
  want = fire_oracle(*args, dtype=np.float64)
  got = fire_gpu(*args, math_mode=_lib.MATH_TF32X3_TC, device=gpu_device)
  assert not np.isnan(got).any()
  assert rel_err(got, want) < FIRE_RTOL, rel_err(got, want)
  again = fire_gpu(*args, math_mode=_lib.MATH_TF32X3_TC, device=gpu_device)
  assert np.array_equal(got, again)            # deterministic: fixed summation order
