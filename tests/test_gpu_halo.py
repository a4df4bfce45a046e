"""The stage-isolated 3x3 tensor-core convolution (entry sqdet_conv3x3_halo) against the numpy
oracle: ragged tiles on both axes, the ConvDet head's 72-channel output (partial last channel chunk), BN-style scale/shift, a channel
window of a wider tensor, and a grid with more items than SMs."""
import numpy as np
import pytest

import oracle
from gpu_util import conv3x3_halo_gpu, rel_err

pytestmark = pytest.mark.gpu

CONV_RTOL = 2e-5

CASES = [
    # B, H, W, Cin, Cout
    (1, 24, 78, 768, 72),     # ConvDet head of SqueezeDet: 8h x 16w tiles, split-K
    (2, 22, 76, 384, 72),     # ConvDet head of SqueezeDet+ (ragged both ways)
    (1, 33, 19, 64, 64),      # 16h x 8w tiles, direct epilogue, single K range
    (1, 9, 40, 32, 128),      # one row of tiles, N = 128
    (2, 17, 23, 48, 256),     # two output-channel chunks of 128
    (1, 8, 16, 16, 32),       # exactly one tile, one K chunk
    (6, 40, 48, 32, 32),      # more 128-pixel tiles than SMs
]


@pytest.mark.parametrize('case', CASES)
def test_halo_conv_vs_oracle(case, gpu_device):
  B, H, W, Cin, Cout = case
  rng = np.random.default_rng(sum(case))
  x = rng.normal(size=(B, H, W, Cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, Cin, Cout)) / np.sqrt(9 * Cin)).astype(np.float32)
  b = rng.normal(size=(Cout,)).astype(np.float32)
  want = oracle.conv2d(x, w, b, 1, 'SAME', apply_relu=True, dtype=np.float64)
  got = conv3x3_halo_gpu(x, w, b, relu=True)
  assert got.shape == want.shape and not np.isnan(got).any()
  assert rel_err(got, want) < CONV_RTOL, rel_err(got, want)
  # image borders carry the SAME zero padding: check them on their own scale
  for sl in (np.s_[:, 0], np.s_[:, -1], np.s_[:, :, 0], np.s_[:, :, -1]):
    assert rel_err(got[sl], want[sl]) < CONV_RTOL
  again = conv3x3_halo_gpu(x, w, b, relu=True)
  assert np.array_equal(got, again)            # deterministic


def test_halo_conv_no_relu_affine_and_channel_window(gpu_device):
  rng = np.random.default_rng(3)
  x = rng.normal(size=(1, 15, 18, 32)).astype(np.float32)
  w = (rng.normal(size=(3, 3, 32, 64)) / 17).astype(np.float32)
  b = rng.normal(size=(64,)).astype(np.float32)
  sc = rng.uniform(0.5, 1.5, 64).astype(np.float32)
  sh = rng.normal(size=64).astype(np.float32)
  want = oracle.conv2d(x, w, b, 1, 'SAME', False, np.float64) * sc + sh
  y0 = np.full((1, 15, 18, 96), 7.0, np.float32)
  got = conv3x3_halo_gpu(x, w, b, relu=False, scale=sc, shift=sh, y_cstride=96, y_coff=32, y_init=y0)
  assert rel_err(got[..., 32:], want) < CONV_RTOL
  assert np.all(got[..., :32] == 7.0)          # untouched channels
