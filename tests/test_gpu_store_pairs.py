"""The tensor-core epilogues store each thread's two adjacent output channels as one 8-byte store
when every output row of the chunk starts 8-byte aligned (even channel stride and offset), and
channel by channel otherwise.  Odd strides, odd offsets and odd channel counts (a last pair with
one valid channel) must give the same per-element results and leave the channels outside the
window untouched."""
import numpy as np
import pytest

from squeezedet_b200 import _lib
from gpu_util import assert_within_bound, conv2d_gpu, conv_oracle, fire_gpu, fire_oracle

pytestmark = pytest.mark.gpu
TC = _lib.MATH_TF32X3_TC

CASES = [
    # B, H, W, Cin, Cout, k, y_cstride, y_coff
    (2, 13, 37, 32, 33, 1, 33, 0),      # row mode, odd channel count and stride
    (2, 13, 37, 32, 40, 1, 48, 5),      # row mode, odd offset
    (2, 13, 37, 32, 40, 1, 48, 6),      # row mode, even window inside a wider tensor
    (1, 11, 35, 48, 31, 3, 40, 3),      # halo mode, KC 16, odd count and offset
    (2, 12, 33, 32, 64, 3, 65, 1),      # halo mode, odd stride
    (1, 11, 35, 64, 70, 3, 80, 4),      # halo mode, 72-wide tile, even window
]


@pytest.mark.parametrize('case', CASES)
def test_conv_channel_windows(case, gpu_device):
  B, H, W, Cin, Cout, k, cs, coff = case
  rng = np.random.default_rng(sum(case))
  x = rng.normal(size=(B, H, W, Cin)).astype(np.float32)
  w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(np.float32)
  b = rng.normal(size=Cout).astype(np.float32)
  want, bound = conv_oracle(x, w, b, relu=True)
  y0 = np.full((B, H, W, cs), 7.0, np.float32)
  got = conv2d_gpu(x, w, b, 1, 'SAME', relu=True, y_cstride=cs, y_coff=coff, math_mode=TC,
                   device=gpu_device, y_init=y0)
  assert_within_bound(got[..., coff:coff + Cout], want, bound, k * k * Cin, case)
  assert np.all(got[..., :coff] == 7.0) and np.all(got[..., coff + Cout:] == 7.0), case


@pytest.mark.parametrize('E1,E3', [(33, 64), (64, 31), (64, 64)])
def test_fire_odd_expand_widths(E1, E3, gpu_device):
  """The one-kernel fire: an odd expand1x1 width puts the 3x3 channels at an odd offset of an odd
  channel stride; an odd expand3x3 width leaves a last pair with one valid channel."""
  B, H, W, Cin, S = 2, 13, 37, 32, 16
  rng = np.random.default_rng(E1 + E3)
  x = np.maximum(rng.normal(size=(B, H, W, Cin)), 0).astype(np.float32)
  ws = (rng.normal(size=(1, 1, Cin, S)) * np.sqrt(2.0 / Cin)).astype(np.float32)
  w1 = (rng.normal(size=(1, 1, S, E1)) * np.sqrt(2.0 / S)).astype(np.float32)
  w3 = (rng.normal(size=(3, 3, S, E3)) * np.sqrt(2.0 / (9 * S))).astype(np.float32)
  bs, b1, b3 = [np.abs(rng.normal(0, 0.3, size=(n,))).astype(np.float32) for n in (S, E1, E3)]
  got = fire_gpu(x, ws, bs, w1, b1, w3, b3, math_mode=TC, device=gpu_device)
  assert not np.isnan(got).any()
  want = fire_oracle(x, ws, bs, w1, b1, w3, b3, np.float64)
  err = float(np.abs(got - want).max() / np.abs(want).max())
  assert err < 3e-5, (E1, E3, err)
