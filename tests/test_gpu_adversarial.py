"""Adversarial operand distributions for the tensor-core convolution (conv_tc.cu): the tensor
core's own accumulation must not leave a one-signed bias over a long K (the kernel adds each K
chunk's MMA result into fp32 running sums).  These cases stress it: all-positive (any truncation
bias fully present), heavy-tailed (log-normal: a few products dominate), cancellation-dominated (the sum
is tiny against sum |products|), plus a long K.  Error is measured per output element against the
fp64 oracle on the scale that bounds ANY fp32 summation of the same products,
    |err| <= tol * (|x| (*) |w|),
so a case cannot hide behind a large max.  Both math modes must meet the same bar."""
import numpy as np
import pytest

from squeezedet_b200 import _lib
from gpu_util import adv_tol, assert_within_bound, conv2d_gpu, conv_oracle

pytestmark = pytest.mark.gpu


def _case(kind, rng, shape_x, shape_w):
  if kind == 'positive':
    x = rng.uniform(0.5, 1.5, shape_x)
    w = rng.uniform(0.5, 1.5, shape_w)
  elif kind == 'lognormal':
    x = rng.lognormal(0.0, 1.5, shape_x)
    w = rng.lognormal(0.0, 1.5, shape_w) * rng.choice([-1.0, 1.0], shape_w)
  elif kind == 'lognormal_positive':
    x = rng.lognormal(0.0, 1.5, shape_x)
    w = rng.lognormal(0.0, 1.5, shape_w)
  elif kind == 'cancel':
    # per output: +a and -a pairs along the input channels, plus a small residue
    x = np.abs(rng.normal(size=shape_x)) + 0.5
    w = rng.normal(size=shape_w)
    half = shape_w[2] // 2
    w[:, :, half:2 * half, :] = -w[:, :, :half, :]
    x[..., half:2 * half] = x[..., :half] * (1.0 + 1e-3 * rng.normal(size=x[..., :half].shape))
  else:
    raise ValueError(kind)
  return x.astype(np.float32), w.astype(np.float32)


SHAPES = [
    # B, H, W, Cin, Cout, k, stride (SAME padding)
    (1, 12, 20, 96, 64, 3, 1),    # 864 products per output, 3 segments of 36 MMAs
    (1, 9, 17, 256, 32, 3, 1),    # 2304 products, K chunks of 32
    (1, 16, 24, 768, 16, 1, 1),   # the longest 1x1 of SqueezeDet (fire11 squeeze)
    (1, 12, 20, 48, 64, 3, 1),    # K chunks of 16 (Cin % 32 == 16)
    (1, 10, 18, 80, 48, 3, 1),    # K chunks of 16, 45 of them
    (1, 12, 20, 48, 32, 3, 1),    # K chunks of 16 with a 32-wide output tile
    (2, 17, 29, 3, 64, 3, 1),     # gather mode: K = 27 zero-padded to one 32-row chunk
    (1, 33, 47, 3, 32, 3, 2),     # gather mode, stride 2, 32-wide output tile
    # the ConvDet heads on the 72-wide tile, the longest reductions the shipped nets run
    (1, 12, 20, 768, 72, 3, 1),   # K = 6912 (SqueezeDet)
    (1, 12, 20, 512, 72, 3, 1),   # K = 4608 (SqueezeDet+, VGG16)
    (1, 12, 20, 1024, 72, 3, 1),  # K = 9216 (ResNet50)
]


@pytest.mark.parametrize('math_mode', [_lib.MATH_FP32_SIMT, _lib.MATH_TF32X3_TC])
@pytest.mark.parametrize('kind', ['positive', 'lognormal', 'lognormal_positive', 'cancel'])
@pytest.mark.parametrize('shape', SHAPES)
def test_conv_adversarial_operands(shape, kind, math_mode, gpu_device):
  B, H, W, Cin, Cout, k, stride = shape
  rng = np.random.default_rng(1000 + Cin + k)
  x, w = _case(kind, rng, (B, H, W, Cin), (k, k, Cin, Cout))
  want, bound = conv_oracle(x, w, None, stride)
  got = conv2d_gpu(x, w, None, stride, 'SAME', relu=False, math_mode=math_mode)
  assert not np.isnan(got).any()
  assert_within_bound(got, want, bound, k * k * Cin, (kind, shape))
  tol = adv_tol(k * k * Cin)
  # the error must not be mostly one-sided: the MEAN signed error stays below half the bar
  signed = ((got.astype(np.float64) - want) / bound).mean()
  assert abs(signed) < tol / 2, (kind, shape, float(signed), tol)
