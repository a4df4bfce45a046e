"""The halo tile of the 3x3 tensor-core convolution (conv_tc.cu, halo mode): a CTA computes an
8 x 16 output tile of one image from the 10 x 18 halo of each input-channel chunk and reads the
nine taps as row offsets into it.  Tiles cut by every image edge, images smaller than one tile
(down to 1 x 1), every output-tile width with both K chunk widths, a ragged fire expand pair (a
1x1 and a 3x3 conv in one launch), the affine epilogue with a channel window, and images of a
partial batch.  Each element is checked against the fp64 oracle on the scale that bounds any
fp32 summation of its products, with the bar gpu_util.adv_tol; the ConvDet heads, wide
outputs and a channel window also against a relative bar over the whole tensor and its borders."""
import numpy as np
import pytest

import oracle
from squeezedet_b200 import _lib
from squeezedet_b200.utils import synth
from gpu_util import (assert_rows_equal, assert_within_bound, build, conv2d_gpu, conv_oracle,
                      forward_n, read_tensors, rel_err)

pytestmark = pytest.mark.gpu
TC = _lib.MATH_TF32X3_TC


CASES = [
    # B, H, W, Cin, Cout: output tile NT (pick_nt) and K chunk KC (32 when Cin % 32 == 0, else 16)
    (2, 13, 29, 32, 16),     # NT 16, KC 32; H, W not multiples of 8 / 16
    (1, 5, 11, 48, 16),      # NT 16, KC 16; H < 8 and W < 16: one tile, mostly padding
    (1, 1, 1, 64, 32),       # NT 32, KC 32; a 1 x 1 image: only the centre tap is inside
    (3, 9, 17, 16, 32),      # NT 32, KC 16; one row and one column past a whole tile
    (1, 24, 78, 96, 64),     # NT 64, KC 32; the grid of SqueezeDet's fire6-11 and ConvDet head
    (2, 7, 33, 80, 64),      # NT 64, KC 16; five channel chunks, so both halo buffers recycle
    (1, 23, 1, 48, 40),      # NT 64, KC 16; a one-column image, a partial channel chunk
    (1, 1, 20, 32, 72),      # NT 72, KC 32; a one-row image
    (2, 17, 15, 64, 72),     # NT 72, KC 32; W < 16
]


@pytest.mark.parametrize('case', CASES)
def test_halo_tile_vs_oracle(case, gpu_device):
  B, H, W, Cin, Cout = case
  rng = np.random.default_rng(7 + sum(case))
  x = rng.normal(size=(B, H, W, Cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, Cin, Cout)) / np.sqrt(9 * Cin)).astype(np.float32)
  want, bound = conv_oracle(x, w)
  got = conv2d_gpu(x, w, None, 1, 'SAME', relu=False, math_mode=TC)
  assert got.shape == want.shape
  assert_within_bound(got, want, bound, 9 * Cin, case)
  again = conv2d_gpu(x, w, None, 1, 'SAME', relu=False, math_mode=TC)
  assert got.tobytes() == again.tobytes()                 # bitwise repeatable
  # an image's tiles do not depend on the batch around it
  first = conv2d_gpu(x[:1], w, None, 1, 'SAME', relu=False, math_mode=TC)
  assert first.tobytes() == got[:1].tobytes()


@pytest.mark.parametrize('cin', [32, 48])
def test_halo_tile_affine_and_channel_window(cin, gpu_device):
  """Bias, frozen-BN scale / shift and no ReLU, written into channels [40, 112) of a 128-wide
  tensor: NT 72 for Cin = 32 (KC 32), two 64-wide chunks for Cin = 48 (KC 16)."""
  rng = np.random.default_rng(cin)
  B, H, W, Cout, cs, coff = 2, 11, 21, 72, 128, 40
  x = rng.normal(size=(B, H, W, cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, cin, Cout)) / np.sqrt(9 * cin)).astype(np.float32)
  b = rng.normal(size=Cout).astype(np.float32)
  sc = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
  sh = rng.normal(size=Cout).astype(np.float32)
  want, bound = conv_oracle(x, w, b, scale=sc, shift=sh)
  y0 = np.full((B, H, W, cs), 7.0, np.float32)
  got = conv2d_gpu(x, w, b, 1, 'SAME', relu=False, scale=sc, shift=sh, y_cstride=cs, y_coff=coff,
                   math_mode=TC, y_init=y0)
  assert_within_bound(got[..., coff:coff + Cout], want, bound, 9 * cin, cin)
  assert np.all(got[..., :coff] == 7.0) and np.all(got[..., coff + Cout:] == 7.0)


CONV_RTOL = 2e-5
HALO_CONV_CASES = [
    # B, H, W, Cin, Cout: output tile NT (pick_nt) and K chunk KC (32 when Cin % 32 == 0, else 16)
    (1, 24, 78, 768, 72),     # NT 72, KC 32; the ConvDet head of SqueezeDet
    (2, 22, 76, 384, 72),     # NT 72, KC 32; the ConvDet head of SqueezeDet+ (ragged both ways)
    (1, 33, 19, 64, 64),      # NT 64, KC 32; one chunk, tiles over the right and bottom edges
    (1, 9, 40, 32, 128),      # NT 64, KC 32; two chunks, a second tile row of one image row
    (2, 17, 23, 48, 256),     # NT 64, KC 16; four chunks, three channel chunks
    (1, 8, 16, 16, 32),       # NT 32, KC 16; exactly one tile, one channel chunk
    (6, 40, 48, 32, 32),      # NT 32, KC 32; 90 tiles over six images
]
WINDOW_CASE = (1, 15, 18, 32, 64)   # NT 64, KC 32


@pytest.mark.parametrize('case', HALO_CONV_CASES)
def test_halo_conv_vs_oracle(case, gpu_device):
  B, H, W, Cin, Cout = case
  rng = np.random.default_rng(sum(case))
  x = rng.normal(size=(B, H, W, Cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, Cin, Cout)) / np.sqrt(9 * Cin)).astype(np.float32)
  b = rng.normal(size=(Cout,)).astype(np.float32)
  want = oracle.conv2d(x, w, b, 1, 'SAME', apply_relu=True, dtype=np.float64)
  got = conv2d_gpu(x, w, b, 1, 'SAME', relu=True, math_mode=TC)
  assert got.shape == want.shape and not np.isnan(got).any()
  assert rel_err(got, want) < CONV_RTOL, rel_err(got, want)
  # image borders carry the SAME zero padding: check them on their own scale
  for sl in (np.s_[:, 0], np.s_[:, -1], np.s_[:, :, 0], np.s_[:, :, -1]):
    assert rel_err(got[sl], want[sl]) < CONV_RTOL
  again = conv2d_gpu(x, w, b, 1, 'SAME', relu=True, math_mode=TC)
  assert np.array_equal(got, again)            # deterministic


def test_halo_conv_no_relu_affine_and_channel_window(gpu_device):
  B, H, W, Cin, Cout = WINDOW_CASE
  rng = np.random.default_rng(3)
  x = rng.normal(size=(B, H, W, Cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, Cin, Cout)) / 17).astype(np.float32)
  b = rng.normal(size=(Cout,)).astype(np.float32)
  sc = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
  sh = rng.normal(size=Cout).astype(np.float32)
  want = oracle.conv2d(x, w, b, 1, 'SAME', False, np.float64) * sc + sh
  y0 = np.full((B, H, W, 96), 7.0, np.float32)
  got = conv2d_gpu(x, w, b, 1, 'SAME', relu=False, scale=sc, shift=sh, y_cstride=96, y_coff=32,
                   math_mode=TC, y_init=y0)
  assert rel_err(got[..., 32:], want) < CONV_RTOL
  assert np.all(got[..., :32] == 7.0)          # untouched channels


def test_ragged_expand_pair_and_partial_batch(gpu_device):
  """An engine whose fire2 runs as squeeze + expand pair (too few tiles for the one-kernel fire):
  E1 = 24 != E3 = 72 over a 48-channel squeeze, one launch of 32-wide chunks (one 1x1, three 3x3,
  the last 8 channels wide) with K chunks of 16; then the 72-channel ConvDet head.  Each is
  checked against the oracle applied to the engine's own input tensor.  Forwards of n = 1, 2 of
  the 3 images give bitwise the rows of the full forward."""
  B, H, W = 3, 21, 37
  body = [('conv', 'conv1', 32, 3, 1, 'SAME'), ('fire', 'fire2', 48, 24, 72)]
  _, model, weights = build(body, B, H, W, TC, gpu_device)
  images = synth.synthetic_images(B, H, W, seed=3)
  model.detect(images)
  names = ('fire2/squeeze1x1', 'fire2', 'conv12')
  full = read_tensors(model, names)

  q = full['fire2/squeeze1x1'].astype(np.float64)
  for sub, k, got in (('expand1x1', 1, full['fire2'][..., :24]),
                      ('expand3x3', 3, full['fire2'][..., 24:])):
    kern, bias = weights['fire2/%s/kernels' % sub], weights['fire2/%s/biases' % sub]
    assert_within_bound(got, *conv_oracle(q, kern, bias, relu=True), k * k * 48, sub)
  kern, bias = weights['conv12/kernels'], weights['conv12/biases']
  assert kern.shape == (3, 3, 96, 72)
  assert_within_bound(full['conv12'], *conv_oracle(full['fire2'], kern, bias), 9 * 96, 'conv12')

  for n in (1, 2):
    forward_n(model, images, n)
    assert_rows_equal(read_tensors(model, names), full, n)
