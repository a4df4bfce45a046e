"""The operand ring of the tensor-core convolution (conv_tc.cu): TMA tensor-map loads of the
activations, one bulk copy per weight tile, and full / empty mbarriers per stage instead of a block
barrier.  K chunk counts below, at and just above the three stages, a 216-chunk K (the ConvDet
head's, over which each barrier's phase wraps 72 times), several output-channel chunks in one
launch, both K chunk widths (so both the 128-byte and the 64-byte swizzle), a row-mode pixel count
that is not a multiple of 128, tiles hanging over the image (TMA zero fill), gather mode, and the
one-shot entry called on a second set of buffers; engines whose forwards change the image count
and the input buffer, through the convolution and the one-kernel fire.  Each element is checked
against the fp64 oracle with the bar gpu_util.adv_tol, and bitwise against a repeat run."""
import numpy as np
import pytest

from squeezedet_b200 import _lib
from squeezedet_b200.utils import synth
from gpu_util import (ONE_KERNEL_MIN_TILES, POST_LAUNCHES, assert_rows_equal, assert_within_bound,
                      build, conv2d_gpu, conv_oracle, fire_tiles, read_tensors)

pytestmark = pytest.mark.gpu
TC = _lib.MATH_TF32X3_TC


def check_conv(x, w, stride=1, padding='SAME', seed=0):
  k, Cin = w.shape[0], w.shape[2]
  rng = np.random.default_rng(seed)
  b = rng.normal(size=w.shape[3]).astype(np.float32)
  want, bound = conv_oracle(x, w, b, stride, padding)
  got = conv2d_gpu(x, w, b, stride, padding, relu=False, math_mode=TC)
  assert got.shape == want.shape and not np.isnan(got).any()
  assert_within_bound(got, want, bound, k * k * Cin, (x.shape, w.shape))
  again = conv2d_gpu(x, w, b, stride, padding, relu=False, math_mode=TC)
  assert got.tobytes() == again.tobytes()
  return got


def make(B, H, W, Cin, Cout, k, seed):
  rng = np.random.default_rng(seed)
  x = rng.normal(size=(B, H, W, Cin)).astype(np.float32)
  w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(np.float32)
  return x, w


ROW_CASES = [
    # B, H, W, Cin, Cout: row mode (1x1), K chunks = Cin / KC (KC 32 when Cin % 32 == 0, else 16)
    (1, 4, 5, 16, 16),       # 1 K chunk of 16, M = 20 < one 128-pixel tile
    (2, 7, 11, 32, 40),      # 1 K chunk of 32, M = 154 (a 26-pixel tail tile); NT 64
    (1, 9, 15, 64, 24),      # 2 K chunks of 32
    (3, 5, 13, 48, 16),      # 3 K chunks of 16: exactly the stage count
    (1, 16, 16, 128, 200),   # 4 K chunks of 32 (one past the stages); 4 output-channel chunks
    (2, 3, 29, 112, 96),     # 7 K chunks of 16 (one past two rings)
]


@pytest.mark.parametrize('case', ROW_CASES)
def test_row_mode_ring(case, gpu_device):
  B, H, W, Cin, Cout = case
  check_conv(*make(B, H, W, Cin, Cout, 1, sum(case)), seed=1)


HALO_CASES = [
    # B, H, W, Cin, Cout: halo mode (3x3), 9 K chunks per channel chunk
    (1, 3, 5, 16, 16),       # 9 K chunks of 16, one tile mostly outside the image
    (2, 8, 16, 32, 16),      # 9 K chunks of 32, exactly one tile
    (1, 9, 17, 48, 130),     # 27 K chunks of 16, tiles over the right and bottom edges; 3 chunks
    (1, 9, 17, 768, 72),     # 216 K chunks of 32 (the ConvDet head's K); the 72-wide tile
    (2, 11, 35, 64, 64),     # 18 K chunks of 32, both halo buffers in use
]


@pytest.mark.parametrize('case', HALO_CASES)
def test_halo_mode_ring(case, gpu_device):
  B, H, W, Cin, Cout = case
  x, w = make(B, H, W, Cin, Cout, 3, sum(case))
  got = check_conv(x, w, seed=2)
  # an image's tiles do not depend on the batch around it (a tensor map of one image)
  if B > 1:
    first = conv2d_gpu(x[:1], w, np.random.default_rng(2).normal(size=Cout).astype(np.float32), 1,
                       'SAME', relu=False, math_mode=TC)
    assert first.tobytes() == got[:1].tobytes()


@pytest.mark.parametrize('stride', [1, 2])
def test_gather_mode_ring(stride, gpu_device):
  """3-channel 3x3 convs: cp.async into the swizzled tile, completing on the stage's mbarrier."""
  x, w = make(2, 13, 37, 3, 64, 3, stride)
  check_conv(x, w, stride=stride, seed=3)


def test_oneshot_on_second_buffers(gpu_device):
  """Two one-shot calls of the same shape on different inputs (and so different buffers): each
  encodes its tensor maps for its own input."""
  x1, w = make(1, 10, 20, 32, 32, 3, 11)
  x2 = -2.0 * x1[:, ::-1]
  y1 = check_conv(x1, w, seed=4)
  y2 = check_conv(np.ascontiguousarray(x2), w, seed=4)
  assert not np.array_equal(y1, y2)


def assert_rows_follow_full_forward(model, B, H, W, names, runs, device):
  """For each (i, n) of `runs`, the first a full forward, runs a forward of n images from input
  buffer i (all buffers hold the same images) and checks that the tensors `names` hold bitwise the
  first forward's rows."""
  images = np.ascontiguousarray(synth.synthetic_images(B, H, W, seed=9), np.float32)
  bufs = [_lib.DeviceBuffer.from_numpy(images, device) for _ in range(1 + max(i for i, _ in runs))]
  full = None
  for i, n in runs:
    model.forward_device(bufs[i].ptr, None, n)
    _lib.check(model._lib.sqdet_stream_sync(device, None))
    got = read_tensors(model, names)
    if full is None:
      full = got
    assert_rows_equal(got, full, n, i)
  for buf in bufs:
    buf.free()


def test_cached_maps_follow_image_count(gpu_device):
  """An engine plan caches its tensor maps per (input, image count): forwards of n = 3, 1, 2, 3
  images give bitwise the rows of the first full forward, through row mode (the squeeze),
  halo mode (the expand pair and the head)."""
  B, H, W = 3, 19, 41
  body = [('conv', 'conv1', 32, 3, 1, 'SAME'), ('fire', 'fire2', 32, 64, 64)]
  _, model, _ = build(body, B, H, W, TC, gpu_device)
  assert_rows_follow_full_forward(model, B, H, W, ('fire2/squeeze1x1', 'fire2', 'conv12'),
                                  [(0, 3), (0, 1), (0, 2), (0, 3)], gpu_device)


def test_cached_fire_map_follows_image_count(gpu_device):
  """The same through the one-kernel fire, whose plan caches the halo map of its squeeze: a
  16-channel squeeze on 3 x 64 x 352 (528 tiles, 4 per SM on 132 SMs).  Forwards of n = 3, 1, 2,
  3 images, then from a second input buffer, give bitwise the rows of the first full forward.
  (The fire reads conv1's output, so the second buffer is the input of conv1 only.)"""
  B, H, W = 3, 64, 352
  assert fire_tiles(B, H, W) >= ONE_KERNEL_MIN_TILES
  body = [('conv', 'conv1', 32, 3, 1, 'SAME'), ('fire', 'fire2', 16, 64, 64)]
  _, model, _ = build(body, B, H, W, TC, gpu_device)
  assert model.launches_per_forward() == 3 + POST_LAUNCHES     # conv1, fire2 as one kernel, head
  assert_rows_follow_full_forward(model, B, H, W, ('conv1', 'fire2', 'conv12'),
                                  [(0, 3), (0, 1), (0, 2), (0, 3), (1, 3), (1, 2), (0, 1)],
                                  gpu_device)
