"""Pins oracle.pixfmt.to_bgr bitwise against the installed cv2's cvtColor, for every format of the
generic device-frames path (sqdet_forward_frames)."""
import numpy as np
import pytest

from oracle import pixfmt

cv2 = pytest.importorskip('cv2')

# packed and planar formats take any size; odd widths and heights included
SHAPES = [(1080, 1920), (375, 1242), (7, 13), (3, 1), (1, 5), (2, 2)]
YUV_SHAPES = [(1080, 1920), (376, 1242), (370, 1224), (2, 2), (2, 4), (10, 6)]


def frame(fmt, h, w, rng):
  """(planes for pixfmt.to_bgr, the cv2.cvtColor result they must give)."""
  u8 = lambda *s: rng.integers(0, 256, s, dtype=np.uint8)  # noqa: E731
  if fmt == 'bgr':
    f = u8(h, w, 3)
    return (f,), f
  if fmt in ('rgb', 'bgra', 'rgba'):
    f = u8(h, w, 3 if fmt == 'rgb' else 4)
    code = {'rgb': cv2.COLOR_RGB2BGR, 'bgra': cv2.COLOR_BGRA2BGR, 'rgba': cv2.COLOR_RGBA2BGR}[fmt]
    return (f,), cv2.cvtColor(f, code)
  if fmt == 'rgb_planar':
    r, g, b = u8(h, w), u8(h, w), u8(h, w)
    return (r, g, b), cv2.cvtColor(np.ascontiguousarray(np.stack([r, g, b], -1)), cv2.COLOR_RGB2BGR)
  if fmt == 'nv12':
    y, uv = u8(h, w), u8(h // 2, w)
    return (y, uv), cv2.cvtColor(np.concatenate([y, uv]), cv2.COLOR_YUV2BGR_NV12)
  y, u, v = u8(h, w), u8(h // 2, w // 2), u8(h // 2, w // 2)
  return (y, u, v), cv2.cvtColor(i420_stacked(y, u, v), cv2.COLOR_YUV2BGR_I420)


def i420_stacked(y, u, v):
  """The [3h/2, w] array cv2 takes: Y's rows, then U's bytes, then V's."""
  h, w = y.shape
  return np.concatenate([y.ravel(), u.ravel(), v.ravel()]).reshape(3 * h // 2, w)


@pytest.mark.parametrize('h,w', SHAPES)
@pytest.mark.parametrize('fmt', ['bgr', 'rgb', 'bgra', 'rgba', 'rgb_planar'])
def test_packed_and_planar_bitwise_cv2(fmt, h, w):
  planes, want = frame(fmt, h, w, np.random.default_rng(h * 31 + w))
  got = pixfmt.to_bgr(fmt, planes)
  assert got.dtype == np.uint8 and got.shape == (h, w, 3)
  np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize('h,w', YUV_SHAPES)
@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_yuv_bitwise_cv2(fmt, h, w):
  planes, want = frame(fmt, h, w, np.random.default_rng(h * 31 + w))
  got = pixfmt.to_bgr(fmt, planes)
  assert got.dtype == np.uint8 and got.shape == (h, w, 3)
  np.testing.assert_array_equal(got, want)


def test_i420_every_yuv_triple():
  """All 256^3 (Y, U, V) triples in one 4096 x 4096 frame: 2x2 block b (row-major over the
  2048 x 2048 blocks) has chroma sample b % 65536 and luma 4 * (b // 65536) + {0, 1, 2, 3}."""
  b = np.arange(2048 * 2048).reshape(2048, 2048)
  uv = b % 65536
  u, v = (uv >> 8).astype(np.uint8), (uv & 255).astype(np.uint8)
  base = 4 * (b // 65536)
  luma = np.empty((4096, 4096), np.uint8)
  for k, (r, c) in enumerate([(0, 0), (0, 1), (1, 0), (1, 1)]):
    luma[r::2, c::2] = base + k
  want = cv2.cvtColor(i420_stacked(luma, u, v), cv2.COLOR_YUV2BGR_I420)
  np.testing.assert_array_equal(pixfmt.to_bgr('i420', (luma, u, v)), want)


def test_unknown_format():
  with pytest.raises(ValueError):
    pixfmt.to_bgr('yuy2', (np.zeros((2, 4), np.uint8),))
