"""oracle.png restates cv2.imencode('.png') bitwise without zlib: sizes, contents, every corner
case of libpng's and zlib's writers, and the deflate body against zlib's own Z_RLE."""
import zlib

import cv2
import numpy as np
import pytest

from oracle import png as opng

import png_traps

SIZES = [(1, 1), (1, 2), (2, 1), (1, 17), (17, 1), (2, 3), (8, 8), (15, 31), (20, 30), (64, 64),
         (61, 97), (100, 1), (1, 3000), (376, 1241)]
KINDS = ('noise', 'flat', 'grad', 'half')


def content(kind, h, w, rng):
  if kind == 'noise':
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
  if kind == 'flat':
    return np.full((h, w, 3), 77, np.uint8)
  if kind == 'grad':
    y, x = np.mgrid[:h, :w]
    return ((y[..., None] * 3 + x[..., None] * 5 + np.arange(3) * 40) % 256).astype(np.uint8)
  img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
  img[:, w // 2:] = 50
  return img


def cv2_png(img):
  ok, buf = cv2.imencode('.png', img)
  assert ok
  return buf.tobytes()


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('h,w', SIZES)
def test_encode_bitwise(h, w, kind):
  img = content(kind, h, w, np.random.default_rng(h * 1000 + w))
  assert opng.encode(img) == cv2_png(img)


@pytest.mark.parametrize('h,w', [(375, 1242)])
def test_camera_size_noise(h, w):
  img = np.random.default_rng(0).integers(0, 256, (h, w, 3), dtype=np.uint8)
  info = {}
  assert opng.encode(img, info) == cv2_png(img)
  assert 'stored' in info['blocks']


@pytest.mark.parametrize('name', sorted(png_traps.traps()))
def test_traps(name):
  img, check = png_traps.traps()[name]
  info = {}
  assert opng.encode(img, info) == cv2_png(img)
  assert check(info), (name, info)


def test_one_pixel_wide_rows_use_filter_none():
  img = np.random.default_rng(3).integers(0, 256, (5, 1, 3), dtype=np.uint8)
  assert opng.filter_rows(img).reshape(5, 4)[:, 0].tolist() == [0] * 5
  assert opng.encode(img) == cv2_png(img)


def test_window_headers():
  """Every zlib window field libpng can leave, at the sizes where it changes."""
  seen = set()
  for w in png_traps.header_widths():
    img = np.zeros((1, w, 3), np.uint8)
    got = cv2_png(img)
    assert got[41:43] == opng.zlib_header(3 * w + 1), w
    seen.add(got[41] >> 4)
  assert seen == set(range(8))


@pytest.mark.parametrize('kind', KINDS)
def test_deflate_body_is_zlib_rle(kind):
  """Everything after the 2-byte header, Adler-32 included, is zlib's level-1 Z_RLE stream."""
  img = content(kind, 97, 211, np.random.default_rng(5))
  data = opng.filter_rows(img)
  c = zlib.compressobj(1, zlib.DEFLATED, 15, 8, zlib.Z_RLE)
  z = c.compress(data.tobytes()) + c.flush()
  assert opng.deflate_rle(data) == z[2:-4]
  assert opng.adler32(data) == zlib.adler32(data.tobytes())
  for name, (img, _) in png_traps.traps().items():
    data = opng.filter_rows(img)
    c = zlib.compressobj(1, zlib.DEFLATED, 15, 8, zlib.Z_RLE)
    assert opng.deflate_rle(data) == (c.compress(data.tobytes()) + c.flush())[2:-4], name


def test_crc32():
  for b in (b'', b'IEND', bytes(range(256)) * 3):
    assert opng.crc32(b) == zlib.crc32(b)


def test_cv2_side_limits():
  """cv2.imencode writes sides up to 1000000 (libpng's user limits) and refuses longer ones; the
  oracle refuses the same."""
  for shape in ((1, 1000000), (1000000, 1)):
    assert cv2.imencode('.png', np.zeros(shape + (3,), np.uint8))[0]
  for shape in ((1, 1000001), (1000001, 1)):
    try:
      ok = cv2.imencode('.png', np.zeros(shape + (3,), np.uint8))[0]
    except cv2.error:
      ok = False
    assert not ok, shape
    with pytest.raises(ValueError, match='1000000'):
      opng.encode(np.zeros(shape + (3,), np.uint8))
