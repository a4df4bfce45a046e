"""oracle.jpeg is cv2.imencode('.jpg', ...) byte for byte: sizes, qualities, contents, every pixel
format through cv2.cvtColor, and crops at odd origins."""
import cv2
import numpy as np
import pytest

from oracle import jpeg, pixfmt

SIZES = [(1, 1), (1, 17), (17, 1), (2, 3), (8, 8), (15, 31), (16, 16), (17, 23), (61, 97),
         (375, 1242), (370, 1224), (376, 1241)]
QUALITIES = [1, 10, 50, 75, 95, 100]
KINDS = ('noise', 'grad', 'flat', 'check', 'blocks', 'dots')


def content(kind, h, w, c, rng):
  """uint8 [h, w, c]: noise, gradients, flat (EOB only), 0/255 checkerboards of pixels (the
  largest AC coefficients; at low quality zero runs of 16 and more: ZRL) or of 8x8 blocks (DC
  differences of category 11), or isolated dots on flat grey."""
  if kind == 'noise':
    return rng.integers(0, 256, (h, w, c), dtype=np.uint8)
  y, x = np.mgrid[:h, :w]
  if kind == 'grad':
    return ((y[..., None] * 3 + x[..., None] * 5 + np.arange(c) * 40) % 256).astype(np.uint8)
  if kind == 'flat':
    return np.full((h, w, c), 77, np.uint8)
  if kind in ('check', 'blocks'):     # 0/255 per pixel, or per 8x8 block (DC category 11)
    cell = (y + x) % 2 if kind == 'check' else (y // 8 + x // 8) % 2
    return np.repeat((cell * 255).astype(np.uint8)[..., None], c, axis=2)
  img = np.full((h, w, c), 128, np.uint8)
  img[(y % 8 == 7) & (x % 8 == 7)] = 255
  return img


def cv2_jpeg(bgr, quality):
  return cv2.imencode('.jpg', np.ascontiguousarray(bgr), [cv2.IMWRITE_JPEG_QUALITY, quality])[1].tobytes()


@pytest.mark.parametrize('quality', QUALITIES)
@pytest.mark.parametrize('size', SIZES, ids=lambda s: '%dx%d' % s)
def test_sizes_qualities_contents(size, quality):
  rng = np.random.default_rng(size[0] * 1000 + size[1] + quality)
  for kind in KINDS:
    img = content(kind, *size, 3, rng)
    assert jpeg.encode(img, quality) == cv2_jpeg(img, quality), kind


def test_contents_reach_the_coder_edges():
  """The contents exercise what they are there for: DC category 11, ZRL, and 0xFF stuffing."""
  rng = np.random.default_rng(0)
  yq, _, _ = jpeg.coefficients(content('blocks', 16, 16, 3, rng), 100)
  assert np.abs(np.diff(np.concatenate([[0], yq[..., 0].ravel()]))).max() >= 1024
  yq, _, _ = jpeg.coefficients(content('check', 16, 16, 3, rng), 10)
  nz = [np.nonzero(b[1:])[0] for b in yq.reshape(-1, 64)]
  assert any(len(k) and (k[0] >= 16 or (np.diff(k) > 16).any()) for k in nz)
  data = jpeg.encode(content('noise', 61, 97, 3, rng), 95)
  scan = data[len(jpeg.header(61, 97, 95)):-2]
  assert b'\xff\x00' in scan


@pytest.mark.parametrize('fmt', pixfmt.FORMATS)
def test_every_format_through_cvtcolor(fmt):
  rng = np.random.default_rng(len(fmt))
  h, w = 62, 98
  if fmt in ('bgr', 'rgb', 'bgra', 'rgba'):
    planes = [rng.integers(0, 256, (h, w, 4 if 'a' in fmt else 3), dtype=np.uint8)]
  elif fmt == 'rgb_planar':
    planes = list(rng.integers(0, 256, (3, h, w), dtype=np.uint8))
  elif fmt == 'nv12':
    planes = [rng.integers(0, 256, (h, w), dtype=np.uint8),
              rng.integers(0, 256, (h // 2, w), dtype=np.uint8)]
  else:
    planes = [rng.integers(0, 256, (h, w), dtype=np.uint8),
              rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8),
              rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8)]
  bgr = pixfmt.to_bgr(fmt, planes)
  for quality in (50, 95):
    assert jpeg.encode(bgr, quality) == cv2_jpeg(bgr, quality)


@pytest.mark.parametrize('crop', [(1, 1, 17, 23), (3, 5, 61, 33), (7, 9, 1, 1), (5, 0, 40, 57)])
def test_crops_at_odd_origins(crop):
  rng = np.random.default_rng(9)
  frame = content('noise', 64, 80, 3, rng)
  x, y, w, h = crop
  sub = frame[y:y + h, x:x + w]
  assert jpeg.encode(sub, 95) == cv2_jpeg(sub, 95)


def test_reciprocal_is_rounding_division():
  """libjpeg-turbo's reciprocal multiply equals division by 8 q rounded half away from zero for
  every coefficient an 8-bit FDCT can produce."""
  x = np.arange(-(1 << 15) + 1, 1 << 15, dtype=np.int64)
  for q in range(1, 256):
    d = 8 * q
    want = np.sign(x) * ((np.abs(x) + d // 2) // d)
    assert (jpeg.quantize(x, d) == want).all(), d


def test_quantization_tables_clamp():
  qy, qc = jpeg.quant_tables(1)
  assert qy.max() == qc.max() == 255
  qy, qc = jpeg.quant_tables(100)
  assert qy.min() == qc.min() == qy.max() == 1
  with pytest.raises(ValueError):
    jpeg.quant_tables(0)
