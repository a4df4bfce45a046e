"""oracle.jpeg_decode_reduced.decode(f, reduce=s) is bitwise cv2.imdecode(f,
IMREAD_REDUCED_COLOR_s) for s in 2, 4, 8: every sampling at every width and height remainder
modulo 8 * hmax * 8 (planes down to one chroma sample), qualities 1 to 100, restart intervals,
EXIF orientations, progressive files, the handmade SOF1 files whose dequantized coefficients
overflow 16 bits, and other encoders' files.  reduce=1 is the full-size decode, and the size
limits apply to the reduced size."""
import cv2
import numpy as np
import pytest

from oracle import jpeg_decode as D
from oracle import jpeg_decode_reduced as R

import jpeg_corpus as J
import progressive_writer as PW

FLAGS = {1: cv2.IMREAD_COLOR, 2: cv2.IMREAD_REDUCED_COLOR_2, 4: cv2.IMREAD_REDUCED_COLOR_4,
         8: cv2.IMREAD_REDUCED_COLOR_8}
SCALES = (2, 4, 8)


def imdecode(f, s):
  return cv2.imdecode(np.frombuffer(f, np.uint8), FLAGS[s])


def same(f, name):
  for s in SCALES:
    want = imdecode(f, s)
    got = R.decode(f, s)
    assert want is not None and got.shape == want.shape, (name, s)
    assert np.array_equal(got, want), (name, s, int(np.abs(got.astype(int) - want).max()))


def reduced_shape(f, s):
  info = D.parse(f)
  h, w = R.output_size(info, s)
  return (w, h) if info.orientation >= 5 else (h, w)


# every sampling the decoder takes, with grayscale; (hmax, vmax) sets the remainders swept
LAYOUTS = [('gray', None, 1, 1), ('444', 0x111111, 1, 1), ('422', 0x211111, 2, 1),
           ('440', 0x121111, 1, 2), ('420', 0x221111, 2, 2), ('411', 0x411111, 4, 1)]


@pytest.mark.parametrize('name,samp,hmax,vmax', LAYOUTS, ids=[x[0] for x in LAYOUTS])
def test_every_remainder(name, samp, hmax, vmax):
  # widths 1 .. 64 * hmax and heights 1 .. 64 * vmax, paired by a stride, so that every
  # remainder modulo the MCU at 1/8 (and so at 1/2 and 1/4) is met in each direction
  rng = np.random.default_rng(hmax * 10 + vmax + (samp or 0) % 97)
  nw, nh = 64 * hmax, 64 * vmax
  n = max(nw, nh)
  for k in range(n):
    w, h = k % nw + 1, (k * 37) % nh + 1
    q = (1, 50, 95, 100)[k % 4]
    kind = J.KINDS[k % len(J.KINDS)]
    if samp is None:
      f = J.encode(J.content(kind, h, w, 1, rng)[..., 0], cv2.IMWRITE_JPEG_QUALITY, q)
    else:
      f = J.encode(J.content(kind, h, w, 3, rng), cv2.IMWRITE_JPEG_QUALITY, q,
                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)
    same(f, '%s %dx%d q%d' % (name, h, w, q))


def test_corpus():
  # qualities, restart intervals, optimized tables, split luma/chroma qualities, orientations
  for name, f in J.corpus(seed=3, big=False):
    same(f, name)


def test_restart_intervals():
  rng = np.random.default_rng(5)
  for samp in J.SAMPLINGS:
    img = J.content('smooth', 53, 77, 3, rng)
    for rst in (1, 3, 7):
      same(J.encode(img, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp, cv2.IMWRITE_JPEG_RST_INTERVAL, rst),
           'rst %d s%06x' % (rst, samp))


@pytest.mark.parametrize('o', range(1, 9))
def test_orientation(o):
  rng = np.random.default_rng(o)
  for samp in (0x221111, 0x211111, 0x121111):
    f = J.encode(J.content('noise', 29, 43, 3, rng), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)
    g = D.with_orientation(f, o, o % 2 == 0)
    same(g, 'exif %d s%06x' % (o, samp))
    assert imdecode(g, 4).shape[:2] == reduced_shape(g, 4)


def test_handmade():
  # SOF1 with 16-bit tables scaled until the 16-bit dequantization wraps and the 32-bit sums of
  # the reduced IDCTs overflow; colour-space markers; data and RSTs libjpeg skips
  for name, f in J.handmade():
    same(f, name)


def test_foreign():
  for name, f, _ in J.foreign()[::3]:
    same(f, name)


@pytest.mark.parametrize('samp', J.SAMPLINGS)
def test_progressive_cv2(samp):
  rng = np.random.default_rng(samp & 0xFFF)
  for zi, (h, w) in enumerate(J.SIZES[1::2]):
    q = (1, 50, 95, 100)[zi % 4]
    same(J.encode(J.content(J.KINDS[zi % len(J.KINDS)], h, w, 3, rng), cv2.IMWRITE_JPEG_PROGRESSIVE, 1,
                  cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp,
                  cv2.IMWRITE_JPEG_RST_INTERVAL, zi % 3), 'prog %dx%d s%06x' % (h, w, samp))


def test_progressive_scripts():
  rng = np.random.default_rng(7)
  src = J.encode(J.content('smooth', 37, 58, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90)
  gray = J.encode(J.content('noise', 33, 47, 1, rng)[..., 0], cv2.IMWRITE_JPEG_QUALITY, 80)
  for name, script in PW.COMPLETE.items():
    same(PW.write(gray if name.startswith('gray') else src, script), name)


def test_reduce_1_is_the_full_decode():
  rng = np.random.default_rng(8)
  for samp in J.SAMPLINGS:
    f = J.encode(J.content('noise', 41, 59, 3, rng), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)
    assert np.array_equal(R.decode(f, 1), D.decode(f))
    assert np.array_equal(R.decode(f, 1), J.imdecode(f))
  with pytest.raises(ValueError):
    R.decode(f, 3)


def test_plan():
  # the chroma IDCT-size rule: 4:2:0 chroma doubles (no upsampling), the others stay at luma's
  # size and are upsampled; fancy only above 1/8
  rng = np.random.default_rng(9)
  want = {0x221111: {2: (8, 1, 1), 4: (4, 1, 1), 8: (2, 1, 1)},
          0x211111: {2: (4, 2, 1), 4: (2, 2, 1), 8: (1, 2, 1)},
          0x121111: {2: (4, 1, 2), 4: (2, 1, 2), 8: (1, 1, 2)},
          0x411111: {2: (4, 4, 1), 4: (2, 4, 1), 8: (1, 4, 1)},
          0x111111: {2: (4, 1, 1), 4: (2, 1, 1), 8: (1, 1, 1)}}
  for samp, by_s in want.items():
    info = D.parse(J.encode(J.content('flat', 16, 16, 3, rng), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp))
    for s, (n, fh, fv) in by_s.items():
      luma, cb, cr = R.plan(info, s)
      assert luma.size == 8 // s and (luma.fh, luma.fv) == (1, 1)
      assert cb == cr and (cb.size, cb.fh, cb.fv) == (n, fh, fv) and cb.fancy == (s < 8)


def header_only(h, w):
  """A 4:2:0 file from cv2 with its frame header claiming h x w: parsed, never decoded."""
  f = bytearray(J.encode(np.zeros((16, 16, 3), np.uint8)))
  k = f.index(b'\xff\xc0')
  f[k + 5:k + 9] = h.to_bytes(2, 'big') + w.to_bytes(2, 'big')
  return bytes(f)


def test_size_limits_apply_to_the_reduced_size():
  big = header_only(30000, 40000)
  with pytest.raises(D.Unsupported) as e:
    D.parse(big)
  assert e.value.reason == D.TOO_LARGE
  for s in SCALES:
    for progressive in (False, True):
      with pytest.raises(D.Unsupported) as e:
        R.parse(big, s, progressive)
      assert e.value.reason == R.CODED_TOO_LARGE and str(e.value) == R.CODED_TOO_LARGE_TEXT
  with pytest.raises(cv2.error):
    imdecode(big, 1)
  assert imdecode(big, 8).shape == (3750, 5000, 3)
  # a side above 65500 is refused at any scale, by libjpeg as by the oracle
  wide = header_only(16, 65501)
  for s in (1,) + SCALES:
    assert imdecode(wide, s) is None
    with pytest.raises(D.Unsupported) as e:
      R.parse(wide, s)
    assert e.value.reason == D.TOO_LARGE
  # 65500 x 65500 is over 2^30 pixels at 1/1 but not at 1/2 and below
  most = header_only(65500, 65500)
  with pytest.raises(D.Unsupported) as e:
    R.parse(most, 2)
  assert e.value.reason == R.CODED_TOO_LARGE
