"""The size limits of cv2's JPEG codec, kept in both directions without a GPU: cv2.imencode writes
sides up to 65500 (libjpeg's JPEG_MAX_DIMENSION), and cv2.imdecode decodes sides up to 65500 and at
most 2^30 pixels (cv2's default CV_IO_MAX_IMAGE_PIXELS).  The encoder refuses the sizes cv2 does
not write, the decoder's parse and the oracle's refuse the files cv2 does not decode, and the
oracles stay cv2 at every quality and on strips as long as a JPEG may be."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import jpeg as E
from oracle import jpeg_decode as D
from squeezedet_b200 import _lib
from squeezedet_b200 import jpeg as sj
from squeezedet_b200.jpeg import jpeg_info

import jpeg_corpus as J

MAX_SIDE = 65500
FAKE = 1 << 40            # never dereferenced: the size checks come first
STRIPS = [(1, MAX_SIDE), (MAX_SIDE, 1), (16, MAX_SIDE), (MAX_SIDE, 16)]


def with_size(f, h, w):
  """f with the height and width of its SOF0 replaced (its data is then short or long for them:
  libjpeg warns and fills or skips)."""
  b = bytearray(f)
  k = bytes(b).index(b'\xff\xc0')
  b[k + 5:k + 9] = h.to_bytes(2, 'big') + w.to_bytes(2, 'big')
  return bytes(b)


@pytest.fixture(scope='module')
def small():
  """A 16x16 cv2 file, 4:2:0."""
  return J.encode(J.content('smooth', 16, 16, 3, np.random.default_rng(0)), cv2.IMWRITE_JPEG_QUALITY, 90)


# ---- cv2's limits, and what the parses say ---------------------------------------------------------
# (coded height, coded width, what cv2.imdecode does: 'decodes', 'none' or 'raises'); a file cv2
# decodes is supported, any other refused as TOO_LARGE.  65500 x 16393 = 2^30 - 324 pixels is not
# decoded here (3 GB for nothing the 32768 x 32768 row does not show).
ROWS = [(MAX_SIDE, 16, 'decodes'), (16, MAX_SIDE, 'decodes'),
        (MAX_SIDE + 1, 16, 'none'), (16, MAX_SIDE + 1, 'none'),
        (65535, 16, 'none'), (16, 65535, 'none'), (65535, 65535, 'none'),
        (32768, 32768, 'decodes'), (32768, 32769, 'raises'),
        (MAX_SIDE, 16394, 'raises'), (MAX_SIDE, 16393, None)]


def cv2_outcome(f):
  try:
    img = J.imdecode(f)
  except cv2.error:
    return 'raises', None
  return ('none', None) if img is None else ('decodes', img.shape)


@pytest.mark.parametrize('h,w,cv', ROWS, ids=['%dx%d' % r[:2] for r in ROWS])
def test_cv2_limits_and_parse(small, h, w, cv):
  f = with_size(small, h, w)
  if cv is not None:
    got, shape = cv2_outcome(f)
    assert got == cv, 'cv2.imdecode of a %dx%d file: %s, not %s' % (w, h, got, cv)
    if shape is not None:
      assert shape == (h, w, 3)
  else:
    assert h * w == (1 << 30) - 324
  supported = cv in ('decodes', None)
  i = jpeg_info(f)
  assert i['supported'] == supported, i
  assert i['reason'] == (D.OK if supported else D.TOO_LARGE), i
  if supported:
    p = D.parse(f)
    assert (i['coded_height'], i['coded_width']) == (p.height, p.width) == (h, w)
  else:
    with pytest.raises(D.Unsupported) as e:
      D.parse(f)
    assert e.value.reason == D.TOO_LARGE
    assert i['reason_text'] == D.REASONS[D.TOO_LARGE] == 'larger than cv2 decodes'


def test_limits_apply_to_the_coded_size(small):
  """Orientation 6 swaps the sides after decoding; the limits are on the sides SOF gives, as in
  cv2."""
  wide = D.with_orientation(with_size(small, 16, MAX_SIDE + 1), 6)
  assert J.imdecode(wide) is None
  i = jpeg_info(wide)
  assert not i['supported'] and i['reason'] == D.TOO_LARGE, i
  with pytest.raises(D.Unsupported) as e:
    D.parse(wide)
  assert e.value.reason == D.TOO_LARGE
  tall = D.with_orientation(with_size(small, MAX_SIDE, 16), 6)
  i = jpeg_info(tall)
  assert i['supported'] and (i['height'], i['width']) == (16, MAX_SIDE) == D.parse(tall).out_hw, i


def sizes(f):
  """(sqdet_jpeg_decode_staging_bytes, sqdet_jpeg_decode_scratch_bytes) of file f."""
  lib = _lib.load()
  buf = C.create_string_buffer(f, len(f))
  ptrs, lens = (C.c_void_p * 1)(C.addressof(buf)), (C.c_int64 * 1)(len(f))
  return lib.sqdet_jpeg_decode_staging_bytes(1, ptrs, lens), lib.sqdet_jpeg_decode_scratch_bytes(1, ptrs, lens)


@pytest.mark.parametrize('samp', [0x221111, 0x111111, None], ids=['420', '444', 'gray'])
@pytest.mark.parametrize('hw', [(32768, 32768), (MAX_SIDE, 16393), (16393, MAX_SIDE)], ids=str)
def test_scratch_of_the_largest_files(samp, hw):
  """The scratch of the largest files the decoder takes holds at least their coefficients, 128
  bytes per block: the layout arithmetic does not overflow.  Files past the limits get -1."""
  img = J.content('smooth', 16, 16, 3, np.random.default_rng(1))
  f = J.encode(img[..., 0]) if samp is None else J.encode(img, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)
  g = with_size(f, *hw)
  info = D.parse(g)
  _, mcols, mrows = D.mcu_geometry(info)
  blocks = mcols * mrows * (sum(c.h * c.v for c in info.comps) if len(info.comps) == 3 else 1)
  staging, scratch = sizes(g)
  assert 0 < staging < len(g) + 16384
  assert scratch >= blocks * 128 >= 1 << 31
  assert sizes(with_size(f, hw[0], hw[1] + 1)) == (-1, -1)


def test_decode_refuses_past_the_limits(small):
  """sqdet_decode_jpeg refuses such a file before any device work, naming it."""
  lib = _lib.load()
  for h, w in [(16, MAX_SIDE + 1), (32768, 32769), (65535, 65535)]:
    files = [small, with_size(small, h, w)]
    bufs = [C.create_string_buffer(f, len(f)) for f in files]
    rc = lib.sqdet_decode_jpeg(2, (C.c_void_p * 2)(*[C.addressof(b) for b in bufs]),
                               (C.c_int64 * 2)(*[len(f) for f in files]), (C.c_void_p * 2)(FAKE, FAKE),
                               (C.c_int64 * 2)(3 * 16, 3 * 16), FAKE, 1 << 40, FAKE, 1 << 40, FAKE, None)
    assert rc == -3
    msg = lib.sqdet_last_error()
    assert b'file 1' in msg and b'larger than cv2 decodes' in msg, msg
  assert sj.JPEG_TOO_LARGE == D.TOO_LARGE


# ---- the encoder's limits ------------------------------------------------------------------------
@pytest.mark.parametrize('h,w,ok', [(1, MAX_SIDE, True), (MAX_SIDE, 1, True),
                                    (1, MAX_SIDE + 1, False), (MAX_SIDE + 1, 1, False)])
def test_cv2_imencode_limit(h, w, ok):
  assert cv2.imencode('.jpg', np.zeros((h, w, 3), np.uint8))[0] == ok


def test_max_bytes_limit():
  lib = _lib.load()
  for h, w in [(1, MAX_SIDE + 1), (MAX_SIDE + 1, 1), (65535, 65535)]:
    assert lib.sqdet_jpeg_max_bytes(h, w) == -1
    assert b'65500' in lib.sqdet_last_error()
    with pytest.raises(ValueError, match='65500'):
      sj.max_bytes(h, w)
  for h, w in [(MAX_SIDE, MAX_SIDE), (1, MAX_SIDE), (MAX_SIDE, 1)]:
    blocks = -(-h // 16) * -(-w // 16) * 6
    want = len(E.header(h, w, 95)) + 2 * -(-blocks * (22 + 63 * 26) // 8) + 2
    assert lib.sqdet_jpeg_max_bytes(h, w) == sj.max_bytes(h, w) == want


def crop_arrays(frame_hw, crop):
  """Frame 0 a small one, frame 1 of frame_hw cropped to crop (x, y, w, h)."""
  hs = (C.c_int32 * 2)(16, frame_hw[0])
  ws = (C.c_int32 * 2)(16, frame_hw[1])
  cr = (C.c_int32 * 8)(0, 0, 16, 16, *crop)
  return hs, ws, cr


@pytest.mark.parametrize('frame_hw,crop', [((70000, 8), (0, 3, 8, MAX_SIDE + 1)),
                                           ((8, 100000), (7, 0, MAX_SIDE + 1, 8))], ids=['tall', 'wide'])
def test_encoder_refuses_longer_crops(frame_hw, crop):
  """A crop longer than 65500 of a larger frame is refused by the scratch size and the encode,
  naming the frame, before anything touches the (fake) device pointers; the same crop 1 shorter
  is sized."""
  lib = _lib.load()
  hs, ws, cr = crop_arrays(frame_hw, crop)
  assert lib.sqdet_jpeg_scratch_bytes(2, hs, ws, cr) == -1
  msg = lib.sqdet_last_error()
  assert b'frame 1' in msg and b'65500' in msg, msg
  host = (C.c_uint8 * 64)()
  planes = (C.c_void_p * 6)(*[C.addressof(host)] * 6)
  rc = lib.sqdet_encode_jpeg(2, 0, planes, None, hs, ws, cr, 95, FAKE, 1 << 20, FAKE, FAKE, 1 << 40, None)
  msg = lib.sqdet_last_error()
  assert rc == -1 and b'frame 1' in msg and b'65500' in msg, msg
  x, y, w, h = crop
  hs, ws, cr = crop_arrays(frame_hw, (x, y, min(w, MAX_SIDE), min(h, MAX_SIDE)))
  assert lib.sqdet_jpeg_scratch_bytes(2, hs, ws, cr) > 0


def test_oracle_encode_refuses_longer_sides():
  for h, w in [(1, MAX_SIDE + 1), (MAX_SIDE + 1, 1)]:
    with pytest.raises(ValueError, match='65500'):
      E.encode(np.zeros((h, w, 3), np.uint8))


# ---- the oracles at every quality and on the longest strips ---------------------------------------
def cv2_jpeg(bgr, quality):
  return cv2.imencode('.jpg', np.ascontiguousarray(bgr), [cv2.IMWRITE_JPEG_QUALITY, quality])[1].tobytes()


@pytest.mark.parametrize('quality', range(1, 101))
def test_oracle_encode_every_quality(quality):
  """Below 50 the tables scale by 5000 / quality, and at low qualities entries clamp to 255."""
  rng = np.random.default_rng(quality)
  for h, w in [(17, 23), (61, 97)]:
    for kind in ('noise', 'check'):
      img = J.content(kind, h, w, 3, rng)
      assert E.encode(img, quality) == cv2_jpeg(img, quality), (h, w, kind)


@pytest.mark.parametrize('hw', [(1, MAX_SIDE), (MAX_SIDE, 1), (16, MAX_SIDE)], ids=str)
def test_oracle_encode_longest_strips(hw):
  rng = np.random.default_rng(hw[0])
  for kind, quality in (('smooth', 95), ('noise', 50)):
    img = J.content(kind, *hw, 3, rng)
    assert E.encode(img, quality) == cv2_jpeg(img, quality), kind


@pytest.mark.parametrize('hw', STRIPS, ids=str)
def test_oracle_decode_longest_strips(hw):
  rng = np.random.default_rng(hw[1])
  img = J.content('smooth', *hw, 3, rng)
  files = [('gray', J.encode(img[..., 0], cv2.IMWRITE_JPEG_QUALITY, 90))]
  files += [('s%06x' % s, J.encode(img, cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, s))
            for s in J.SAMPLINGS]
  for name, f in files:
    assert np.array_equal(D.decode(f), J.imdecode(f)), name
