"""The _params decode entry points on the host: sqdet_jpeg_parse_params reports the reduced,
oriented frame size the oracle decodes to, a scale_denom other than 1, 2, 4 or 8 is an argument
error, the size limits apply to the reduced size with SQDET_JPEG_CODED_TOO_LARGE for files cv2
decodes only reduced, and {progressive, 1} sizes are the plain and _progressive functions'
sizes.  No GPU: nothing here is decoded."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import jpeg_decode as D
from oracle import jpeg_decode_reduced as R
from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import decode_jpeg_device, jpeg_info

import jpeg_corpus as J

INVALID_ARG, UNSUPPORTED = -1, -3


def files():
  rng = np.random.default_rng(11)
  out = [f for _, f in J.corpus(seed=4, big=False)[::4]]
  for samp in J.SAMPLINGS:
    out.append(J.encode(J.content('noise', 45, 71, 3, rng), cv2.IMWRITE_JPEG_PROGRESSIVE, 1,
                        cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp, cv2.IMWRITE_JPEG_RST_INTERVAL, 2))
  out.append(D.with_orientation(J.encode(J.content('smooth', 37, 58, 3, rng), cv2.IMWRITE_JPEG_PROGRESSIVE, 1), 6))
  return out


def header_only(h, w):
  """A 4:2:0 file with its frame header claiming h x w: parsed, never decoded."""
  f = bytearray(J.encode(np.zeros((16, 16, 3), np.uint8)))
  k = f.index(b'\xff\xc0')
  f[k + 5:k + 9] = h.to_bytes(2, 'big') + w.to_bytes(2, 'big')
  return bytes(f)


def arrays(fs):
  bufs = [C.create_string_buffer(f, len(f)) for f in fs]
  return bufs, (C.c_void_p * len(fs))(*[C.addressof(b) for b in bufs]), (C.c_int64 * len(fs))(*map(len, fs))


def params(progressive=0, scale=1, reserved=(0, 0)):
  p = _lib.JpegDecodeParams(progressive, scale)
  p.reserved[0], p.reserved[1] = reserved
  return p


@pytest.mark.parametrize('s', (1, 2, 4, 8))
def test_parse_reports_the_reduced_size(s):
  for f in files():
    info, _ = R.parse(f, s)
    h, w = R.output_size(info, s)
    i = jpeg_info(f, progressive=True, reduce=s)
    assert i['supported'] and i['reason'] == 0, i['reason_text']
    assert (i['height'], i['width']) == ((w, h) if info.orientation >= 5 else (h, w))
    assert (i['coded_height'], i['coded_width']) == (info.height, info.width)
    if s > 1:
      assert cv2.imdecode(np.frombuffer(f, np.uint8), getattr(cv2, 'IMREAD_REDUCED_COLOR_%d' % s)).shape[:2] \
          == (i['height'], i['width'])


def test_params_1_sizes_are_the_old_sizes():
  lib = _lib.load()
  fs = files()
  seq = [f for f in fs if jpeg_info(f)['supported']]
  for batch, prog in ((seq, 0), (fs, 1), (fs[:1], 1), (seq[-3:], 0)):
    _, ptrs, lens = arrays(batch)
    kind = '_progressive' if prog else ''
    p = params(prog, 1)
    for fn in ('sqdet_jpeg_decode_staging_bytes', 'sqdet_jpeg_decode_scratch_bytes'):
      old = getattr(lib, fn + kind)(len(batch), ptrs, lens)
      assert old > 0 and getattr(lib, fn + '_params')(len(batch), ptrs, lens, C.byref(p)) == old, fn
    for f in batch:
      a, b = jpeg_info(f, progressive=bool(prog)), _lib.JpegInfo()
      assert lib.sqdet_jpeg_parse_params(C.create_string_buffer(f, len(f)), len(f), C.byref(p), C.byref(b)) == 0
      assert {k: int(getattr(b, k)) for k, _ in _lib.JpegInfo._fields_ if k not in ('reserved', 'supported')} \
          == {k: v for k, v in a.items() if k not in ('supported', 'reason_text')}


def test_reduced_scratch_shrinks_staging_does_not():
  lib = _lib.load()
  f = J.encode(J.content('smooth', 480, 640, 3, np.random.default_rng(3)), cv2.IMWRITE_JPEG_QUALITY, 95)
  _, ptrs, lens = arrays([f])
  sizes = {s: (lib.sqdet_jpeg_decode_staging_bytes_params(1, ptrs, lens, C.byref(params(0, s))),
               lib.sqdet_jpeg_decode_scratch_bytes_params(1, ptrs, lens, C.byref(params(0, s))))
           for s in (1, 2, 4, 8)}
  assert len({st for st, _ in sizes.values()}) == 1
  # the coefficients stay; the planes shrink: luma to 1/s, 4:2:0 chroma to 2/s (its IDCT at 1/2
  # is the full 8 x 8 one); each scratch region starts 256-byte aligned
  al = lambda x: -(-x // 256) * 256
  plane_bytes = lambda s: al(640 * 480 // s ** 2) + 2 * al(320 * 240 * 4 // s ** 2 if s > 1 else 320 * 240)
  for s in (1, 2, 4):
    assert sizes[s][1] - sizes[8][1] == plane_bytes(s) - plane_bytes(8), s


def test_bad_params_are_argument_errors():
  lib = _lib.load()
  f = J.encode(J.content('smooth', 20, 24, 3, np.random.default_rng(0)))
  _, ptrs, lens = arrays([f])
  out = _lib.JpegInfo()
  for p, what in ((params(0, 3), 'scale_denom'), (params(0, 0), 'scale_denom'), (params(1, 16), 'scale_denom'),
                  (params(0, -2), 'scale_denom'), (params(2, 2), 'progressive'), (params(0, 2, (1, 0)), 'reserved')):
    assert lib.sqdet_jpeg_parse_params(ptrs[0], len(f), C.byref(p), C.byref(out)) == INVALID_ARG
    assert what.encode() in lib.sqdet_last_error()
    assert lib.sqdet_jpeg_decode_staging_bytes_params(1, ptrs, lens, C.byref(p)) == -1
    assert lib.sqdet_jpeg_decode_scratch_bytes_params(1, ptrs, lens, C.byref(p)) == -1
    rc = lib.sqdet_decode_jpeg_params(1, ptrs, lens, C.byref(p), None, None, None, 0, None, 0, None, None)
    assert rc == INVALID_ARG and b'sqdet_decode_jpeg_params' in lib.sqdet_last_error()
  assert lib.sqdet_jpeg_parse_params(ptrs[0], len(f), None, C.byref(out)) == INVALID_ARG
  for s in (0, 3, 16, None):
    with pytest.raises(ValueError, match='reduce'):
      jpeg_info(f, reduce=s)
    with pytest.raises(ValueError, match='reduce'):
      decode_jpeg_device([f], 'cuda:0', reduce=s)


def test_plain_files_only_without_progressive():
  f = J.encode(J.content('smooth', 20, 24, 3, np.random.default_rng(0)), cv2.IMWRITE_JPEG_PROGRESSIVE, 1)
  for s in (2, 4, 8):
    i = jpeg_info(f, reduce=s)
    assert not i['supported'] and i['reason'] == D.PROGRESSIVE
    assert jpeg_info(f, progressive=True, reduce=s)['supported']


def test_size_reasons_follow_the_reduced_size():
  lib = _lib.load()
  big = header_only(30000, 40000)
  i = jpeg_info(big)
  assert i['reason'] == D.TOO_LARGE
  for s in (2, 4, 8):
    for prog in (False, True):
      i = jpeg_info(big, progressive=prog, reduce=s)
      assert not i['supported'] and i['reason'] == R.CODED_TOO_LARGE == 15
      assert i['reason_text'] == R.CODED_TOO_LARGE_TEXT
    _, ptrs, lens = arrays([big])
    assert lib.sqdet_jpeg_decode_scratch_bytes_params(1, ptrs, lens, C.byref(params(0, s))) == -1
    assert R.CODED_TOO_LARGE_TEXT.encode() in lib.sqdet_last_error()
    # refused before any device work, and routed to cv2, which decodes it at this scale
    with pytest.raises(ValueError, match='decode it with cv2.imdecode'):
      decode_jpeg_device([big], 'cuda:0', reduce=s)
  # a side above 65500 stays TOO_LARGE at every scale, as does a reduced size above 2^30 pixels
  for s in (1, 2, 4, 8):
    assert jpeg_info(header_only(16, 65501), reduce=s)['reason'] == D.TOO_LARGE
  assert jpeg_info(header_only(65500, 65500), reduce=2)['reason'] == R.CODED_TOO_LARGE
  with pytest.raises(ValueError, match='nor does cv2.imdecode'):
    decode_jpeg_device([header_only(30000, 40000)], 'cuda:0')
  # and 40000x30000 at 1/2 and 1/8 is what cv2 decodes, 1/1 what it refuses
  with pytest.raises(cv2.error):
    cv2.imdecode(np.frombuffer(big, np.uint8), cv2.IMREAD_COLOR)
  assert cv2.imdecode(np.frombuffer(big, np.uint8), cv2.IMREAD_REDUCED_COLOR_8).shape == (3750, 5000, 3)
