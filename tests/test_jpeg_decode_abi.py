"""sqdet_jpeg_parse reports sizes, sampling, orientation and refusal reasons on the host, and
sqdet_decode_jpeg refuses bad arguments before any device work, so without a GPU too."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import jpeg_decode as D
from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import jpeg_info

import jpeg_corpus as J

FAKE = 1 << 40            # never dereferenced: the argument checks come first


def img(h=20, w=24, c=3):
  x = J.content('smooth', h, w, 3, np.random.default_rng(0))
  return x if c == 3 else cv2.cvtColor(x, cv2.COLOR_BGR2GRAY)


def segment(marker, body):
  return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, 'big') + body


def with_sof(f, marker=None, precision=None):
  """f with its SOF0 marker or precision replaced."""
  b = bytearray(f)
  k = bytes(b).index(b'\xff\xc0')
  if marker is not None:
    b[k + 1] = marker
  if precision is not None:
    b[k + 4] = precision
  return bytes(b)


def four_components(f):
  """f with a CMYK-like SOF0 of four 1x1 components in place of its own."""
  k = f.index(b'\xff\xc0')
  n = int.from_bytes(f[k + 2:k + 4], 'big')
  body = bytes(f[k + 4:k + 9]) + bytes([4]) + b''.join(bytes([c, 0x11, 0]) for c in (1, 2, 3, 4))
  return f[:k] + segment(0xC0, body) + f[k + 2 + n:]


@pytest.mark.parametrize('samp,hv', [(0x111111, (1, 1)), (0x211111, (2, 1)), (0x121111, (1, 2)),
                                     (0x221111, (2, 2)), (0x411111, (4, 1))])
def test_parse_sizes_and_sampling(samp, hv):
  f = J.encode(img(37, 58), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp, cv2.IMWRITE_JPEG_RST_INTERVAL, 3)
  i = jpeg_info(f)
  assert i['supported'] and i['reason'] == 0
  assert (i['height'], i['width'], i['coded_height'], i['coded_width']) == (37, 58, 37, 58)
  assert (i['components'], i['h_samp'], i['v_samp'], i['restart_interval']) == (3, hv[0], hv[1], 3)
  assert i['scan_offset'] == D.parse(f).scan


def test_parse_gray_and_orientation():
  g = jpeg_info(J.encode(img(c=1)))
  assert g['supported'] and g['components'] == 1 and (g['h_samp'], g['v_samp']) == (1, 1)
  base = J.encode(img(37, 58))
  for o in range(1, 9):
    i = jpeg_info(D.with_orientation(base, o, o % 2 == 1))
    assert i['orientation'] == o
    assert (i['height'], i['width']) == ((58, 37) if o >= 5 else (37, 58))
    assert (i['coded_height'], i['coded_width']) == (37, 58)


def reason(f):
  i = jpeg_info(f)
  assert not i['supported']
  return i['reason']


def test_refusal_reasons():
  f = J.encode(img())
  assert reason(J.encode(img(), cv2.IMWRITE_JPEG_PROGRESSIVE, 1)) == D.PROGRESSIVE
  assert reason(with_sof(f, marker=0xC9)) == D.ARITHMETIC
  assert reason(with_sof(f, marker=0xC3)) == D.LOSSLESS
  assert reason(with_sof(f, precision=12)) == D.PRECISION
  assert reason(four_components(f)) == D.COMPONENTS
  assert reason(J.component_ids(f, (1, 2, 3), jfif=False, adobe=0)) == D.COLOR_TRANSFORM
  assert reason(J.component_ids(f, (82, 71, 66), jfif=False)) == D.COLOR_TRANSFORM
  assert reason(J.bad_huffman(f, 'over')) == D.MALFORMED
  assert reason(J.bad_huffman(f, 'dc16')) == D.MALFORMED
  for cut in (3, 10, 100, D.parse(f).scan - 5):
    assert reason(f[:cut]) == D.MALFORMED
  for bad in (with_sof(f, marker=0xC2), four_components(f), with_sof(f, precision=12),
              J.component_ids(f, (82, 71, 66), jfif=False), J.bad_huffman(f, 'over'), f[:10]):
    with pytest.raises(D.Unsupported) as e:
      D.parse(bad)
    assert e.value.reason == reason(bad)
    assert jpeg_info(bad)['reason_text'] == D.REASONS[e.value.reason]


def test_handmade_files_parse():
  for name, f in J.handmade():
    i = jpeg_info(f)
    assert i['supported'], name
    assert (i['height'], i['width']) == D.parse(f).out_hw, name


def test_adobe_ycc_is_decoded():
  f = J.encode(img())
  g = f[:2] + segment(0xEE, b'Adobe' + bytes([0, 100, 0, 0, 0, 0, 1])) + f[2:]
  assert jpeg_info(g)['supported']
  assert np.array_equal(D.decode(g), J.imdecode(g))


def call(n=1, files=None, lengths=None, outs=FAKE, pitches=None, staging=FAKE, sb=1 << 40,
         scratch=FAKE, cb=1 << 40, status=FAKE):
  lib = _lib.load()
  f = J.encode(img())
  files = [f] * max(n, 1) if files is None else files
  bufs = [C.create_string_buffer(x, len(x)) for x in files]
  ptrs = (C.c_void_p * len(files))(*[C.addressof(b) for b in bufs])
  lens = (C.c_int64 * len(files))(*([len(x) for x in files] if lengths is None else lengths))
  op = None if outs is None else (C.c_void_p * len(files))(*[outs] * len(files))
  pp = (C.c_int64 * len(files))(*([3 * 24] * len(files) if pitches is None else pitches))
  return lib.sqdet_decode_jpeg(n, ptrs, lens, op, pp, staging, sb, scratch, cb, status, None)


def refused(rc, *words, code=-1):
  assert rc == code
  msg = _lib.load().sqdet_last_error()
  assert all(w.encode() in msg for w in words), msg


def test_decode_refusals():
  refused(call(outs=None), 'null')
  refused(call(staging=None), 'null')
  refused(call(scratch=None), 'null')
  refused(call(status=None), 'null')
  refused(call(n=0), 'n must be in [1, 128]')
  refused(call(n=129, files=[J.encode(img())] * 129), 'n must be in [1, 128]')
  refused(call(lengths=[3]), 'file 0', 'length')
  prog = J.encode(img(), cv2.IMWRITE_JPEG_PROGRESSIVE, 1)
  refused(call(n=2, files=[J.encode(img()), prog]), 'file 1', 'progressive', code=-3)
  refused(call(scratch=FAKE + 8), '256-byte aligned')
  refused(call(status=FAKE + 2), '4-byte aligned')
  refused(call(sb=10), 'staging_bytes')
  refused(call(cb=10), 'scratch_bytes')
  refused(call(), 'staging_pinned')          # a fake staging pointer is not pinned host memory


def test_sizes():
  lib = _lib.load()
  f = J.encode(img())
  buf = C.create_string_buffer(f, len(f))
  ptrs = (C.c_void_p * 1)(C.addressof(buf))
  lens = (C.c_int64 * 1)(len(f))
  sb = lib.sqdet_jpeg_decode_staging_bytes(1, ptrs, lens)
  cb = lib.sqdet_jpeg_decode_scratch_bytes(1, ptrs, lens)
  assert len(f) < sb < len(f) + 16384 and cb > sb
  assert lib.sqdet_jpeg_decode_staging_bytes(0, ptrs, lens) == -1
  bad = (C.c_int64 * 1)(2)
  assert lib.sqdet_jpeg_decode_scratch_bytes(1, ptrs, bad) == -1
  assert lib.sqdet_jpeg_decode_set_subsequence_bits(33) == -1
  assert lib.sqdet_jpeg_decode_set_subsequence_bits(0) == 0
