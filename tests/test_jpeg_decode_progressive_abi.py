"""sqdet_jpeg_parse_progressive reports what oracle.jpeg_decode_progressive reports, the progressive
size functions behave as documented, and sqdet_decode_jpeg_progressive refuses bad arguments before
any device work, so without a GPU too.  The plain entry points keep refusing progressive files."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import jpeg_decode as D
from oracle import jpeg_decode_progressive as P
from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import jpeg_info

import jpeg_corpus as J
import progressive_writer as W

FAKE = 1 << 40            # never dereferenced: the argument checks come first
PROG = cv2.IMWRITE_JPEG_PROGRESSIVE


def img(h=20, w=24):
  return J.content('smooth', h, w, 3, np.random.default_rng(0))


def files():
  rng = np.random.default_rng(1)
  out = [J.encode(J.content('noise', 37, 58, 3, rng), PROG, 1, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, s,
                  cv2.IMWRITE_JPEG_RST_INTERVAL, r) for s, r in zip(J.SAMPLINGS, (0, 1, 3, 0, 2))]
  out.append(D.with_orientation(J.encode(img(37, 58), PROG, 1), 6))
  out.append(J.encode(J.content('smooth', 33, 47, 1, rng)[..., 0], PROG, 1))
  f = J.encode(img(37, 58), cv2.IMWRITE_JPEG_QUALITY, 90)
  for d in (W.COMPLETE, W.UNSMOOTHED, W.SMOOTHED, W.BAD, W.BOGUS):
    out += [W.write(f, s) for s in d.values()]
  out += [f, J.encode(img(), PROG, 1)[:200], J.bad_huffman(f, 'over')]
  k = f.index(b'\xff\xc0')
  for marker in (0xC6, 0xCA, 0xCE):
    out.append(f[:k + 1] + bytes([marker]) + f[k + 2:])
  return out


def test_parse_matches_oracle():
  for f in files():
    i = jpeg_info(f, progressive=True)
    try:
      info, scans = P.parse(f)
      want = 0
    except P.Unsupported as e:
      want = e.reason
    assert i['reason'] == want and i['supported'] == (want == 0), (i['reason_text'], want)
    if want:
      assert i['reason_text'] == P.REASONS[want]
      continue
    assert i['scan_offset'] == (info.scan if scans is None else scans[0].start)
    assert (i['height'], i['width']) == info.out_hw
    assert i['components'] == len(info.comps)


def test_plain_entry_points_unchanged():
  f = J.encode(img(), PROG, 1)
  assert jpeg_info(f)['reason'] == D.PROGRESSIVE
  assert jpeg_info(f, progressive=True)['supported']


def sizes(fs, kind='_progressive'):
  lib = _lib.load()
  bufs = [C.create_string_buffer(x, len(x)) for x in fs]
  ptrs = (C.c_void_p * len(fs))(*[C.addressof(b) for b in bufs])
  lens = (C.c_int64 * len(fs))(*[len(x) for x in fs])
  return (getattr(lib, 'sqdet_jpeg_decode_staging_bytes' + kind)(len(fs), ptrs, lens),
          getattr(lib, 'sqdet_jpeg_decode_scratch_bytes' + kind)(len(fs), ptrs, lens))


def test_sizes():
  p = J.encode(img(), PROG, 1)
  b = J.encode(img())
  sb, cb = sizes([p])
  assert len(p) < sb < len(p) + 65536 and cb > sb
  bs, bc = sizes([b], '')
  ms, mc = sizes([b, p])
  assert ms >= bs + sb - 4096 and mc > bc and mc > cb
  assert sizes([b] * 3) == sizes([b] * 3, '')
  assert sizes([W.write(b, W.BAD['Al 14'])]) == (-1, -1)
  assert sizes([p] * 129) == (-1, -1)


def call(n=1, fs=None, lengths=None, outs=FAKE, pitches=None, staging=FAKE, sb=1 << 40,
         scratch=FAKE, cb=1 << 40, status=FAKE):
  lib = _lib.load()
  fs = [J.encode(img(), PROG, 1)] * max(n, 1) if fs is None else fs
  bufs = [C.create_string_buffer(x, len(x)) for x in fs]
  ptrs = (C.c_void_p * len(fs))(*[C.addressof(b) for b in bufs])
  lens = (C.c_int64 * len(fs))(*([len(x) for x in fs] if lengths is None else lengths))
  op = None if outs is None else (C.c_void_p * len(fs))(*[outs] * len(fs))
  pp = (C.c_int64 * len(fs))(*([3 * 24] * len(fs) if pitches is None else pitches))
  return lib.sqdet_decode_jpeg_progressive(n, ptrs, lens, op, pp, staging, sb, scratch, cb, status, None)


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
  refused(call(n=129, fs=[J.encode(img(), PROG, 1)] * 129), 'n must be in [1, 128]')
  refused(call(lengths=[3]), 'file 0', 'length')
  bad = W.write(J.encode(img()), W.BOGUS['AC before DC'])
  refused(call(n=2, fs=[J.encode(img()), bad]), 'file 1', 'scan script libjpeg warns on', code=-3)
  refused(call(scratch=FAKE + 8), '256-byte aligned')
  refused(call(status=FAKE + 2), '4-byte aligned')
  refused(call(sb=10), 'staging_bytes', 'sqdet_jpeg_decode_staging_bytes_progressive')
  refused(call(cb=10), 'scratch_bytes', 'sqdet_jpeg_decode_scratch_bytes_progressive')
  refused(call(), 'staging_pinned')
  refused(call(pitches=[3]), 'staging_pinned')


def test_parse_bad_arguments():
  lib = _lib.load()
  info = _lib.JpegInfo()
  assert lib.sqdet_jpeg_parse_progressive(None, 4, C.byref(info)) == -1
  assert lib.sqdet_jpeg_parse_progressive(b'\xff\xd8\xff\xd9', -1, C.byref(info)) == -1


def test_trailing_markers_parse():
  """RSTn markers after a scan's last interval are skipped, as libjpeg skips them."""
  f = J.encode(img(32, 48), PROG, 1)
  for index, count in ((0, 1), (3, 2), (9, 9)):
    g = W.with_trailing_rst(f, index, count)
    assert jpeg_info(g, progressive=True)['supported']
    assert np.array_equal(P.decode(g), J.imdecode(g))
    sb, _ = sizes([g])
    assert 0 < sb < 8 * len(g) + 6144 * 10


def test_staging_follows_the_file_not_its_dri():
  """A DRI asks for intervals the markers do not delimit: the staging stays bounded by the file's
  bytes, and the scans are corrupt (the oracle agrees)."""
  gray = J.encode(J.content('smooth', 4096, 4096, 1, np.random.default_rng(2))[..., 0], PROG, 1)
  for g in (gray, W.with_dri(gray, 1), W.with_dri(gray, 7)):
    sb, cb = sizes([g])
    assert 0 < sb < 8 * len(g) + 6144 * 6, (len(g), sb)
    assert cb > 4096 * 4096
  small = W.with_dri(J.encode(img(32, 48), PROG, 1), 1)
  assert jpeg_info(small, progressive=True)['supported']
  with pytest.raises(D.CorruptData):
    P.decode(small)


def test_scans_past_the_cap_are_checked():
  f = J.encode(img(37, 58), cv2.IMWRITE_JPEG_QUALITY, 90)
  dc = [((0, 1, 2), 0, 0, 0, 13)] + [((0, 1, 2), 0, 0, a + 1, a) for a in range(12, -1, -1)]
  ac = [((c,), k, k, 0, 1) for c in (0, 1, 2) for k in range(1, 64)] + \
       [((c,), k, k, 1, 0) for c in (0, 1, 2) for k in range(1, 64)]
  over = W.write(f, dc + ac)
  assert jpeg_info(over, progressive=True)['reason'] == P.TOO_MANY_SCANS
  bad = W.write(f, dc + ac + [((0,), 1, 63, 0, 14)])
  assert jpeg_info(bad, progressive=True)['reason'] == P.BAD_PROGRESSION == reason_of(bad)
  assert J.imdecode(bad) is None
  bogus = W.write(f, dc + ac + [((0,), 1, 63, 3, 2)])
  assert jpeg_info(bogus, progressive=True)['reason'] == P.TOO_MANY_SCANS == reason_of(bogus)


def reason_of(g):
  with pytest.raises(P.Unsupported) as e:
    P.parse(g)
  return e.value.reason
