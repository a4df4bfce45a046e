"""The _options decode entry points on the host: with any_layout = 1, sqdet_jpeg_parse_options
accepts and refuses what oracle.jpeg_decode_layouts does, with its reasons and sizes; bad options
are argument errors; and any_layout = 0 is the _params functions file by file, reason by reason
and byte by byte.  No GPU: nothing here is decoded."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import jpeg_decode as D
from oracle import jpeg_decode_layouts as L
from oracle import jpeg_decode_reduced as R
from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import decode_jpeg_device, jpeg_info

import jpeg_corpus as J
import jpeg_layouts as JL

INVALID_ARG = -1
SCALES = (1, 2, 4, 8)


def arrays(fs):
  bufs = [C.create_string_buffer(f, len(f)) for f in fs]
  return bufs, (C.c_void_p * len(fs))(*[C.addressof(b) for b in bufs]), (C.c_int64 * len(fs))(*map(len, fs))


def options(progressive=1, scale=1, any_layout=1, reserved=None):
  o = _lib.JpegDecodeOptions(progressive, scale, any_layout)
  for k, v in enumerate(reserved or ()):
    o.reserved[k] = v
  return o


def parse_options(f, o):
  lib = _lib.load()
  info = _lib.JpegInfo()
  rc = lib.sqdet_jpeg_parse_options(C.create_string_buffer(f, len(f)), len(f), C.byref(o), C.byref(info))
  return rc, info


@pytest.mark.parametrize('s', SCALES)
def test_parse_matches_the_oracle(s):
  for name, f in JL.corpus() + JL.remainders([(2, 2), (1, 1), (1, 1), (2, 2)]):
    info, _, _ = L.parse(f, s, progressive=True)
    h, w = R.output_size(info, s)
    i = jpeg_info(f, progressive=True, reduce=s, any_layout=True)
    assert i['supported'] and i['reason'] == 0, (name, i['reason_text'])
    assert (i['height'], i['width']) == ((w, h) if info.orientation >= 5 else (h, w)), name
    assert (i['coded_height'], i['coded_width'], i['components']) == (info.height, info.width, len(info.comps))
    assert (i['h_samp'], i['v_samp']) == ((info.comps[0].h, info.comps[0].v) if len(info.comps) > 1 else (1, 1))
    _, ptrs, lens = arrays([f])
    o = options(1, s)
    assert _lib.load().sqdet_jpeg_decode_staging_bytes_options(1, ptrs, lens, C.byref(o)) > len(f)
    assert _lib.load().sqdet_jpeg_decode_scratch_bytes_options(1, ptrs, lens, C.byref(o)) > 0


def test_refusals_match_the_oracle():
  for name, f, reason in JL.refused():
    for prog in (0, 1):
      try:
        L.parse(f, 1, progressive=bool(prog))
        want = 0
      except D.Unsupported as e:
        want = e.reason
      rc, info = parse_options(f, options(prog))
      assert (rc != 0, info.reason) == (want != 0, want), (name, prog)
      if prog:
        assert want == reason
    i = jpeg_info(f, progressive=True, any_layout=True)
    assert i['reason_text'] == L.REASONS[reason]
    with pytest.raises(ValueError, match='nor does cv2.imdecode decode it'):
      decode_jpeg_device([f], 'cuda:0', progressive=True, any_layout=True)
  # the files cv2 decodes that the any-layout decoder still routes to it
  prog = J.encode(J.content('smooth', 20, 24, 3, np.random.default_rng(0)), cv2.IMWRITE_JPEG_PROGRESSIVE, 1)
  assert jpeg_info(prog, any_layout=True)['reason'] == D.PROGRESSIVE
  with pytest.raises(ValueError, match='decode it with cv2.imdecode'):
    decode_jpeg_device([prog], 'cuda:0', any_layout=True)


def test_bad_options_are_argument_errors():
  lib = _lib.load()
  f = JL.make(16, 16, [(1, 1)] * 4)
  _, ptrs, lens = arrays([f])
  out = _lib.JpegInfo()
  for o, what in ((options(1, 3), 'scale_denom'), (options(2, 1), 'progressive'),
                  (options(0, 1, 2), 'any_layout'), (options(0, 1, -1), 'any_layout'),
                  (options(0, 1, 1, (0, 0, 0, 0, 1)), 'reserved'), (options(1, 2, 0, (7,)), 'reserved')):
    assert lib.sqdet_jpeg_parse_options(ptrs[0], len(f), C.byref(o), C.byref(out)) == INVALID_ARG
    assert what.encode() in lib.sqdet_last_error() and b'sqdet_jpeg_parse_options' in lib.sqdet_last_error()
    assert lib.sqdet_jpeg_decode_staging_bytes_options(1, ptrs, lens, C.byref(o)) == -1
    assert lib.sqdet_jpeg_decode_scratch_bytes_options(1, ptrs, lens, C.byref(o)) == -1
    rc = lib.sqdet_decode_jpeg_options(1, ptrs, lens, C.byref(o), None, None, None, 0, None, 0, None, None)
    assert rc == INVALID_ARG and b'sqdet_decode_jpeg_options' in lib.sqdet_last_error()
  assert lib.sqdet_jpeg_parse_options(ptrs[0], len(f), None, C.byref(out)) == INVALID_ARG
  assert b'options is null' in lib.sqdet_last_error()


def _info(i):
  return {k: int(getattr(i, k)) for k, _ in _lib.JpegInfo._fields_}


@pytest.mark.parametrize('s', SCALES)
def test_any_layout_0_is_params(s):
  lib = _lib.load()
  fs = [f for _, f in J.corpus(seed=2, big=False)[::3]] + [r[1] for r in J.refused()] + \
      [f for _, f in JL.corpus()[::2]] + [f for _, f, _ in JL.refused()]
  for prog in (0, 1):
    p, o = _lib.JpegDecodeParams(prog, s), options(prog, s, 0)
    for f in fs:
      a, b = _lib.JpegInfo(), _lib.JpegInfo()
      buf = C.create_string_buffer(f, len(f))
      rc = lib.sqdet_jpeg_parse_params(buf, len(f), C.byref(p), C.byref(a))
      msg = lib.sqdet_last_error().replace(b'_params', b'')
      assert lib.sqdet_jpeg_parse_options(buf, len(f), C.byref(o), C.byref(b)) == rc
      assert _info(a) == _info(b)
      if rc:
        assert lib.sqdet_last_error().replace(b'_options', b'') == msg
    ok = [f for f in fs if jpeg_info(f, progressive=bool(prog), reduce=s)['supported']]
    for batch in (ok, ok[:1], ok[-5:], fs[:4]):
      _, ptrs, lens = arrays(batch)
      for fn in ('sqdet_jpeg_decode_staging_bytes', 'sqdet_jpeg_decode_scratch_bytes'):
        assert getattr(lib, fn + '_params')(len(batch), ptrs, lens, C.byref(p)) == \
            getattr(lib, fn + '_options')(len(batch), ptrs, lens, C.byref(o)), fn


def test_without_any_layout_the_old_refusals_stay():
  for name, f in JL.corpus():
    for s in SCALES:
      if not jpeg_info(f, progressive=True, reduce=s)['supported']:
        assert jpeg_info(f, progressive=True, reduce=s)['reason'] in (D.COMPONENTS, D.COLOR_TRANSFORM, D.SAMPLING)
        assert jpeg_info(f, progressive=True, reduce=s, any_layout=True)['supported'], name


def test_wide_progressive_frame_goes_to_cv2():
  f = JL.wide_progressive()
  i = jpeg_info(f, progressive=True, any_layout=True)
  assert not i['supported'] and i['reason'] == D.SAMPLING
  with pytest.raises(ValueError, match='decode it with cv2.imdecode'):
    decode_jpeg_device([f], 'cuda:0', progressive=True, any_layout=True)
  assert cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR) is not None
