"""sqdet_encode_jpeg_progressive and its size functions refuse what the _params functions refuse,
before any device work (so without a GPU too), and their bound is the documented worst case."""
import ctypes as C

import pytest

from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import SAMPLINGS, encode_jpeg_device, max_bytes

FAKE = 1 << 40            # never dereferenced: the argument checks come first


def params(**kw):
  p = dict(quality=95, luma_quality=-1, chroma_quality=-1, sampling=0x221111, optimize=0, restart_interval=0)
  p.update(kw)
  return _lib.JpegParams(*[p[k] for k, _ in _lib.JpegParams._fields_])


def sizes(n=1, h=16, w=16):
  return (C.c_int32 * n)(*[h] * n), (C.c_int32 * n)(*[w] * n)


def encode(p, h=16, w=16):
  lib = _lib.load()
  buf = (C.c_uint8 * 4096)()
  planes = (C.c_void_p * 3)(C.addressof(buf), None, None)
  hs, ws = sizes(1, h, w)
  return lib.sqdet_encode_jpeg_progressive(1, 0, planes, None, hs, ws, None, p, FAKE, 1 << 20, FAKE, FAKE,
                                           1 << 40, None)


def refused(rc, *words):
  assert rc == -1
  msg = _lib.load().sqdet_last_error()
  assert all(w.encode() in msg for w in words), msg


BAD = [(dict(quality=0), 'quality'), (dict(quality=101), 'quality'),
       (dict(luma_quality=0), 'luma_quality'), (dict(luma_quality=101), 'luma_quality'),
       (dict(chroma_quality=-2), 'chroma_quality'), (dict(chroma_quality=101), 'chroma_quality'),
       (dict(sampling=0x221112), 'sampling'), (dict(sampling=0), 'sampling'), (dict(sampling=0x441111), 'sampling'),
       (dict(optimize=2), 'optimize'), (dict(optimize=-1), 'optimize'),
       (dict(restart_interval=-1), 'restart_interval'), (dict(restart_interval=65536), 'restart_interval')]


@pytest.mark.parametrize('kw,word', BAD)
def test_refusals(kw, word):
  lib = _lib.load()
  p = params(**kw)
  refused(encode(C.byref(p)), 'sqdet_encode_jpeg_progressive', word)
  assert lib.sqdet_jpeg_max_bytes_progressive(16, 16, C.byref(p)) == -1
  hs, ws = sizes()
  assert lib.sqdet_jpeg_scratch_bytes_progressive(1, hs, ws, None, C.byref(p)) == -1


def test_null_params():
  lib = _lib.load()
  refused(encode(None), 'null')
  assert lib.sqdet_jpeg_max_bytes_progressive(16, 16, None) == -1
  hs, ws = sizes()
  assert lib.sqdet_jpeg_scratch_bytes_progressive(1, hs, ws, None, None) == -1


def test_refused_sizes_give_minus_one():
  lib = _lib.load()
  p = params(restart_interval=3, sampling=0x111111)
  for h, w in ((0, 16), (16, 0), (65501, 16), (16, 65501)):
    assert lib.sqdet_jpeg_max_bytes_progressive(h, w, C.byref(p)) == -1
    hs, ws = sizes(1, h, w)
    assert lib.sqdet_jpeg_scratch_bytes_progressive(1, hs, ws, None, C.byref(p)) == -1
    refused(encode(C.byref(p), h, w), 'sqdet_encode_jpeg_progressive')
  hs, ws = sizes(129)
  assert lib.sqdet_jpeg_scratch_bytes_progressive(129, hs, ws, None, C.byref(p)) == -1


# jpeg_simple_progression: (component: 3 for the interleaved DC scans, Ss, Se, Ah)
SCANS = [(3, 0, 0, 0), (0, 1, 5, 0), (2, 1, 63, 0), (1, 1, 63, 0), (0, 6, 63, 0), (0, 1, 63, 2),
         (3, 0, 0, 1), (2, 1, 63, 1), (1, 1, 63, 1), (0, 1, 63, 1)]


@pytest.mark.parametrize('sampling', list(SAMPLINGS))
def test_bounds_arithmetic(sampling):
  """Headers + every scan's longest units with a padding byte per interval, every byte stuffed, RSTn
  between a scan's intervals, EOI."""
  hs, vs = {'411': (4, 1), '420': (2, 2), '422': (2, 1), '440': (1, 2), '444': (1, 1)}[sampling]
  for h, w in ((1, 1), (17, 23), (375, 1242), (65500, 65500)):
    mcus = -(-h // (8 * vs)) * -(-w // (8 * hs))
    for r in (0, 1, 7, 65535):
      data = rst = 0
      for c, ss, se, ah in SCANS:
        units = mcus * (hs * vs + 2) if c == 3 else mcus if c else -(-h // 8) * -(-w // 8)
        bits = (1 if ah else 27) if ss == 0 else (17 if ah else 26) * (se - ss + 1) + 30
        span = r * ((hs * vs + 2) if c == 3 else 1)
        ints = -(-units // span) if r else 1
        data += (units * bits + 7) // 8 + ints
        rst += ints - 1
      headers = 177 + 10 * (21 + 256) + 2 * 14 + 8 * 10
      want = headers + (6 if r else 0) + 2 * data + 2 * rst + 2
      for optimize in (False, True):
        assert max_bytes(h, w, progressive=True, sampling=sampling, optimize=optimize, restart_interval=r) == want


def test_scratch_and_bound_exceed_baseline():
  lib = _lib.load()
  hs, ws = sizes(2, 1080, 1920)
  base = lib.sqdet_jpeg_scratch_bytes_params(2, hs, ws, None, C.byref(params(optimize=1)))
  assert lib.sqdet_jpeg_scratch_bytes_progressive(2, hs, ws, None, C.byref(params())) > base
  assert max_bytes(1080, 1920, progressive=True) > max_bytes(1080, 1920, optimize=True)


def test_python_checks_mirror_the_abi():
  """The keyword is checked as the ABI checks its parameters, before any device work."""
  for kw in (dict(quality=0), dict(luma_quality=101), dict(chroma_quality=0), dict(sampling='421'),
             dict(restart_interval=-1), dict(restart_interval=65536)):
    word = list(kw)[0]
    with pytest.raises(ValueError, match=word):
      max_bytes(16, 16, progressive=True, **kw)
    with pytest.raises(ValueError, match=word):
      encode_jpeg_device([None], 'bgr', progressive=True, **kw)
  lib = _lib.load()
  assert max_bytes(61, 97, progressive=True, restart_interval=9, sampling='444') == \
      lib.sqdet_jpeg_max_bytes_progressive(61, 97, C.byref(params(restart_interval=9, sampling=0x111111)))
  with pytest.raises(ValueError):
    max_bytes(0, 16, progressive=True)
