"""sqdet_encode_jpeg_params and its size functions refuse bad parameters before any device work (so
without a GPU too), and their bounds grow with the sampling, optimized tables and restart
intervals as the worst case needs."""
import ctypes as C

import pytest

from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import SAMPLINGS, jpeg_params, max_bytes

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
  return lib.sqdet_encode_jpeg_params(1, 0, planes, None, hs, ws, None, p, FAKE, 1 << 20, FAKE, FAKE,
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
  refused(encode(C.byref(p)), 'sqdet_encode_jpeg', word)
  assert lib.sqdet_jpeg_max_bytes_params(16, 16, C.byref(p)) == -1
  hs, ws = sizes()
  assert lib.sqdet_jpeg_scratch_bytes_params(1, hs, ws, None, C.byref(p)) == -1


def test_null_params():
  lib = _lib.load()
  refused(encode(None), 'null')
  assert lib.sqdet_jpeg_max_bytes_params(16, 16, None) == -1
  hs, ws = sizes()
  assert lib.sqdet_jpeg_scratch_bytes_params(1, hs, ws, None, None) == -1


def test_refused_sizes_give_minus_one():
  lib = _lib.load()
  p = params(optimize=1, restart_interval=3, sampling=0x111111)
  for h, w in ((0, 16), (16, 0), (65501, 16), (16, 65501)):
    assert lib.sqdet_jpeg_max_bytes_params(h, w, C.byref(p)) == -1
    hs, ws = sizes(1, h, w)
    assert lib.sqdet_jpeg_scratch_bytes_params(1, hs, ws, None, C.byref(p)) == -1
  hs, ws = sizes(129)
  assert lib.sqdet_jpeg_scratch_bytes_params(129, hs, ws, None, C.byref(p)) == -1


def test_defaults_are_the_old_functions():
  lib = _lib.load()
  for h, w in ((1, 1), (17, 23), (1080, 1920), (65500, 65500)):
    for q in (1, 95, 100):
      p = params(quality=q)
      assert lib.sqdet_jpeg_max_bytes_params(h, w, C.byref(p)) == lib.sqdet_jpeg_max_bytes(h, w)
      hs, ws = sizes(3, h, w)
      assert lib.sqdet_jpeg_scratch_bytes_params(3, hs, ws, None, C.byref(p)) == \
          lib.sqdet_jpeg_scratch_bytes(3, hs, ws, None)
  # quality does not change the bounds; luma and chroma quality do only through 4:4:4
  assert max_bytes(100, 100, quality=1) == max_bytes(100, 100)
  assert max_bytes(100, 100, luma_quality=50, chroma_quality=50) == max_bytes(100, 100)
  assert max_bytes(100, 100, luma_quality=50, chroma_quality=60) == max_bytes(100, 100, sampling='444')


def blocks(h, w, sampling):
  hs, vs = {'411': (4, 1), '420': (2, 2), '422': (2, 1), '440': (1, 2), '444': (1, 1)}[sampling]
  mcus = -(-h // (8 * vs)) * -(-w // (8 * hs))
  return mcus, mcus * (hs * vs + 2)


@pytest.mark.parametrize('sampling', list(SAMPLINGS))
def test_bounds_arithmetic(sampling):
  """header + every byte stuffed + RSTn between intervals + EOI, from the longest block codes."""
  for h, w in ((1, 1), (17, 23), (375, 1242), (65500, 65500)):
    mcus, nb = blocks(h, w, sampling)
    for optimize in (False, True):
      for r in (0, 1, 7, 65535):
        bits = (27 if optimize else 22) + 63 * 26
        ints = -(-mcus // r) if r else 1
        data = (nb * bits + 7) // 8 + (ints if r else 0)
        want = 623 + (6 if r else 0) + 2 * data + 2 * (ints - 1) + 2
        assert max_bytes(h, w, sampling=sampling, optimize=optimize, restart_interval=r) == want


def test_scratch_grows_with_the_settings():
  lib = _lib.load()
  hs, ws = sizes(2, 1080, 1920)
  base = lib.sqdet_jpeg_scratch_bytes_params(2, hs, ws, None, C.byref(params()))
  for kw in (dict(sampling=0x111111), dict(optimize=1), dict(restart_interval=1)):
    assert lib.sqdet_jpeg_scratch_bytes_params(2, hs, ws, None, C.byref(params(**kw))) > base


def test_python_checks_mirror_the_abi():
  for kw in (dict(quality=0), dict(luma_quality=101), dict(chroma_quality=0), dict(sampling='421'),
             dict(restart_interval=-1), dict(restart_interval=65536)):
    with pytest.raises(ValueError):
      jpeg_params(**kw)
  p = jpeg_params(quality=80, sampling='444', optimize=True, restart_interval=9, luma_quality=70)
  assert (p.quality, p.luma_quality, p.chroma_quality, p.sampling, p.optimize, p.restart_interval) == \
      (80, 70, -1, 0x111111, 1, 9)
