"""sqdet_encode_png and its size functions refuse bad arguments before any device work, so without
a GPU too, and give the sizes the encoder needs.  The refusals both encoders share are in
test_encode_abi."""
import ctypes as C

import numpy as np
import pytest

from oracle import png as opng
from squeezedet_b200 import _lib
from squeezedet_b200 import png as spng

FMT_BGR = 0
FAKE = 1 << 40            # never dereferenced: the argument checks come first


def arrays(n=1, h=16, w=16, crops=None):
  hs, ws = (C.c_int32 * n)(*[h] * n), (C.c_int32 * n)(*[w] * n)
  cr = None if crops is None else (C.c_int32 * (4 * n))(*crops)
  return hs, ws, cr


def host_planes(n=1):
  buf = (C.c_uint8 * 4096)()
  p = (C.c_void_p * (3 * n))(*[C.addressof(buf)] * (3 * n))
  p._keep = buf
  return p


def encode(h=16, w=16, crops=None):
  lib = _lib.load()
  hs, ws, cr = arrays(1, h, w, crops)
  return lib.sqdet_encode_png(1, FMT_BGR, host_planes(), None, hs, ws, cr, FAKE, 1 << 20, FAKE, FAKE,
                              1 << 40, None)


def refused(rc, *words):
  assert rc == -1
  msg = _lib.load().sqdet_last_error()
  assert all(w.encode() in msg for w in words), msg


def test_symbols_declared():
  lib = _lib.load()
  for name in ('sqdet_png_max_bytes', 'sqdet_png_scratch_bytes', 'sqdet_encode_png'):
    assert name in _lib.SIGNATURES and getattr(lib, name)


def test_side_limits():
  """cv2.imencode writes up to 1000000 pixels wide and high and refuses beyond; so does the encoder,
  before any allocation, in C and in Python."""
  lib = _lib.load()
  assert lib.sqdet_png_max_bytes(1, 1000000) > 3000000
  assert lib.sqdet_png_max_bytes(1000000, 1) > 4000000
  for h, w in ((1, 1000001), (1000001, 1), (0, 5), (5, 0)):
    assert lib.sqdet_png_max_bytes(h, w) == -1
    with pytest.raises(ValueError, match='1000000'):
      spng.max_bytes(h, w)
  hs, ws, _ = arrays(1, 1, 1000001)
  assert lib.sqdet_png_scratch_bytes(1, hs, ws, None) == -1
  refused(encode(h=1, w=1000001), '1000000')
  # a crop within the limit of a frame beyond it is accepted up to the device checks
  refused(encode(h=1, w=1000001, crops=[1, 0, 1000000, 1]), 'not inside one device allocation')
  hs, ws, cr = arrays(1, 1, 1000001, [1, 0, 1000000, 1])
  assert lib.sqdet_png_scratch_bytes(1, hs, ws, cr) > 0


def test_scratch_is_64_bit():
  """The largest accepted sizes give scratch sizes past 2^32 without overflow."""
  lib = _lib.load()
  hs, ws, _ = arrays(2, 1000000, 1000000)
  sb = lib.sqdet_png_scratch_bytes(2, hs, ws, None)
  assert sb > 2 * 3 * 1000000 * 1000000 * 3
  assert lib.sqdet_png_max_bytes(1000000, 1000000) > 9 * 3 * 10 ** 12 // 8


@pytest.mark.parametrize('h,w', [(1, 1), (2, 3), (64, 64), (3, 1820), (120, 300)])
def test_max_bytes_holds_noise(h, w):
  """sqdet_png_max_bytes is above the largest file the oracle makes: noise, all stored blocks."""
  img = np.random.default_rng(h + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
  assert len(opng.encode(img)) <= spng.max_bytes(h, w)
