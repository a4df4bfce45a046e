"""sqdet_encode_jpeg and its size functions refuse bad arguments before any device work, so without
a GPU too, and give the sizes the encoder needs.  The refusals both encoders share are in
test_encode_abi."""
import ctypes as C

import numpy as np
import pytest

from oracle import jpeg as ojpeg
from squeezedet_b200 import _lib

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


def encode(n=1, h=16, w=16, quality=95):
  lib = _lib.load()
  hs, ws, _ = arrays(n, h, w)
  return lib.sqdet_encode_jpeg(n, FMT_BGR, host_planes(n), None, hs, ws, None, quality, FAKE, 1 << 20,
                               FAKE, FAKE, 1 << 40, None)


def refused(rc, *words):
  assert rc == -1
  msg = _lib.load().sqdet_last_error()
  assert all(w.encode() in msg for w in words), msg


def test_quality_and_side():
  """The refusals of sqdet_encode_jpeg's own: the quality, and sides past 65500.  The ones it shares
  with sqdet_encode_png are in test_encode_abi."""
  refused(encode(quality=0), 'quality')
  refused(encode(quality=101), 'quality')
  refused(encode(h=70000, w=8), '65500')


def test_max_bytes():
  lib = _lib.load()
  assert lib.sqdet_jpeg_max_bytes(0, 5) == -1
  assert lib.sqdet_jpeg_max_bytes(5, 65536) == -1
  for h, w in [(1, 1), (8, 8), (17, 23), (1080, 1920)]:
    blocks = -(-h // 16) * -(-w // 16) * 6
    header = len(ojpeg.header(h, w, 95))
    # every block's longest codes (a chroma DC of category 11, 63 AC codes of 16 + 10 bits), each
    # byte stuffed, plus the header and EOI
    assert lib.sqdet_jpeg_max_bytes(h, w) == header + 2 * -(-blocks * (22 + 63 * 26) // 8) + 2


def test_max_bytes_holds_the_largest_oracle_files():
  lib = _lib.load()
  rng = np.random.default_rng(0)
  for h, w in [(1, 1), (8, 8), (16, 16), (17, 23)]:
    y, x = np.mgrid[:h, :w]
    check = np.repeat((((y + x) % 2) * 255).astype(np.uint8)[..., None], 3, axis=2)
    for img in (check, rng.integers(0, 256, (h, w, 3), dtype=np.uint8)):
      assert len(ojpeg.encode(img, 100)) <= lib.sqdet_jpeg_max_bytes(h, w)


def test_scratch_bytes():
  lib = _lib.load()
  hs, ws, _ = arrays(2, 1080, 1920)
  one = lib.sqdet_jpeg_scratch_bytes(1, hs, ws, None)
  two = lib.sqdet_jpeg_scratch_bytes(2, hs, ws, None)
  blocks = 68 * 120 * 6
  # at least the coefficients and the worst-case bit stream of each frame
  assert one >= blocks * 64 * 2 + blocks * (22 + 63 * 26) // 8
  assert two >= 2 * one - 4096
  hs, ws, cr = arrays(1, 1080, 1920, [0, 0, 16, 16])
  assert lib.sqdet_jpeg_scratch_bytes(1, hs, ws, cr) < one
  # frames run 16 to a launch group and groups reuse the scratch
  hs, ws, _ = arrays(128, 64, 64)
  assert lib.sqdet_jpeg_scratch_bytes(128, hs, ws, None) == lib.sqdet_jpeg_scratch_bytes(16, hs, ws, None)
  assert lib.sqdet_jpeg_scratch_bytes(0, hs, ws, None) == -1
  assert lib.sqdet_jpeg_scratch_bytes(129, hs, ws, None) == -1
  assert lib.sqdet_jpeg_scratch_bytes(1, None, ws, None) == -1
  hs, ws, cr = arrays(1, 8, 8, [4, 0, 8, 8])
  assert lib.sqdet_jpeg_scratch_bytes(1, hs, ws, cr) == -1


def test_python_checks():
  from squeezedet_b200.jpeg import encode_jpeg_device, max_bytes
  with pytest.raises(ValueError):
    encode_jpeg_device([], 'bgr')
  with pytest.raises(ValueError):
    encode_jpeg_device([np.zeros((4, 4, 3), np.uint8)], 'yuyv')
  with pytest.raises(ValueError):
    encode_jpeg_device([np.zeros((4, 4, 3), np.uint8)], 'bgr', quality=0)
  with pytest.raises(ValueError):
    encode_jpeg_device([np.zeros((4, 4, 3), np.uint8)], 'bgr')      # not a CUDA tensor
  with pytest.raises(ValueError):
    max_bytes(0, 4)
