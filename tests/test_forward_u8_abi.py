"""sqdet_forward_u8 refuses a null engine before any device work, so without a GPU too."""
import ctypes

from squeezedet_b200 import _lib


def test_forward_u8_rejects_null_engine():
  lib = _lib.load()
  buf = (ctypes.c_uint8 * 16)()
  assert lib.sqdet_forward_u8(None, ctypes.addressof(buf), 1, None) == -1
  assert b'null' in lib.sqdet_last_error()
  assert lib.sqdet_forward_u8(None, None, 1, None) == -1
  assert b'null' in lib.sqdet_last_error()
