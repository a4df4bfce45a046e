"""sqdet_forward_frames_u8 refuses a null engine or null arrays before any device work, so without
a GPU too."""
import ctypes

from squeezedet_b200 import _lib


def test_forward_frames_u8_rejects_null_arguments():
  lib = _lib.load()
  buf = (ctypes.c_uint8 * 48)()
  ptrs = (ctypes.c_void_p * 1)(ctypes.addressof(buf))
  hs, ws = (ctypes.c_int32 * 1)(4), (ctypes.c_int32 * 1)(4)
  pitches = (ctypes.c_int64 * 1)(12)
  for args in [(None, 1, ptrs, hs, ws, pitches), (None, 1, ptrs, hs, ws, None),
               (None, 1, None, None, None, None)]:
    assert lib.sqdet_forward_frames_u8(*args, 0, 0, None) == -1
    assert b'null' in lib.sqdet_last_error()
