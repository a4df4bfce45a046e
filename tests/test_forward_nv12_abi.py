"""sqdet_forward_frames_nv12 refuses a null engine or null arrays before any device work, so without
a GPU too."""
import ctypes

from squeezedet_b200 import _lib


def test_forward_frames_nv12_rejects_null_arguments():
  lib = _lib.load()
  buf = (ctypes.c_uint8 * 24)()
  planes = (ctypes.c_void_p * 1)(ctypes.addressof(buf))
  hs, ws = (ctypes.c_int32 * 1)(4), (ctypes.c_int32 * 1)(4)
  pitches = (ctypes.c_int64 * 1)(4)
  crops = (ctypes.c_int32 * 4)(0, 0, 4, 4)
  for args in [(None, 1, planes, pitches, planes, pitches, hs, ws, crops),
               (None, 1, planes, None, planes, None, hs, ws, None),
               (None, 1, None, None, None, None, None, None, None)]:
    assert lib.sqdet_forward_frames_nv12(*args, 0, 0, None) == -1
    assert b'null' in lib.sqdet_last_error()
