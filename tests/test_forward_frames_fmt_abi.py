"""sqdet_forward_frames refuses a null engine, null arrays or an unknown format before any device
work, so without a GPU too."""
import ctypes

from squeezedet_b200 import _lib

FMT_BGR, FMT_I420 = 0, 6


def test_forward_frames_rejects_null_arguments():
  lib = _lib.load()
  buf = (ctypes.c_uint8 * 48)()
  planes = (ctypes.c_void_p * 3)(*[ctypes.addressof(buf)] * 3)
  hs, ws = (ctypes.c_int32 * 1)(4), (ctypes.c_int32 * 1)(4)
  pitches = (ctypes.c_int64 * 3)(12, 2, 2)
  crops = (ctypes.c_int32 * 4)(0, 0, 4, 4)
  for fmt in (FMT_BGR, FMT_I420):
    for args in [(None, 1, fmt, planes, pitches, hs, ws, crops),
                 (None, 1, fmt, planes, None, hs, ws, None),
                 (None, 1, fmt, None, None, None, None, None)]:
      assert lib.sqdet_forward_frames(*args, 0, 0, None) == -1
      assert b'null' in lib.sqdet_last_error()


def test_forward_frames_rejects_unknown_format():
  lib = _lib.load()
  for fmt in (-1, 7):
    assert lib.sqdet_forward_frames(None, 1, fmt, None, None, None, None, None, 0, 0, None) == -1
    assert b'format' in lib.sqdet_last_error()
