"""The partial-batch entry points (sqdet_forward_n, sqdet_submit_frames_n) check their arguments
before touching a device, so they run without a GPU."""
import ctypes

from squeezedet_b200 import _lib

ERR_INVALID_ARG = -1


def test_partial_batch_calls_reject_null_engine_without_device():
  lib = _lib.load()
  one = ctypes.c_int32(1)
  frames = (ctypes.c_void_p * 1)(None)
  for n in (0, 1, 2):
    assert lib.sqdet_forward_n(None, None, n, None) == ERR_INVALID_ARG
    assert b'null' in lib.sqdet_last_error()
    assert lib.sqdet_submit_frames_n(None, n, frames, ctypes.byref(one), ctypes.byref(one), 1, 1,
                                     None, None) == ERR_INVALID_ARG
    assert b'null' in lib.sqdet_last_error()
