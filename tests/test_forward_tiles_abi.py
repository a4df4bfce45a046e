"""sqdet_forward_tiles, sqdet_merge_tiles and sqdet_tile_results_dev refuse a null engine or null
arrays before any device work, so without a GPU too."""
import ctypes

from squeezedet_b200 import _lib

FMT_BGR, FMT_NV12 = 0, 5


def test_forward_tiles_rejects_null_arguments():
  lib = _lib.load()
  buf = (ctypes.c_uint8 * 48)()
  planes = (ctypes.c_void_p * 3)(*[ctypes.addressof(buf)] * 3)
  pitches = (ctypes.c_int64 * 3)(12, 4, 0)
  hs, ws = (ctypes.c_int32 * 1)(4), (ctypes.c_int32 * 1)(4)
  tiles = (ctypes.c_int32 * 5)(0, 0, 0, 4, 4)
  for fmt in (FMT_BGR, FMT_NV12):
    for args in [(None, 1, fmt, planes, pitches, hs, ws, 1, tiles),
                 (None, 1, fmt, planes, None, hs, ws, 1, None),
                 (None, 1, fmt, None, None, None, None, 1, None)]:
      assert lib.sqdet_forward_tiles(*args, 0, None) == -1
      assert b'null' in lib.sqdet_last_error()


def test_merge_tiles_rejects_null_arguments():
  lib = _lib.load()
  frames = (ctypes.c_int32 * 2)(0, 0)
  xy = (ctypes.c_int32 * 4)(0, 0, 100, 0)
  fake = 1 << 40           # never dereferenced: the null check comes first
  for args in [(None, fake, fake, 16, 2, frames, xy), (fake, fake, fake, 16, 2, None, xy),
               (fake, fake, fake, 16, 2, frames, None), (fake, None, None, 16, 2, frames, xy)]:
    assert lib.sqdet_merge_tiles(*args, 1, 3, 64, ctypes.c_float(0.005), ctypes.c_float(0.4),
                                 fake, fake, 64, None) == -1
    assert b'null' in lib.sqdet_last_error()
  assert lib.sqdet_merge_tiles(fake, fake, fake, 16, 2, frames, xy, 1, 3, 64, ctypes.c_float(0.005),
                               ctypes.c_float(0.4), None, fake, 64, None) == -1
  assert b'null' in lib.sqdet_last_error()


def test_tile_results_dev_rejects_null_engine():
  lib = _lib.load()
  p, c, md = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_int32()
  assert lib.sqdet_tile_results_dev(None, ctypes.byref(p), ctypes.byref(c), ctypes.byref(md)) == -1
  assert b'null' in lib.sqdet_last_error()
