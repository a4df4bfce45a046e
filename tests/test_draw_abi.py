"""sqdet_draw_dets refuses null arrays, bad counts and a bad style before any device work, so
without a GPU too."""
import ctypes

from squeezedet_b200 import _lib

FMT_BGR, FMT_NV12 = 0, 5


def style(classes=3, names=(b'car', b'pedestrian', b'cyclist'), font_scale=0.3, null_colours=False):
  colours = (ctypes.c_uint8 * (3 * max(classes, 1)))()
  st = _lib.DrawStyle(classes, (ctypes.c_char_p * len(names))(*names),
                      None if null_colours else colours, 0.4, font_scale)
  st._keep = colours
  return st


def test_draw_dets_rejects_null_arguments():
  lib = _lib.load()
  buf = (ctypes.c_uint8 * 48)()
  planes = (ctypes.c_void_p * 3)(*[ctypes.addressof(buf)] * 3)
  hs, ws = (ctypes.c_int32 * 1)(4), (ctypes.c_int32 * 1)(4)
  fake = 1 << 40           # never dereferenced: the null check comes first
  st = style()
  for fmt in (FMT_BGR, FMT_NV12):
    for args in [(None, None, hs, ws, None, fake, fake, 8, ctypes.byref(st)),
                 (planes, None, None, ws, None, fake, fake, 8, ctypes.byref(st)),
                 (planes, None, hs, None, None, fake, fake, 8, ctypes.byref(st)),
                 (planes, None, hs, ws, None, None, fake, 8, ctypes.byref(st)),
                 (planes, None, hs, ws, None, fake, None, 8, ctypes.byref(st)),
                 (planes, None, hs, ws, None, fake, fake, 8, None),
                 (planes, None, hs, ws, None, fake, fake, 8, ctypes.byref(style(null_colours=True)))]:
      assert lib.sqdet_draw_dets(1, fmt, *args, None) == -1
      assert b'null' in lib.sqdet_last_error()


def test_draw_dets_rejects_bad_counts_and_style():
  """n, max_dets and the style are checked before the frames' memory."""
  lib = _lib.load()
  buf = (ctypes.c_uint8 * 48)()
  planes = (ctypes.c_void_p * 3)(*[ctypes.addressof(buf)] * 3)
  hs, ws = (ctypes.c_int32 * 1)(4), (ctypes.c_int32 * 1)(4)
  fake = 1 << 40

  def refused(n=1, fmt=FMT_BGR, max_dets=8, st=None):
    st = style() if st is None else st
    return lib.sqdet_draw_dets(n, fmt, planes, None, hs, ws, None, fake, fake, max_dets,
                               ctypes.byref(st), None), lib.sqdet_last_error()

  assert refused(fmt=7) == (-1, b'sqdet_draw_dets: unknown format')
  assert refused(n=0)[0] == -1 and b'n must be in [1, 128]' in refused(n=0)[1]
  assert refused(n=129)[0] == -1
  assert refused(max_dets=0) == (-1, b'sqdet_draw_dets: max_dets must be at least 1')
  assert refused(st=style(classes=0))[0] == -1
  assert refused(st=style(classes=65, names=(b'x',) * 65))[0] == -1
  for name in (b'x' * 32, b'a\tb', b'caf\xc3\xa9'):
    rc, msg = refused(st=style(names=(b'car', name, b'cyclist')))
    assert rc == -1 and b'class name 1' in msg
  for fs in (0.0, -1.0, float('nan'), float('inf'), 2000.0):
    rc, msg = refused(st=style(font_scale=fs))
    assert rc == -1 and b'font_scale' in msg
