"""CPU restatement of the colour conversions in front of the generic device-frames path
(sqdet_forward_frames) — test infrastructure, like the rest of oracle/.

Each format is converted as the cv2.cvtColor code beside it does, and PINNED bitwise against the
installed cv2 (tests/test_oracle_pixfmt.py):

  bgr         packed B,G,R [h, w, 3]              (no conversion)
  rgb         packed R,G,B [h, w, 3]              COLOR_RGB2BGR
  bgra        packed B,G,R,A [h, w, 4]            COLOR_BGRA2BGR
  rgba        packed R,G,B,A [h, w, 4]            COLOR_RGBA2BGR
  rgb_planar  planes R, G, B, each [h, w]          COLOR_RGB2BGR of the stacked [h, w, 3]
  nv12        luma [h, w], U,V pairs [h/2, w]      COLOR_YUV2BGR_NV12
  i420        luma [h, w], U, V each [h/2, w/2]    COLOR_YUV2BGR_I420

The packed and planar formats are byte gathers; I420 is NV12 with its chroma interleaved."""
import numpy as np

from . import nv12

FORMATS = ('bgr', 'rgb', 'bgra', 'rgba', 'rgb_planar', 'nv12', 'i420')
# fmt -> (planes, channels of a packed frame, the B, G, R channel indices)
_PACKED = {'bgr': (3, (0, 1, 2)), 'rgb': (3, (2, 1, 0)), 'bgra': (4, (0, 1, 2)),
           'rgba': (4, (2, 1, 0))}


def to_bgr(fmt, planes):
  """The uint8 BGR [h, w, 3] frame of `planes`, a sequence of uint8 arrays laid out as `fmt`
  (one packed frame, three R, G, B planes, luma + chroma, or Y, U, V)."""
  planes = [np.asarray(p, np.uint8) for p in planes]
  if fmt in _PACKED:
    ch, order = _PACKED[fmt]
    (f,) = planes
    assert f.ndim == 3 and f.shape[2] == ch, (fmt, f.shape)
    return np.ascontiguousarray(f[:, :, list(order)])
  if fmt == 'rgb_planar':
    r, g, b = planes
    assert r.shape == g.shape == b.shape and r.ndim == 2, (r.shape, g.shape, b.shape)
    return np.stack([b, g, r], axis=-1)
  if fmt == 'nv12':
    luma, chroma = planes
    return nv12.nv12_to_bgr(luma, chroma)
  if fmt == 'i420':
    y, u, v = planes
    h, w = y.shape
    assert u.shape == v.shape == (h // 2, w // 2), (y.shape, u.shape, v.shape)
    return nv12.nv12_to_bgr(y, np.stack([u, v], axis=-1).reshape(h // 2, w))
  raise ValueError('unknown pixel format %r' % (fmt,))
