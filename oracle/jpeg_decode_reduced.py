"""cv2.imdecode(buf, cv2.IMREAD_REDUCED_COLOR_s) for s = 2, 4, 8 of every file
oracle.jpeg_decode_progressive decodes, restated in numpy.

cv2 4.13 sets libjpeg-turbo 3.1's scale_num = 1, scale_denom = s and decodes straight to the
reduced size (jdmaster.c, jddctmgr.c, jdsample.c, jidctred.c):
  size      ceil(H / s) x ceil(W / s), then the EXIF orientation, as at full size
  plan      luma's IDCT is m = 8 / s; another component's starts at m and doubles while it is
            below 8 and both hmax * m % (h * size * 2) and vmax * m % (v * size * 2) are 0 (so
            4:2:0 chroma runs at 2m and is not upsampled; 4:2:2, 4:4:0 and 4:1:1 chroma stays at m)
  IDCTs     jpeg_idct_4x4 and jpeg_idct_2x2 as libjpeg-turbo's SSE2 code computes them, and the C
            jpeg_idct_1x1; 8 is oracle.jpeg_decode's islow
  upsample  fancy (oracle.jpeg_decode.upsample) only while m > 1, replication at 1/8
  limits    a coded side above 65500 is refused at every scale (libjpeg); cv2's 2^30 pixels apply
            to the reduced size; a file of more coded pixels whose reduced size fits is refused
            as CODED_TOO_LARGE (the device decoder does not size its coefficients; cv2 decodes it)
The entropy decoding is oracle.jpeg_decode's and oracle.jpeg_decode_progressive's, unchanged.
tests/test_oracle_jpeg_decode_reduced.py pins it bitwise against cv2."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle import jpeg_decode as D
from oracle import jpeg_decode_progressive as P
from oracle.jpeg_decode import (F0_765, F0_899, F1_847, F2_562, _s16, _w16, idct_islow, orient,
                                ycc_to_bgr)

REDUCTIONS = (1, 2, 4, 8)
# a coded size above MAX_PIXELS whose reduced size is not: cv2 decodes it at that scale, but its
# coefficients alone (2 bytes per coded sample) would be gigabytes, so the device decoder refuses it
CODED_TOO_LARGE = 15
CODED_TOO_LARGE_TEXT = 'more than 2^30 coded pixels, which cv2 decodes at this scale'
REASONS = P.REASONS + (CODED_TOO_LARGE_TEXT,)


class Unsupported(P.Unsupported):
  def __init__(self, reason):
    ValueError.__init__(self, REASONS[reason])
    self.reason = reason


def _frame_size(b):
  """(height, width) of the first SOF0/1/2 segment, walking the markers as the parsers do."""
  i = 2
  while i + 4 <= len(b):
    while i + 1 < len(b) and b[i] == 0xFF and b[i + 1] == 0xFF:
      i += 1
    m, n = b[i + 1], D._u16(b, i + 2)
    if m in (0xC0, 0xC1, 0xC2):
      return D._u16(b, i + 5), D._u16(b, i + 7)
    i += 2 + n
  raise ValueError('no frame header')


def parse(b, reduce=1, progressive=True):
  """oracle.jpeg_decode_progressive.parse (or, without progressive, oracle.jpeg_decode.parse) with
  the size limits of scale 1 / reduce -> (Info, scans or None), or Unsupported."""
  b = bytes(b)
  try:
    return P.parse(b) if progressive else (D.parse(b), None)
  except D.Unsupported as e:
    reason = e.reason
  if reason == D.TOO_LARGE:
    # raised at the frame header, after every check before it; the side limit holds at every scale
    hh, ww = _frame_size(b)
    if hh <= D.MAX_SIDE and ww <= D.MAX_SIDE and -(-hh // reduce) * -(-ww // reduce) <= D.MAX_PIXELS:
      reason = CODED_TOO_LARGE
  raise Unsupported(reason)



# jidctred constants, 13 fraction bits
F0_211, F0_509, F0_601, F0_720, F0_850 = 1730, 4176, 4926, 5906, 6967
F1_061, F1_272, F1_451, F2_172, F3_624 = 8697, 10426, 11893, 17799, 29692


def _dequantize(coef, q):
  """(JCOEF values as int32, their 16-bit products with q as the SIMD code's pmullw leaves them,
  both [..., 8, 8])."""
  c16 = coef.astype(np.int16).astype(np.int32)
  q16 = q.astype(np.uint16).view(np.int16).astype(np.int32)
  shape = coef.shape[:-1] + (8, 8)
  return c16.reshape(shape), _w16(c16 * q16).reshape(shape)


def _red4_pass(g, shift):
  """jpeg_idct_4x4's 1-D pass over inputs g(0..7) (input 4 unused), in 32-bit arithmetic that
  wraps as paddd does -> its four outputs, descaled by `shift`."""
  tmp0 = g(0) << 14
  tmp2 = g(2) * F1_847 - g(6) * F0_765
  t10, t12 = tmp0 + tmp2, tmp0 - tmp2
  z1, z2, z3, z4 = g(7), g(5), g(3), g(1)
  odd0 = z1 * -F0_211 + z2 * F1_451 + z3 * -F2_172 + z4 * F1_061
  odd2 = z1 * -F0_509 + z2 * -F0_601 + z3 * F0_899 + z4 * F2_562
  rnd = np.int32(1 << (shift - 1))
  return [(o + rnd) >> shift for o in (t10 + odd2, t12 + odd0, t12 - odd0, t10 - odd2)]


def idct_4x4(coef, q):
  """jpeg_idct_4x4 of quantized coefficients [..., 64] -> uint8 samples [..., 4, 4], as cv2's
  libjpeg-turbo runs it on x86-64 (jsimd_idct_4x4_sse2): dequantization by a 16-bit multiply; a
  block whose rows 1, 2, 3, 5, 6 and 7 are all zero takes its dequantized row 0 << 2 (16-bit) as
  the column pass's result, the others the column pass saturated to 16 bits; the row pass in 32
  bits, saturated to 8."""
  c, d = _dequantize(coef, q)
  ws = np.stack(_red4_pass(lambda k: d[..., k, :], 12), axis=-2)          # [..., 4, 8]
  ws = _s16(ws)
  dc_only = (c[..., [1, 2, 3, 5, 6, 7], :] == 0).all(axis=(-1, -2))
  ws_dc = np.broadcast_to(_w16(d[..., :1, :] << 2), ws.shape)
  ws = np.where(dc_only[..., None, None], ws_dc, ws).astype(np.int32)
  v = np.stack(_red4_pass(lambda k: ws[..., :, k], 19), axis=-1)           # [..., 4 rows, 4 cols]
  return (np.clip(v, -128, 127) + 128).astype(np.uint8)


def idct_2x2(coef, q):
  """jpeg_idct_2x2 -> uint8 samples [..., 2, 2], as jsimd_idct_2x2_sse2 computes it: no zero
  test; the column pass's column 0 kept in 32 bits and columns 1, 3, 5, 7 saturated to 16; the
  row pass's in0 << 15 wrapping in 32 bits; the output saturated to 8 bits."""
  _, d = _dequantize(coef, q)
  odd = lambda g: g(1) * F3_624 - g(3) * F1_272 + g(5) * F0_850 - g(7) * F0_720
  col = lambda k: d[..., k, :]
  t10, t0 = col(0) << 15, odd(col)
  rnd = np.int32(1 << 12)
  ws = np.stack([(t10 + t0 + rnd) >> 13, (t10 - t0 + rnd) >> 13], axis=-2)  # [..., 2, 8]
  ws[..., :, 1:] = _s16(ws[..., :, 1:])        # columns 2, 4, 6 are never read
  row = lambda k: ws[..., :, k]
  t10, t0 = row(0) << 15, odd(row)
  rnd = np.int32(1 << 19)
  v = np.stack([(t10 + t0 + rnd) >> 20, (t10 - t0 + rnd) >> 20], axis=-1)
  return (np.clip(v, -128, 127) + 128).astype(np.uint8)


# jidctred.c's range_limit[x & RANGE_MASK] for 8-bit samples: x + 128 clamped, with x taken
# modulo 1024 in [-512, 511]
_RANGE_1X1 = np.concatenate([np.arange(128, 256), np.full(384, 255), np.zeros(384),
                             np.arange(0, 128)]).astype(np.uint8)


def idct_1x1(coef, q):
  """jpeg_idct_1x1 (C; libjpeg-turbo has no SIMD one) -> uint8 [..., 1, 1]: the DC times its
  quantizer (both 16-bit signed, product exact), descaled by 3 and range-limited."""
  dc = coef[..., 0].astype(np.int16).astype(np.int64)
  q0 = np.int64(np.array(q[0], np.uint16).view(np.int16))
  return _RANGE_1X1[((dc * q0 + 4) >> 3) & 1023][..., None, None]


IDCTS = {8: idct_islow, 4: idct_4x4, 2: idct_2x2, 1: idct_1x1}


@dataclass
class CompPlan:
  size: int           # the component's scaled IDCT: an n x n block per 8 x 8 coefficients
  height: int         # its samples at that scale (libjpeg's downsampled_height / _width)
  width: int
  fh: int             # its upsampling to the output: factors, and whether fancy
  fv: int
  fancy: bool


def plan(info, reduce=1):
  """Per component, as jpeg_calc_output_dimensions and jinit_upsampler decide it at scale_denom =
  reduce: luma's IDCT is m = 8 / reduce; another component's starts at m and doubles while it is
  below 8 and both hmax * m % (h * size * 2) and vmax * m % (v * size * 2) are 0; it is then
  upsampled by hmax * m / (h * size) and vmax * m / (v * size), fancily only while m > 1."""
  m = 8 // reduce
  out = []
  for c in info.comps:
    n = m
    while n < 8 and (info.hmax * m) % (c.h * n * 2) == 0 and (info.vmax * m) % (c.v * n * 2) == 0:
      n *= 2
    out.append(CompPlan(n, -(-info.height * c.v * n // (info.vmax * 8)),
                        -(-info.width * c.h * n // (info.hmax * 8)),
                        info.hmax * m // (c.h * n), info.vmax * m // (c.v * n), m > 1))
  return out


def output_size(info, reduce=1):
  """(height, width) decoded at scale 1 / reduce, before the orientation."""
  return -(-info.height // reduce), -(-info.width // reduce)


def frame(info, grids, qts, reduce=1):
  """Per-component coefficient grids and quantization tables -> the oriented BGR frame at scale
  1 / reduce: each component's scaled IDCT, cropped to its samples, upsampled, converted."""
  H, W = output_size(info, reduce)
  pl = plan(info, reduce)
  planes = []
  for p, grid, q in zip(pl, grids, qts):
    px = IDCTS[p.size](grid, q)                                     # [bh, bw, n, n]
    bh, bw = grid.shape[:2]
    planes.append(px.transpose(0, 2, 1, 3).reshape(bh * p.size, bw * p.size)[:p.height, :p.width])
  if len(planes) == 1:
    bgr = np.repeat(planes[0][:H, :W, None], 3, axis=2)
  else:
    up = [upsample(x, p.fh, p.fv, H, W, p.fancy) for x, p in zip(planes[1:], pl[1:])]
    bgr = ycc_to_bgr(planes[0][:H, :W], *up)
  return np.ascontiguousarray(orient(bgr, info.orientation))




def upsample(c, fh, fv, H, W, fancy):
  """oracle.jpeg_decode.upsample with fancy upsampling on; replication with it off."""
  if fancy:
    return D.upsample(c, fh, fv, H, W)
  return np.repeat(np.repeat(c.astype(np.int32), fv, axis=0), fh, axis=1)[:H, :W]


def decode(b, reduce=1):
  """cv2.imdecode(b, cv2.IMREAD_REDUCED_COLOR_<reduce>) -> uint8 [H, W, 3] BGR of a sequential or
  progressive file; reduce=1 is oracle.jpeg_decode_progressive.decode (IMREAD_COLOR).
  Unsupported for files outside the supported set, CorruptData for bad entropy data."""
  if reduce not in REDUCTIONS:
    raise ValueError('reduce must be one of %s, got %r' % (REDUCTIONS, reduce))
  b = bytes(b)
  if reduce == 1:
    return P.decode(b)
  info, scans = parse(b, reduce)
  if scans is None:
    grids = D.decode_coefficients(b, info)
    qts = [info.qt[c.tq] for c in info.comps]
  else:
    grids = P.coefficients(b, info, scans)
    qts = [info.qt.get(ci, np.zeros(64, np.uint16)) for ci in range(len(info.comps))]
  return frame(info, grids, qts, reduce)
