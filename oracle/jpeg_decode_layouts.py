"""cv2.imdecode(buf, IMREAD_COLOR or IMREAD_REDUCED_COLOR_s) of Huffman-coded 8-bit files of every
colour space and sampling libjpeg-turbo decodes, restated in numpy.

On top of the other decode oracles (their entropy decoding, IDCTs and reduced plan, unchanged),
with cv2 4.13's bundled libjpeg-turbo 3.1:
  colour    default_decompress_parms: 3 components are YCbCr after a JFIF APP0, else RGB for an
            Adobe APP14 transform 0 (YCbCr for any other), else RGB for ids 'R', 'G', 'B', else
            YCbCr; 4 components are YCCK for an Adobe transform other than 0, else CMYK
  sampling  factors 1..4; jinit_upsampler needs max_h / h and max_v / v integral, and
            per_scan_setup at most 10 blocks in an interleaved MCU (libjpeg rejects the others:
            BAD_SAMPLING, and cv2 returns None).  A progressive frame of more than 10 blocks per
            MCU without an interleaved scan that wide is SAMPLING: cv2 decodes it, the device
            decoder does not
  upsample  each component by (max_h * m / (h * n), max_v * m / (v * n)) from its planned IDCT n
            (oracle.jpeg_decode_reduced.plan, luma's m = 8 / s), as jinit_upsampler picks it:
            h2v1 and h2v2 fancy when fancy upsampling is on and the downsampled width is above 2,
            h1v2 fancy when it is on, replication otherwise (oracle.jpeg_decode.upsample)
  convert   YCbCr: ycc_rgb_convert; RGB: the planes as they are; CMYK: libjpeg's raw CMYK, YCCK:
            ycck_cmyk_convert (C, M, Y = 255 - the clamped YCbCr->RGB, K unchanged); then cv2's
            icvCvt_CMYK2BGR: B = K - ((255 - Y) * K >> 8), G from M, R from C
  orient    the EXIF orientation, as at every other layout
parse(b, reduce, progressive) accepts exactly what sqdet_jpeg_parse_options accepts with
any_layout = 1.  tests/test_oracle_jpeg_decode_layouts.py pins it bitwise against cv2."""
from __future__ import annotations

import numpy as np

from oracle import jpeg_decode as D
from oracle import jpeg_decode_progressive as P
from oracle import jpeg_decode_reduced as R

BAD_SAMPLING = 16
REASONS = R.REASONS + ('sampling libjpeg rejects',)
MAX_BLOCKS = 10                        # libjpeg's D_MAX_BLOCKS_IN_MCU
GRAY, YCC, RGB, CMYK, YCCK = 'gray', 'ycc', 'rgb', 'cmyk', 'ycck'


class Unsupported(R.Unsupported):
  def __init__(self, reason):
    ValueError.__init__(self, REASONS[reason])
    self.reason = reason


def _tables(m, body, qt, dc, ac):
  if m == 0xDB:
    j = 0
    while j < len(body):
      pq, tq = body[j] >> 4, body[j] & 15
      size = 128 if pq else 64
      if pq > 1 or tq > 3 or j + 1 + size > len(body):
        raise Unsupported(D.MALFORMED)
      raw = np.frombuffer(body[j + 1:j + 1 + size], '>u2' if pq else 'u1').astype(np.uint16)
      q = np.zeros(64, np.uint16)
      q[D.ZIGZAG] = raw
      qt[tq] = q
      j += 1 + size
  elif m == 0xC4:
    j = 0
    while j < len(body):
      if j + 17 > len(body):
        raise Unsupported(D.MALFORMED)
      tc, th = body[j] >> 4, body[j] & 15
      bits = list(body[j + 1:j + 17])
      cnt = sum(bits)
      if tc > 1 or th > 3 or cnt > 256 or j + 17 + cnt > len(body):
        raise Unsupported(D.MALFORMED)
      (ac if tc else dc)[th] = (bits, list(body[j + 17:j + 17 + cnt]))
      j += 17 + cnt


def parse(b, reduce=1, progressive=False):
  """Headers (and, for an SOF2 file with progressive, every scan) -> (Info, scans or None,
  colour space), or Unsupported with sqdet_jpeg_parse_options' reason.  Info.qt holds, for a
  progressive file, each component's latched table under its index."""
  b = bytes(b)
  if len(b) < 4 or b[0] != 0xFF or b[1] != 0xD8:
    raise Unsupported(D.MALFORMED)
  qt, dc, ac = {}, {}, {}
  restart, orientation, adobe = 0, 1, None
  frame = None
  saw_exif = jfif = False
  scans, latched, space = [], {}, None
  bogus = too_many = False
  bits = None
  i = 2
  while True:
    while i + 1 < len(b) and b[i] == 0xFF and b[i + 1] == 0xFF:
      i += 1
    if scans and (i >= len(b) or (i + 1 < len(b) and b[i] == 0xFF and b[i + 1] == 0xD9)):
      break                     # EOI, or no EOI: libjpeg ends the image there
    if i + 2 > len(b) or b[i] != 0xFF:
      raise Unsupported(D.MALFORMED)
    m = b[i + 1]
    i += 2
    if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
      raise Unsupported(D.MALFORMED)
    n = D._u16(b, i) if i + 2 <= len(b) else -1
    if n < 2 or i + n > len(b):
      raise Unsupported(D.MALFORMED)
    body = b[i + 2:i + n]
    i += n
    _tables(m, body, qt, dc, ac)
    if scans:
      if 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
        raise Unsupported(D.MALFORMED)
    elif (m == 0xC2 and not progressive) or m in (0xC5, 0xC6, 0xCA, 0xCE):
      raise Unsupported(D.PROGRESSIVE)
    elif m in (0xC9, 0xCB, 0xCD, 0xCF):
      raise Unsupported(D.ARITHMETIC)
    elif m in (0xC3, 0xC7):
      raise Unsupported(D.LOSSLESS)
    if m in (0xC0, 0xC1, 0xC2) and not scans:
      if frame is not None or len(body) < 6:
        raise Unsupported(D.MALFORMED)
      hh, ww, nc = D._u16(body, 1), D._u16(body, 3), body[5]
      if body[0] != 8:
        raise Unsupported(D.PRECISION)
      if len(body) != 6 + 3 * nc:
        raise Unsupported(D.MALFORMED)
      if nc not in (1, 3, 4):
        raise Unsupported(D.COMPONENTS)
      comps = [D.Component(body[6 + 3 * k], body[7 + 3 * k] >> 4, body[7 + 3 * k] & 15,
                           body[8 + 3 * k]) for k in range(nc)]
      if any(c.tq > 3 or not 1 <= c.h <= 4 or not 1 <= c.v <= 4 for c in comps):
        raise Unsupported(D.MALFORMED)
      if hh == 0 or ww == 0:
        raise Unsupported(D.SIZE)
      if hh > D.MAX_SIDE or ww > D.MAX_SIDE:
        raise Unsupported(D.TOO_LARGE)
      if hh * ww > D.MAX_PIXELS:
        raise Unsupported(D.TOO_LARGE if -(-hh // reduce) * -(-ww // reduce) > D.MAX_PIXELS
                          else R.CODED_TOO_LARGE)
      if nc > 1:
        hmax, vmax = max(c.h for c in comps), max(c.v for c in comps)
        if any(hmax % c.h or vmax % c.v for c in comps):
          raise Unsupported(BAD_SAMPLING)
        if m != 0xC2 and sum(c.h * c.v for c in comps) > MAX_BLOCKS:
          raise Unsupported(BAD_SAMPLING)
      frame = (hh, ww, comps, m == 0xC2)
      bits = [[-1] * 64 for _ in comps]
    elif m == 0xDD:
      if len(body) != 2:
        raise Unsupported(D.MALFORMED)
      restart = D._u16(body, 0)
    elif scans and 0xE0 <= m <= 0xEF:
      pass                      # APPn after the first scan: read by neither libjpeg nor cv2
    elif m == 0xE1 and not saw_exif and body[:6] == b'Exif\x00\x00':
      saw_exif = True
      orientation = D.exif_orientation(body)
    elif m == 0xE0 and len(body) >= 14 and body[:5] == b'JFIF\x00':
      jfif = True
    elif m == 0xEE and len(body) >= 12 and body[:5] == b'Adobe':
      adobe = body[11]
    elif m == 0xDA:
      if frame is None or len(body) < 1:
        raise Unsupported(D.MALFORMED)
      hh, ww, comps, sof2 = frame
      ns = body[0]
      if not scans:
        ids = [c.cid for c in comps]
        if len(comps) == 1:
          space = GRAY
        elif len(comps) == 4:
          space = YCCK if adobe else CMYK
        elif not jfif and (adobe == 0 if adobe is not None else ids == [82, 71, 66]):
          space = RGB
        else:
          space = YCC
      if not sof2:                     # the one scan of a sequential file
        if len(body) != 4 + 2 * ns:
          raise Unsupported(D.MALFORMED)
        if ns != len(comps) or [body[1 + 2 * k] for k in range(ns)] != [c.cid for c in comps]:
          raise Unsupported(D.SAMPLING)
        for k, c in enumerate(comps):
          c.td, c.ta = body[2 + 2 * k] >> 4, body[2 + 2 * k] & 15
          if c.td > 3 or c.ta > 3 or c.td not in dc or c.ta not in ac or c.tq not in qt:
            raise Unsupported(D.MALFORMED)
          if not D.huff_ok(*dc[c.td], True) or not D.huff_ok(*ac[c.ta], False):
            raise Unsupported(D.MALFORMED)
        if body[1 + 2 * ns:4 + 2 * ns] != b'\x00\x3f\x00':
          raise Unsupported(D.MALFORMED)
        info = D.Info(hh, ww, comps, qt, dc, ac, restart, orientation, i)
        info.hmax, info.vmax = max(c.h for c in comps), max(c.v for c in comps)
        return info, None, space
      if len(body) != 4 + 2 * ns or not 1 <= ns <= 4:
        raise Unsupported(D.MALFORMED)
      idx = [next((ci for ci, c in enumerate(comps) if c.cid == body[1 + 2 * k]), None)
             for k in range(ns)]
      if None in idx:
        raise Unsupported(D.MALFORMED)
      if any(y <= x for x, y in zip(idx, idx[1:])):
        raise Unsupported(D.SAMPLING)
      if ns > 1 and sum(comps[ci].h * comps[ci].v for ci in idx) > MAX_BLOCKS:
        raise Unsupported(BAD_SAMPLING)
      ss, se, ah, al = body[1 + 2 * ns], body[2 + 2 * ns], body[3 + 2 * ns] >> 4, body[3 + 2 * ns] & 15
      for ci in idx:                   # latch_quant_tables
        if ci not in latched:
          if comps[ci].tq not in qt:
            raise Unsupported(D.MALFORMED)
          latched[ci] = qt[comps[ci].tq].copy()
      dc_band = ss == 0
      bad = (se != 0) if dc_band else (ss > se or se > 63 or ns != 1)
      if (ah != 0 and al != ah - 1) or al > 13 or bad:
        raise Unsupported(P.BAD_PROGRESSION)
      for ci in idx:
        cb = bits[ci]
        if not dc_band and cb[0] < 0:
          bogus = True
        for k in range(ss, se + 1):
          if ah != max(cb[k], 0) or (ah == 0 and cb[k] >= 0):
            bogus = True
          cb[k] = al
      tables = []
      for k, ci in enumerate(idx):
        td, ta = body[2 + 2 * k] >> 4, body[2 + 2 * k] & 15
        if dc_band and ah == 0:
          if td > 3 or td not in dc or not D.huff_ok(*dc[td], True):
            raise Unsupported(D.MALFORMED)
          tables.append(dc[td])
        elif not dc_band:
          if ta > 3 or ta not in ac or not D.huff_ok(*ac[ta], False):
            raise Unsupported(D.MALFORMED)
          tables.append(ac[ta])
        else:
          tables.append(None)
      end = P._data_end(b, i)
      if len(scans) == P.MAX_SCANS:
        too_many = True
      else:
        scans.append(P.Scan(idx, ss, se, ah, al, tables, restart, i, end))
      i = end
  if too_many:
    raise Unsupported(P.TOO_MANY_SCANS)
  if bogus:
    raise Unsupported(P.BOGUS_PROGRESSION)
  hh, ww, comps, _ = frame
  if P.smoothed(comps, latched, bits):
    raise Unsupported(P.SMOOTHED)
  if len(comps) > 1 and sum(c.h * c.v for c in comps) > MAX_BLOCKS:
    raise Unsupported(D.SAMPLING)      # cv2 decodes it; the device decoder's MCUs hold 10 blocks
  info = D.Info(hh, ww, comps, latched, dc, ac, 0, orientation, scans[0].start)
  info.hmax, info.vmax = max(c.h for c in comps), max(c.v for c in comps)
  return info, scans, space


def to_bgr(space, planes):
  """Upsampled planes (int arrays [H, W]) of a colour space -> uint8 [H, W, 3] BGR, as cv2 gets
  it from libjpeg."""
  if space == GRAY:
    return np.repeat(planes[0][..., None], 3, axis=2).astype(np.uint8)
  if space == RGB:
    return np.stack([planes[2], planes[1], planes[0]], axis=-1).astype(np.uint8)
  if space == YCC:
    return D.ycc_to_bgr(*planes)
  if space == YCCK:
    bgr = D.ycc_to_bgr(*planes[:3]).astype(np.int32)
    c, m, y = 255 - bgr[..., 2], 255 - bgr[..., 1], 255 - bgr[..., 0]     # ycck_cmyk_convert
  else:
    c, m, y = (p.astype(np.int32) for p in planes[:3])
  k = planes[3].astype(np.int32)
  return np.stack([k - ((255 - y) * k >> 8), k - ((255 - m) * k >> 8), k - ((255 - c) * k >> 8)],
                  axis=-1).astype(np.uint8)


def decode(b, reduce=1, progressive=False):
  """cv2.imdecode(b, IMREAD_COLOR) (reduce 1) or IMREAD_REDUCED_COLOR_<reduce> -> uint8 [H, W, 3]
  BGR.  Unsupported for files outside the supported set, CorruptData for bad entropy data."""
  if reduce not in R.REDUCTIONS:
    raise ValueError('reduce must be one of %s, got %r' % (R.REDUCTIONS, reduce))
  b = bytes(b)
  info, scans, space = parse(b, reduce, progressive)
  if scans is None:
    grids = D.decode_coefficients(b, info)
    qts = [info.qt[c.tq] for c in info.comps]
  else:
    grids = P.coefficients(b, info, scans)
    qts = [info.qt.get(ci, np.zeros(64, np.uint16)) for ci in range(len(info.comps))]
  H, W = R.output_size(info, reduce)
  planes = []
  for p, grid, q in zip(R.plan(info, reduce), grids, qts):
    px = R.IDCTS[p.size](grid, q)
    bh, bw = grid.shape[:2]
    plane = px.transpose(0, 2, 1, 3).reshape(bh * p.size, bw * p.size)[:p.height, :p.width]
    planes.append(R.upsample(plane, p.fh, p.fv, H, W, p.fancy) if len(grids) > 1 else plane[:H, :W])
  return np.ascontiguousarray(D.orient(to_bgr(space, planes), info.orientation))
