"""cv2.imdecode(buf, cv2.IMREAD_COLOR) of a baseline or extended sequential JPEG, restated in numpy.

cv2 4.13 decodes with its bundled libjpeg-turbo 3.1 at its defaults: Huffman decode with DC
prediction reset at each restart marker, the integer "islow" IDCT as its SIMD code computes it,
fancy (triangle-filter) chroma upsampling where libjpeg-turbo has it (h2v1 and h2v2 when the chroma
is wider than 2 samples, h1v2 always) and replication otherwise, libjpeg's fixed-point YCbCr->RGB
tables, grayscale replicated to three channels, then the EXIF orientation applied as cv2 applies
it.  tests/test_oracle_jpeg_decode.py pins every step bitwise against cv2.

parse() accepts exactly what sqdet_jpeg_parse accepts and raises Unsupported with the same reason
codes for the rest."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

# refusal reasons, as sqdet_jpeg_info.reason reports them
OK, MALFORMED, PROGRESSIVE, ARITHMETIC, LOSSLESS, PRECISION, COMPONENTS, COLOR_TRANSFORM, \
    SAMPLING, SIZE, TOO_LARGE = range(11)
REASONS = ('ok', 'malformed or truncated header', 'progressive', 'arithmetic coding', 'lossless',
           'not 8-bit samples', 'not 1 or 3 components', 'RGB-coded',
           'unsupported sampling', 'zero height or width', 'larger than cv2 decodes')
# the largest coded file cv2.imdecode decodes: libjpeg's JPEG_MAX_DIMENSION per side (None above
# it) and cv2's default CV_IO_MAX_IMAGE_PIXELS (cv2.error above it)
MAX_SIDE = 65500
MAX_PIXELS = 1 << 30

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5,
                   12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                   58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
# luma sampling (h, v) -> name; chroma is 1x1 in every supported layout
LAYOUTS = {(1, 1): '4:4:4', (2, 1): '4:2:2', (1, 2): '4:4:0', (2, 2): '4:2:0', (4, 1): '4:1:1'}


class Unsupported(ValueError):
  def __init__(self, reason):
    super().__init__(REASONS[reason])
    self.reason = reason


@dataclass
class Component:
  cid: int
  h: int
  v: int
  tq: int
  td: int = 0
  ta: int = 0


@dataclass
class Info:
  height: int                 # as decoded, before orientation
  width: int
  comps: list
  qt: dict                    # table id -> 64 uint16 in natural order
  dc: dict                    # table id -> (bits[16], vals)
  ac: dict
  restart: int = 0
  orientation: int = 1
  scan: int = 0               # offset of the entropy-coded segment
  hmax: int = 1
  vmax: int = 1
  extra: dict = field(default_factory=dict)

  @property
  def out_hw(self):
    return (self.width, self.height) if self.orientation >= 5 else (self.height, self.width)


def _u16(b, i):
  if i + 2 > len(b):
    raise Unsupported(MALFORMED)
  return (b[i] << 8) | b[i + 1]


def exif_orientation(seg):
  """The Orientation tag (0x0112) of IFD0 in an APP1 'Exif\\0\\0' body, or 1.  As cv2 reads it:
  the first 0x0112 entry, its u16 at entry offset 8 in the TIFF byte order whatever the entry's
  type and count, with only the entry's bytes [0, 10) needed inside the segment; a value outside
  1..8 means 1."""
  if len(seg) < 14 or seg[:6] != b'Exif\x00\x00':
    return 1
  t = seg[6:]
  if t[:2] == b'II':
    rd = lambda i, n: int.from_bytes(t[i:i + n], 'little')
  elif t[:2] == b'MM':
    rd = lambda i, n: int.from_bytes(t[i:i + n], 'big')
  else:
    return 1
  if rd(2, 2) != 42:
    return 1
  ifd = rd(4, 4)
  if ifd + 2 > len(t):
    return 1
  for e in range(rd(ifd, 2)):
    p = ifd + 2 + 12 * e
    if p + 10 > len(t):
      break
    if rd(p, 2) == 0x0112:
      o = rd(p + 8, 2)
      return o if 1 <= o <= 8 else 1
  return 1


def parse(b):
  """Headers up to the first SOS -> Info, or Unsupported."""
  b = bytes(b)
  if len(b) < 4 or b[0] != 0xFF or b[1] != 0xD8:
    raise Unsupported(MALFORMED)
  qt, dc, ac = {}, {}, {}
  restart, orientation, adobe = 0, 1, None
  frame = None
  saw_exif = jfif = False
  i = 2
  while True:
    while i < len(b) and b[i] == 0xFF and i + 1 < len(b) and b[i + 1] == 0xFF:
      i += 1                               # fill bytes
    if i + 2 > len(b) or b[i] != 0xFF:
      raise Unsupported(MALFORMED)
    m = b[i + 1]
    i += 2
    if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
      raise Unsupported(MALFORMED)
    n = _u16(b, i)
    if n < 2 or i + n > len(b):
      raise Unsupported(MALFORMED)
    body = b[i + 2:i + n]
    i += n
    if m in (0xC2, 0xC6, 0xCA, 0xCE):
      raise Unsupported(PROGRESSIVE)
    if m in (0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF):
      raise Unsupported(ARITHMETIC)
    if m in (0xC3, 0xC7, 0xCB, 0xCF):
      raise Unsupported(LOSSLESS)
    if m in (0xC5, 0xC6, 0xC7):
      raise Unsupported(PROGRESSIVE)       # hierarchical
    if m in (0xC0, 0xC1):
      if frame is not None or len(body) < 6:
        raise Unsupported(MALFORMED)
      p, hh, ww, nc = body[0], _u16(body, 1), _u16(body, 3), body[5]
      if p != 8:
        raise Unsupported(PRECISION)
      if len(body) != 6 + 3 * nc:
        raise Unsupported(MALFORMED)
      if nc not in (1, 3):
        raise Unsupported(COMPONENTS)
      comps = [Component(body[6 + 3 * k], body[7 + 3 * k] >> 4, body[7 + 3 * k] & 15,
                         body[8 + 3 * k]) for k in range(nc)]
      if hh == 0 or ww == 0:
        raise Unsupported(SIZE)
      if hh > MAX_SIDE or ww > MAX_SIDE or hh * ww > MAX_PIXELS:
        raise Unsupported(TOO_LARGE)
      if any(c.tq > 3 or not 1 <= c.h <= 4 or not 1 <= c.v <= 4 for c in comps):
        raise Unsupported(MALFORMED)
      if nc == 3 and ((comps[0].h, comps[0].v) not in LAYOUTS
                      or any((c.h, c.v) != (1, 1) for c in comps[1:])):
        raise Unsupported(SAMPLING)
      frame = (hh, ww, comps)
    elif m == 0xDB:
      j = 0
      while j < len(body):
        pq, tq = body[j] >> 4, body[j] & 15
        size = 128 if pq else 64
        if pq > 1 or tq > 3 or j + 1 + size > len(body):
          raise Unsupported(MALFORMED)
        raw = np.frombuffer(body[j + 1:j + 1 + size], '>u2' if pq else 'u1').astype(np.uint16)
        q = np.zeros(64, np.uint16)
        q[ZIGZAG] = raw
        qt[tq] = q
        j += 1 + size
    elif m == 0xC4:
      j = 0
      while j < len(body):
        if j + 17 > len(body):
          raise Unsupported(MALFORMED)
        tc, th = body[j] >> 4, body[j] & 15
        bits = list(body[j + 1:j + 17])
        cnt = sum(bits)
        if tc > 1 or th > 3 or cnt > 256 or j + 17 + cnt > len(body):
          raise Unsupported(MALFORMED)
        (ac if tc else dc)[th] = (bits, list(body[j + 17:j + 17 + cnt]))
        j += 17 + cnt
    elif m == 0xDD:
      if len(body) != 2:
        raise Unsupported(MALFORMED)
      restart = _u16(body, 0)
    elif m == 0xE1 and not saw_exif and body[:6] == b'Exif\x00\x00':
      saw_exif = True
      orientation = exif_orientation(body)
    elif m == 0xE0 and len(body) >= 14 and body[:5] == b'JFIF\x00':
      jfif = True
    elif m == 0xEE and len(body) >= 12 and body[:5] == b'Adobe':
      adobe = body[11]
    elif m == 0xDA:
      if frame is None or len(body) < 1:
        raise Unsupported(MALFORMED)
      hh, ww, comps = frame
      ns = body[0]
      if len(body) != 4 + 2 * ns:
        raise Unsupported(MALFORMED)
      ids = [body[1 + 2 * k] for k in range(ns)]
      if ns != len(comps) or ids != [c.cid for c in comps]:
        raise Unsupported(SAMPLING)        # multi-scan sequential files
      for k, c in enumerate(comps):
        c.td, c.ta = body[2 + 2 * k] >> 4, body[2 + 2 * k] & 15
        if c.td > 3 or c.ta > 3:
          raise Unsupported(MALFORMED)
        if c.td not in dc or c.ta not in ac or c.tq not in qt:
          raise Unsupported(MALFORMED)
        if not huff_ok(*dc[c.td], True) or not huff_ok(*ac[c.ta], False):
          raise Unsupported(MALFORMED)
      ss, se, ahal = body[1 + 2 * ns], body[2 + 2 * ns], body[3 + 2 * ns]
      if ss != 0 or se != 63 or ahal != 0:
        raise Unsupported(MALFORMED)
      # libjpeg's colour space of 3 components: YCbCr after a JFIF APP0; else as an Adobe APP14's
      # transform says (0: RGB); else RGB for component ids 'R', 'G', 'B'
      if len(comps) == 3 and not jfif and (adobe == 0 if adobe is not None else ids == [82, 71, 66]):
        raise Unsupported(COLOR_TRANSFORM)
      info = Info(hh, ww, comps, qt, dc, ac, restart, orientation, i)
      info.hmax = max(c.h for c in comps)
      info.vmax = max(c.v for c in comps)
      return info
    # APPn, COM and anything else sequential files may carry: skipped


def huff_ok(bits, vals, dc):
  """libjpeg's checks of a Huffman table a scan uses: no length's codes run past its all-ones
  code, and a DC table's symbols are categories 0..15."""
  code = 0
  for ln in range(1, 17):
    code += bits[ln - 1]
    if code >= 1 << ln:
      return False
    code <<= 1
  return not dc or all(v <= 15 for v in vals)


def huff_lut(bits, vals):
  """16-bit peek -> (length, symbol); length 0 for a code not in the table."""
  lut_len = np.zeros(1 << 16, np.int32)
  lut_sym = np.zeros(1 << 16, np.int32)
  code, k = 0, 0
  for ln in range(1, 17):
    for _ in range(bits[ln - 1]):
      if code >= (1 << ln):
        return lut_len.tolist(), lut_sym.tolist()   # over-subscribed: the rest never decode
      lo = code << (16 - ln)
      hi = (code + 1) << (16 - ln)
      lut_len[lo:hi] = ln
      lut_sym[lo:hi] = vals[k]
      code += 1
      k += 1
    code <<= 1
  return lut_len.tolist(), lut_sym.tolist()


class CorruptData(ValueError):
  pass


def entropy_intervals(b, start):
  """The destuffed bytes of each restart interval of the scan starting at b[start]."""
  out, cur = [], bytearray()
  i, n = start, len(b)
  while i < n:
    x = b[i]
    if x != 0xFF:
      cur.append(x)
      i += 1
      continue
    nx = b[i + 1] if i + 1 < n else None
    if nx == 0x00:
      cur.append(0xFF)
      i += 2
    elif nx == 0xFF:
      i += 1
    elif nx is not None and 0xD0 <= nx <= 0xD7:
      out.append((bytes(cur), nx - 0xD0))
      cur = bytearray()
      i += 2
    else:
      break
  out.append((bytes(cur), None))
  return out


def _extend(v, s):
  return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def mcu_geometry(info):
  """(blocks per MCU as component indices, MCU columns, MCU rows)."""
  if len(info.comps) == 1:
    return [0], -(-info.width // 8), -(-info.height // 8)
  order = [ci for ci, c in enumerate(info.comps) for _ in range(c.h * c.v)]
  return order, -(-info.width // (8 * info.hmax)), -(-info.height // (8 * info.vmax))


def decode_coefficients(b, info):
  """-> per component, quantized coefficients [rows, cols, 64] in natural order (JCOEF values),
  on the component's padded block grid."""
  order, mcols, mrows = mcu_geometry(info)
  comps = info.comps
  single = len(comps) == 1
  grids = []
  for c in comps:
    bh, bw = (mrows, mcols) if single else (mrows * c.v, mcols * c.h)
    grids.append(np.zeros((bh, bw, 64), np.int32))
  luts = {}
  for c in comps:
    luts.setdefault(('d', c.td), huff_lut(*info.dc[c.td]))
    luts.setdefault(('a', c.ta), huff_lut(*info.ac[c.ta]))
  mcus = mcols * mrows
  per = info.restart if info.restart else mcus
  intervals = entropy_intervals(b, info.scan)
  want = -(-mcus // per)
  if len(intervals) < want:
    raise CorruptData('%d restart intervals, expected %d' % (len(intervals), want))
  for r in range(want):
    data, rst = intervals[r]
    if r < want - 1 and rst != r % 8:
      raise CorruptData('restart marker %s, expected %d' % (rst, r % 8))
    buf = data + b'\xff\xff\xff\xff'
    nbits = 8 * len(data)
    p = 0

    def peek16(p):
      q = p >> 3
      return ((buf[q] << 16 | buf[q + 1] << 8 | buf[q + 2]) >> (8 - (p & 7))) & 0xFFFF

    def get(p, s):
      q = p >> 3
      w = int.from_bytes(buf[q:q + 4], 'big')
      return (w >> (32 - (p & 7) - s)) & ((1 << s) - 1)

    pred = [0] * len(comps)
    for m in range(r * per, min(mcus, (r + 1) * per)):
      my, mx = divmod(m, mcols)
      seen = [0] * len(comps)
      for ci in order:
        c = comps[ci]
        dl, ds = luts[('d', c.td)]
        al, asym = luts[('a', c.ta)]
        blk = np.zeros(64, np.int32)
        pk = peek16(p)
        ln = dl[pk]
        if ln == 0:
          raise CorruptData('invalid DC code')
        s = ds[pk]
        p += ln
        if s > 15:
          raise CorruptData('DC category above 15')
        diff = _extend(get(p, s), s) if s else 0
        p += s
        pred[ci] += diff
        blk[0] = ((pred[ci] + 0x8000) & 0xFFFF) - 0x8000
        k = 1
        while k < 64:
          pk = peek16(p)
          ln = al[pk]
          if ln == 0:
            raise CorruptData('invalid AC code')
          rs = asym[pk]
          p += ln
          run, s = rs >> 4, rs & 15
          if s:
            k += run
            if k > 63:
              raise CorruptData('run past coefficient 63')
            blk[ZIGZAG[k]] = _extend(get(p, s), s)
            p += s
            k += 1
          elif run == 15:
            k += 16
            if k > 64:
              raise CorruptData('run past coefficient 63')
          else:
            break
        if p > nbits:
          raise CorruptData('ran off the data')
        if single:
          grids[ci][my, mx] = blk
        else:
          u = seen[ci]
          seen[ci] += 1
          grids[ci][my * c.v + u // c.h, mx * c.h + u % c.h] = blk
  return grids


# jidctint constants, 13 fraction bits
F0_298, F0_390, F0_541, F0_765 = 2446, 3196, 4433, 6270
F0_899, F1_175, F1_501, F1_847 = 7373, 9633, 12299, 15137
F1_961, F2_053, F2_562, F3_072 = 16069, 16819, 20995, 25172


def _w16(x):
  """x wrapped to int16 (a 16-bit SIMD add or multiply), as int32."""
  return x.astype(np.int16).astype(np.int32)


def _s16(x):
  """x saturated to int16 (packssdw), as int32."""
  return np.clip(x, -32768, 32767).astype(np.int32)


def _idct_pass(d, shift):
  """One 1-D islow pass over axis -2 of int16-valued int32 [..., 8, 8], descaled by `shift`, as
  libjpeg-turbo's SIMD islow computes it: products and their sums in 32 bits, but in0 +- in4,
  in7 + in3 and in5 + in1 in 16 bits (they wrap).  Equal to jidctint.c's arithmetic whenever
  those sums fit 16 bits."""
  g = lambda k: d[..., k, :]
  z2, z3 = g(2), g(6)
  z1 = (z2 + z3) * F0_541
  tmp2 = z1 - z3 * F1_847
  tmp3 = z1 + z2 * F0_765
  tmp0 = _w16(g(0) + g(4)) << 13
  tmp1 = _w16(g(0) - g(4)) << 13
  t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
  a0, a1, a2, a3 = g(7), g(5), g(3), g(1)
  z1, z2, z3, z4 = a0 + a3, a1 + a2, _w16(a0 + a2), _w16(a1 + a3)
  z5 = (z3 + z4) * F1_175
  a0, a1, a2, a3 = a0 * F0_298, a1 * F2_053, a2 * F3_072, a3 * F1_501
  z1, z2 = z1 * -F0_899, z2 * -F2_562
  z3, z4 = z3 * -F1_961 + z5, z4 * -F0_390 + z5
  a0 = a0 + z1 + z3
  a1 = a1 + z2 + z4
  a2 = a2 + z2 + z3
  a3 = a3 + z1 + z4
  rnd = np.int32(1 << (shift - 1))
  out = [t10 + a3, t11 + a2, t12 + a1, t13 + a0, t13 - a0, t12 - a1, t11 - a2, t10 - a3]
  return np.stack([(o + rnd) >> shift for o in out], axis=-2)


def idct_islow(coef, q):
  """jpeg_idct_islow of quantized coefficients [..., 64] (natural order) with quant table q ->
  uint8 samples [..., 8, 8], as cv2's libjpeg-turbo runs it: its SIMD islow, which dequantizes
  with a 16-bit multiply, keeps the column pass's results in 16 bits (saturating), takes a block
  whose AC coefficients are all zero as its DC << 2 (16-bit), and clamps the output.  For
  coefficients an 8-bit encoder writes this is jidctint.c's result; it differs only where 16 bits
  overflow."""
  c16 = coef.astype(np.int16).astype(np.int32)                      # JCOEF
  q16 = q.astype(np.uint16).view(np.int16).astype(np.int32)
  shape = coef.shape[:-1] + (8, 8)
  d = _w16(c16 * q16).reshape(shape)                                # int32 sums wrap as paddd does
  ws = _s16(_idct_pass(d, 11))                                      # columns: axis -2 is rows
  dc_only = (c16.reshape(shape)[..., 1:, :] == 0).all(axis=(-1, -2))
  ws_dc = np.broadcast_to(_w16(d[..., :1, :] << 2), shape)
  ws = np.where(dc_only[..., None, None], ws_dc, ws).astype(np.int32)
  rows = np.swapaxes(ws, -1, -2)                                    # each row as a column
  v = _s16(np.swapaxes(_idct_pass(rows, 18), -1, -2))
  return (np.clip(v, -128, 127) + 128).astype(np.uint8)


def component_planes(b, info):
  """Each component's samples at its own resolution, cropped to its downsampled size."""
  grids = decode_coefficients(b, info)
  planes = []
  for c, grid in zip(info.comps, grids):
    px = idct_islow(grid, info.qt[c.tq])                            # [bh, bw, 8, 8]
    bh, bw = grid.shape[:2]
    plane = px.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)
    ch = -(-info.height * c.v // info.vmax)
    cw = -(-info.width * c.h // info.hmax)
    planes.append(plane[:ch, :cw])
  return planes


def upsample(c, fh, fv, H, W):
  """A chroma plane upsampled by (fh, fv) to H x W as libjpeg-turbo does with fancy upsampling
  on."""
  c = c.astype(np.int32)
  ch, cw = c.shape
  if (fh, fv) == (1, 1):
    return c[:H, :W]
  fancy_h = fh == 2 and cw > 2
  if fv == 2 and (fh == 1 or fancy_h):
    up = c[np.maximum(np.arange(ch) - 1, 0)]
    dn = c[np.minimum(np.arange(ch) + 1, ch - 1)]
    rows = np.empty((2 * ch, cw), np.int32)
    rows[0::2] = 3 * c + up
    rows[1::2] = 3 * c + dn
    if fh == 1:                                                     # h1v2: biases 1, 2
      rows[0::2] += 1
      rows[1::2] += 2
      return (rows >> 2)[:H, :W]
    left = rows[:, np.maximum(np.arange(cw) - 1, 0)]                # h2v2: biases 8, 7
    right = rows[:, np.minimum(np.arange(cw) + 1, cw - 1)]
    out = np.empty((2 * ch, 2 * cw), np.int32)
    out[:, 0::2] = (3 * rows + left + 8) >> 4
    out[:, 1::2] = (3 * rows + right + 7) >> 4
    return out[:H, :W]
  if fv == 1 and fancy_h:                                           # h2v1: biases 1, 2
    left = c[:, np.maximum(np.arange(cw) - 1, 0)]
    right = c[:, np.minimum(np.arange(cw) + 1, cw - 1)]
    out = np.empty((ch, 2 * cw), np.int32)
    out[:, 0::2] = (3 * c + left + 1) >> 2
    out[:, 1::2] = (3 * c + right + 2) >> 2
    return out[:H, :W]
  return np.repeat(np.repeat(c, fv, axis=0), fh, axis=1)[:H, :W]


def _fix(x):
  return int(x * 65536 + 0.5)


def ycc_to_bgr(y, cb, cr):
  """jdcolor.c's ycc_rgb_convert (16 fraction bits), as B, G, R."""
  y = y.astype(np.int64)
  cb = cb.astype(np.int64) - 128
  cr = cr.astype(np.int64) - 128
  r = y + ((_fix(1.40200) * cr + 32768) >> 16)
  b = y + ((_fix(1.77200) * cb + 32768) >> 16)
  g = y + ((-_fix(0.34414) * cb + 32768 - _fix(0.71414) * cr) >> 16)
  return np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8)


def orient(img, o):
  """EXIF orientation o applied as cv2.imdecode applies it."""
  if o == 2:
    return img[:, ::-1]
  if o == 3:
    return img[::-1, ::-1]
  if o == 4:
    return img[::-1]
  t = np.swapaxes(img, 0, 1)
  if o == 5:
    return t
  if o == 6:
    return t[:, ::-1]
  if o == 7:
    return t[::-1, ::-1]
  if o == 8:
    return t[::-1]
  return img


def decode(b):
  """cv2.imdecode(b, cv2.IMREAD_COLOR) -> uint8 [H, W, 3] BGR.  Unsupported for files outside the
  supported set, CorruptData for a bad entropy-coded segment."""
  b = bytes(b)
  info = parse(b)
  planes = component_planes(b, info)
  H, W = info.height, info.width
  if len(planes) == 1:
    bgr = np.repeat(planes[0][:H, :W, None], 3, axis=2)
  else:
    c0 = info.comps[0]
    y = planes[0][:H, :W]
    cb = upsample(planes[1], c0.h, c0.v, H, W)
    cr = upsample(planes[2], c0.h, c0.v, H, W)
    bgr = ycc_to_bgr(y, cb, cr)
  return np.ascontiguousarray(orient(bgr, info.orientation))


def with_orientation(jpeg, o, little_endian=False):
  """`jpeg` with an APP1 EXIF segment carrying Orientation o inserted after SOI."""
  if little_endian:
    tiff = b'II' + (42).to_bytes(2, 'little') + (8).to_bytes(4, 'little') + (1).to_bytes(2, 'little') \
        + (0x0112).to_bytes(2, 'little') + (3).to_bytes(2, 'little') + (1).to_bytes(4, 'little') \
        + o.to_bytes(2, 'little') + b'\x00\x00' + (0).to_bytes(4, 'little')
  else:
    tiff = b'MM' + (42).to_bytes(2, 'big') + (8).to_bytes(4, 'big') + (1).to_bytes(2, 'big') \
        + (0x0112).to_bytes(2, 'big') + (3).to_bytes(2, 'big') + (1).to_bytes(4, 'big') \
        + o.to_bytes(2, 'big') + b'\x00\x00' + (0).to_bytes(4, 'big')
  body = b'Exif\x00\x00' + tiff
  seg = b'\xff\xe1' + (len(body) + 2).to_bytes(2, 'big') + body
  return bytes(jpeg[:2]) + seg + bytes(jpeg[2:])
