"""cv2.imdecode(buf, cv2.IMREAD_COLOR) of a progressive (SOF2) Huffman JPEG, restated in numpy and
plain Python.

cv2 4.13's libjpeg-turbo 3.1 reads every scan into a whole-image coefficient buffer and runs its
output pass once the file has ended, so a progressive file decodes to the pixels of a sequential
file holding the final coefficients, unless libjpeg block-smooths it.  This module restates:

  parse     every SOS with the DHT, DQT and DRI in force at that point; per scan its components,
            Ss, Se, Ah, Al, tables, restart interval and entropy-coded bytes.  A component's
            quantization table is latched at the first scan that contains it (a later DQT has no
            effect on it).  Refusals, after oracle.jpeg_decode's:
              BAD_PROGRESSION   what start_pass_phuff_decoder rejects (JERR_BAD_PROGRESSION; cv2
                                returns None): a DC scan with Se != 0, an AC scan with Ss > Se,
                                Se > 63 or more than one component, Ah != 0 with Al != Ah - 1,
                                Al > 13
              BOGUS_PROGRESSION what it warns on (JWRN_BOGUS_PROGRESSION; cv2 decodes): an AC scan
                                before the component's DC, an Ah other than the coefficient's
                                last Al; and a first scan (Ah = 0) of a coefficient already coded,
                                which libjpeg lets overwrite it
              SMOOTHED          files jdcoefct.c's smoothing_ok smooths: every component latched
                                a table whose DC and first nine AC quantizers are nonzero, every
                                component has DC bits, and some coefficient 1..9 of some component
                                is not yet exact (never coded, or its last Al above 0)
              TOO_MANY_SCANS    more than MAX_SCANS scans (the scans past the cap are still
                                checked for the refusals above, which come first)
            Scans whose components are out of the frame's order, or repeated, are refused as
            SAMPLING, as oracle.jpeg_decode refuses them (libjpeg decodes some of them, such as
            Cr before Cb, and rejects others, such as Y, Cr, Cb)
            Sequential files go to oracle.jpeg_decode.parse unchanged.
  scans     jdphuff.c: DC first (pred + diff) << Al stored as JCOEF; DC refinement one raw bit per
            block ORed in as 1 << Al; AC first v << Al with EOBn runs of 2^n + n bits; AC
            refinement's run/size-1 symbols, sign bits and correction bits (+p1 or +m1 where
            (coef & p1) == 0).  An interleaved scan (DC only, any subset of the components) walks
            the frame's MCUs, padding blocks included; a one-component scan walks the component's
            own ceil(w_c / 8) x ceil(h_c / 8) blocks, and its restart interval counts blocks.  A
            restart resets the DC predictors and EOBRUN.
  output    oracle.jpeg_decode's IDCT, upsampling, colour conversion and orientation.

CorruptData for what the device decoder fails a file on: an invalid code, a run past Se, a
refinement symbol of size other than 1, an EOBRUN past its interval, an RSTn out of sequence or
missing, and data that runs out.  tests/test_oracle_jpeg_decode_progressive.py pins it bitwise
against cv2."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle import jpeg_decode as D
from oracle.jpeg_decode import CorruptData, ZIGZAG

BAD_PROGRESSION, BOGUS_PROGRESSION, SMOOTHED, TOO_MANY_SCANS = range(11, 15)
REASONS = D.REASONS + ('scan script libjpeg rejects', 'scan script libjpeg warns on or overwrites',
                       'block-smoothed by libjpeg', 'more than 256 scans')
MAX_SCANS = 256
# the natural-order positions smoothing_ok needs nonzero: Q00, Q01, Q10, Q20, Q11, Q02, Q03, Q12,
# Q21, Q30
SMOOTH_Q = (0, 1, 8, 16, 9, 2, 3, 10, 17, 24)


class Unsupported(D.Unsupported):
  def __init__(self, reason):
    ValueError.__init__(self, REASONS[reason])
    self.reason = reason


@dataclass
class Scan:
  comps: list                 # frame component indices, in frame order
  ss: int
  se: int
  ah: int
  al: int
  tables: list                # per component: (bits, vals) of its DC (first DC scans) or AC table
  restart: int                # MCUs (interleaved) or blocks per interval, 0 for none
  start: int                  # first byte of the entropy-coded data
  end: int                    # the terminating marker's 0xFF (or the file's end)


def _data_end(b, j):
  """The first byte at or after j that starts a marker other than RSTn (or len(b))."""
  n = len(b)
  while True:
    j = b.find(b'\xff', j)
    if j < 0:
      return n
    nx = b[j + 1] if j + 1 < n else None
    if nx is None or not (nx == 0x00 or nx == 0xFF or 0xD0 <= nx <= 0xD7):
      return j
    j += 1


def parse(b):
  """-> (Info, scans): scans None for a sequential file (oracle.jpeg_decode.parse's Info), else
  the list of Scan, with Info.qt holding each component's latched table under its index."""
  b = bytes(b)
  try:
    return D.parse(b), None
  except D.Unsupported as e:
    if e.reason != D.PROGRESSIVE:
      raise Unsupported(e.reason) from None
  # everything before the frame header is what oracle.jpeg_decode.parse accepted
  qt, dc, ac = {}, {}, {}
  restart, orientation, adobe = 0, 1, None
  frame = None
  saw_exif = jfif = False
  scans, latched = [], {}
  bogus = too_many = False
  bits = None                   # per component: the last Al of each coefficient (-1: none)
  i = 2
  while True:
    while i + 1 < len(b) and b[i] == 0xFF and b[i + 1] == 0xFF:
      i += 1
    if scans and i >= len(b):
      break                     # no EOI: libjpeg ends the image there
    if i + 2 > len(b) or b[i] != 0xFF:
      raise Unsupported(D.MALFORMED)
    m = b[i + 1]
    i += 2
    if m == 0xD9 and scans:
      break
    if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
      raise Unsupported(D.MALFORMED)
    n = D._u16(b, i) if i + 2 <= len(b) else -1
    if n < 2 or i + n > len(b):
      raise Unsupported(D.MALFORMED)
    body = b[i + 2:i + n]
    i += n
    if m == 0xC2:
      if frame is not None or len(body) < 6:
        raise Unsupported(D.MALFORMED)
      p, hh, ww, nc = body[0], D._u16(body, 1), D._u16(body, 3), body[5]
      if p != 8:
        raise Unsupported(D.PRECISION)
      if len(body) != 6 + 3 * nc:
        raise Unsupported(D.MALFORMED)
      if nc not in (1, 3):
        raise Unsupported(D.COMPONENTS)
      comps = [D.Component(body[6 + 3 * k], body[7 + 3 * k] >> 4, body[7 + 3 * k] & 15,
                           body[8 + 3 * k]) for k in range(nc)]
      if hh == 0 or ww == 0:
        raise Unsupported(D.SIZE)
      if hh > D.MAX_SIDE or ww > D.MAX_SIDE or hh * ww > D.MAX_PIXELS:
        raise Unsupported(D.TOO_LARGE)
      if any(c.tq > 3 or not 1 <= c.h <= 4 or not 1 <= c.v <= 4 for c in comps):
        raise Unsupported(D.MALFORMED)
      if nc == 3 and ((comps[0].h, comps[0].v) not in D.LAYOUTS
                      or any((c.h, c.v) != (1, 1) for c in comps[1:])):
        raise Unsupported(D.SAMPLING)
      frame = (hh, ww, comps)
      bits = [[-1] * 64 for _ in comps]
    elif m in (0xC0, 0xC1, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF):
      raise Unsupported(D.MALFORMED if frame is not None else D.PROGRESSIVE)
    elif m == 0xDB:
      j = 0
      while j < len(body):
        pq, tq = body[j] >> 4, body[j] & 15
        size = 128 if pq else 64
        if pq > 1 or tq > 3 or j + 1 + size > len(body):
          raise Unsupported(D.MALFORMED)
        raw = np.frombuffer(body[j + 1:j + 1 + size], '>u2' if pq else 'u1').astype(np.uint16)
        q = np.zeros(64, np.uint16)
        q[ZIGZAG] = raw
        qt[tq] = q
        j += 1 + size
    elif m == 0xC4:
      j = 0
      while j < len(body):
        if j + 17 > len(body):
          raise Unsupported(D.MALFORMED)
        tc, th = body[j] >> 4, body[j] & 15
        hb = list(body[j + 1:j + 17])
        cnt = sum(hb)
        if tc > 1 or th > 3 or cnt > 256 or j + 17 + cnt > len(body):
          raise Unsupported(D.MALFORMED)
        (ac if tc else dc)[th] = (hb, list(body[j + 17:j + 17 + cnt]))
        j += 17 + cnt
    elif m == 0xDD:
      if len(body) != 2:
        raise Unsupported(D.MALFORMED)
      restart = D._u16(body, 0)
    elif scans and 0xE0 <= m <= 0xEF:
      pass                     # APPn after the first scan: read by neither libjpeg nor cv2
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
      hh, ww, comps = frame
      ns = body[0]
      if len(body) != 4 + 2 * ns or not 1 <= ns <= 4:
        raise Unsupported(D.MALFORMED)
      ids = [body[1 + 2 * k] for k in range(ns)]
      idx = [next((ci for ci, c in enumerate(comps) if c.cid == x), None) for x in ids]
      if None in idx:
        raise Unsupported(D.MALFORMED)
      if any(b_ <= a_ for a_, b_ in zip(idx, idx[1:])):
        raise Unsupported(D.SAMPLING)       # components out of the frame's order, or repeated
      if not scans and len(comps) == 3 and not jfif and \
          (adobe == 0 if adobe is not None else [c.cid for c in comps] == [82, 71, 66]):
        raise Unsupported(D.COLOR_TRANSFORM)
      ss, se, ah, al = body[1 + 2 * ns], body[2 + 2 * ns], body[3 + 2 * ns] >> 4, body[3 + 2 * ns] & 15
      for ci in idx:                         # latch_quant_tables
        if ci not in latched:
          if comps[ci].tq not in qt:
            raise Unsupported(D.MALFORMED)
          latched[ci] = qt[comps[ci].tq].copy()
      dc_band = ss == 0
      bad = (se != 0) if dc_band else (ss > se or se > 63 or ns != 1)
      if (ah != 0 and al != ah - 1) or al > 13 or bad:
        raise Unsupported(BAD_PROGRESSION)
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
      end = _data_end(b, i)
      # past the cap the scans are still checked, so that a later one libjpeg rejects is reported
      # as libjpeg reports it
      if len(scans) == MAX_SCANS:
        too_many = True
      else:
        scans.append(Scan(idx, ss, se, ah, al, tables, restart, i, end))
      i = end
    # APPn, COM and anything else: skipped
  if too_many:
    raise Unsupported(TOO_MANY_SCANS)
  if bogus:
    raise Unsupported(BOGUS_PROGRESSION)
  if smoothed(frame[2], latched, bits):
    raise Unsupported(SMOOTHED)
  hh, ww, comps = frame
  info = D.Info(hh, ww, comps, latched, dc, ac, 0, orientation, scans[0].start)
  info.hmax = max(c.h for c in comps)
  info.vmax = max(c.v for c in comps)
  return info, scans


def smoothed(comps, latched, bits):
  """jdcoefct.c's smoothing_ok at the output pass, from the final coefficient bits."""
  useful = False
  for ci in range(len(comps)):
    q = latched.get(ci)
    if q is None or any(int(q[k]) == 0 for k in SMOOTH_Q) or bits[ci][0] < 0:
      return False
    useful = useful or any(x != 0 for x in bits[ci][1:10])
  return useful


def grid_shapes(info):
  """Per component: (padded block grid rows, cols) as the coefficient buffer holds it, and the
  component's own block grid (rows, cols) a one-component scan walks."""
  order, mcols, mrows = D.mcu_geometry(info)
  out = []
  for c in info.comps:
    if len(info.comps) == 1:
      pad = (mrows, mcols)
    else:
      pad = (mrows * c.v, mcols * c.h)
    ch = -(-info.height * c.v // info.vmax)
    cw = -(-info.width * c.h // info.hmax)
    out.append((pad, (-(-ch // 8), -(-cw // 8))))
  return out


class _Bits:
  def __init__(self, data):
    self.buf = data + b'\x00' * 8
    self.nbits = 8 * len(data)
    self.p = 0

  def peek16(self):
    q = self.p >> 3
    return ((self.buf[q] << 16 | self.buf[q + 1] << 8 | self.buf[q + 2]) >> (8 - (self.p & 7))) & 0xFFFF

  def get(self, s):
    if not s:
      return 0
    q = self.p >> 3
    w = int.from_bytes(self.buf[q:q + 4], 'big')
    v = (w >> (32 - (self.p & 7) - s)) & ((1 << s) - 1)
    self.p += s
    return v

  def sym(self, lut):
    ln, sy = lut
    pk = self.peek16()
    if ln[pk] == 0:
      raise CorruptData('invalid code')
    self.p += ln[pk]
    return sy[pk]


def _units(info, scan, shapes):
  """The scan's units in order, each the (component, block row, block column) it codes."""
  if len(scan.comps) > 1:
    _, mcols, mrows = D.mcu_geometry(info)
    out = []
    for my in range(mrows):
      for mx in range(mcols):
        out.append([(ci, my * info.comps[ci].v + dy, mx * info.comps[ci].h + dx)
                    for ci in scan.comps for dy in range(info.comps[ci].v)
                    for dx in range(info.comps[ci].h)])
    return out
  ci = scan.comps[0]
  bh, bw = shapes[ci][1]
  return [[(ci, by, bx)] for by in range(bh) for bx in range(bw)]


def _jcoef(v):
  return ((v + 0x8000) & 0xFFFF) - 0x8000


def decode_scan(b, info, scan, grids, shapes):
  """Applies one scan's coefficients to grids (per component [rows, cols, 64] int32)."""
  units = _units(info, scan, shapes)
  if len(info.comps) == 1 and len(scan.comps) > 1:
    raise AssertionError('unreachable')
  per = scan.restart if scan.restart else len(units)
  want = -(-len(units) // per)
  ivs = D.entropy_intervals(b[:scan.end], scan.start)
  if len(ivs) < want:
    raise CorruptData('%d restart intervals, expected %d' % (len(ivs), want))
  luts = [D.huff_lut(*t) if t is not None else None for t in scan.tables]
  lut_of = dict(zip(scan.comps, luts))
  ss, se, ah, al = scan.ss, scan.se, scan.ah, scan.al
  p1, m1 = 1 << al, -1 << al
  for r in range(want):
    data, rst = ivs[r]
    if r < want - 1 and rst != r % 8:
      raise CorruptData('restart marker %s, expected %d' % (rst, r % 8))
    bits = _Bits(data)
    pred = {ci: 0 for ci in scan.comps}
    eobrun = 0
    for unit in units[r * per:(r + 1) * per]:
      for ci, by, bx in unit:
        blk = grids[ci][by, bx]
        if ss == 0 and ah == 0:
          s = bits.sym(lut_of[ci])
          pred[ci] += D._extend(bits.get(s), s) if s else 0
          blk[0] = _jcoef(pred[ci] << al)
        elif ss == 0:
          if bits.get(1):
            blk[0] = _jcoef(blk[0] | p1)
        elif ah == 0:
          if eobrun:
            eobrun -= 1
            continue
          k = ss
          while k <= se:
            rs = bits.sym(lut_of[ci])
            run, s = rs >> 4, rs & 15
            if s:
              k += run
              if k > se:
                raise CorruptData('run past Se')
              blk[ZIGZAG[k]] = _jcoef(D._extend(bits.get(s), s) << al)
              k += 1
            elif run == 15:
              k += 16
              if k > se + 1:
                raise CorruptData('run past Se')
            else:
              eobrun = (1 << run) + bits.get(run) - 1
              break
        else:
          k = ss
          if eobrun == 0:
            while k <= se:
              rs = bits.sym(lut_of[ci])
              run, s = rs >> 4, rs & 15
              val = 0
              if s:
                if s != 1:
                  raise CorruptData('refinement size other than 1')
                val = p1 if bits.get(1) else m1
              elif run != 15:
                eobrun = (1 << run) + bits.get(run)
                break
              while True:                    # past nonzeros (correcting) and `run` zeros
                if k > se:
                  raise CorruptData('run past Se')
                z = ZIGZAG[k]
                if blk[z] != 0:
                  if bits.get(1) and (blk[z] & p1) == 0:
                    blk[z] = _jcoef(blk[z] + (p1 if blk[z] >= 0 else m1))
                else:
                  run -= 1
                  if run < 0:
                    break
                k += 1
              if val:
                blk[ZIGZAG[k]] = val
              k += 1
          if eobrun > 0:
            for kk in range(k, se + 1):
              z = ZIGZAG[kk]
              if blk[z] != 0 and bits.get(1) and (blk[z] & p1) == 0:
                blk[z] = _jcoef(blk[z] + (p1 if blk[z] >= 0 else m1))
            eobrun -= 1
      if bits.p > bits.nbits:
        raise CorruptData('ran off the data')
    if eobrun:
      raise CorruptData('EOBRUN past the interval')


def coefficients(b, info, scans):
  """-> per component, the final coefficients [rows, cols, 64] on its padded block grid."""
  shapes = grid_shapes(info)
  grids = [np.zeros(pad + (64,), np.int32) for pad, _ in shapes]
  for scan in scans:
    decode_scan(b, info, scan, grids, shapes)
  return grids


def decode(b):
  """cv2.imdecode(b, cv2.IMREAD_COLOR) -> uint8 [H, W, 3] BGR, of a sequential or progressive
  file.  Unsupported for files outside the supported set, CorruptData for bad entropy data."""
  b = bytes(b)
  info, scans = parse(b)
  if scans is None:
    return D.decode(b)
  grids = coefficients(b, info, scans)
  planes = []
  for ci, (c, grid) in enumerate(zip(info.comps, grids)):
    q = info.qt.get(ci, np.zeros(64, np.uint16))
    px = D.idct_islow(grid, q)
    bh, bw = grid.shape[:2]
    plane = px.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)
    planes.append(plane[:-(-info.height * c.v // info.vmax), :-(-info.width * c.h // info.hmax)])
  H, W = info.height, info.width
  if len(planes) == 1:
    bgr = np.repeat(planes[0][:H, :W, None], 3, axis=2)
  else:
    c0 = info.comps[0]
    bgr = D.ycc_to_bgr(planes[0][:H, :W], D.upsample(planes[1], c0.h, c0.v, H, W),
                       D.upsample(planes[2], c0.h, c0.v, H, W))
  return np.ascontiguousarray(D.orient(bgr, info.orientation))
