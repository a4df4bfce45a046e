"""CPU restatement of cv2.imencode('.jpg', ..., [cv2.IMWRITE_JPEG_PROGRESSIVE, 1, ...]): libjpeg-
turbo's progressive Huffman writer with jpeg_simple_progression's ten scans, over the quantized
coefficients oracle/jpeg_params.py computes (a progressive file holds exactly the baseline file's
coefficients).  PINNED bitwise against the installed cv2 (tests/test_oracle_jpeg_progressive.py).

encode(bgr, quality, sampling=..., restart_interval=..., luma_quality=..., chroma_quality=...,
causes=None) is what cv2 writes with IMWRITE_JPEG_PROGRESSIVE and those parameters (optimize has no
effect: progressive files always carry each scan's optimal tables).

  file      SOI, JFIF APP0, DQT x 2, SOF2 (SOF0's contents), then per scan its DHT segments, (first
            scan only, with an interval) DRI, SOS and the scan's entropy-coded data, then EOI
  scans     SCANS: (components, Ss, Se, Ah, Al).  Scans 1 and 7 (the DC scans) are interleaved
            over the MCUs as the baseline scan is, dummy blocks included (a dummy block's DC is the
            last real block's before it in its MCU).  The others cover one component's
            ceil(w_c / 8) x ceil(h_c / 8) blocks in raster order, and an MCU there is one block
  tables    every Huffman scan gets its own optimal tables (jpeg_gen_optimal_table of the scan's
            symbol counts): DC luma then DC chroma before scan 1, the component's AC table before
            each AC scan, none before scan 7.  SOS names the table each component uses, 0 where
            the scan uses none
  DC first  (dc >> Al) as an arithmetic shift, coded as the baseline DC difference against the
            component's last one (0 at the scan's and each interval's start)
  DC refine bit Al of each DC, one raw bit per block
  AC first  the band's |v| >> Al (sign restored as the baseline codes it); a block whose band ends in
            zeros adds 1 to EOBRUN instead of an EOB symbol
  AC refine coefficients with |v| >> Al == 1 are newly nonzero (run/1 symbol, 1 sign bit: 1 for
            positive); larger ones are already known and get one correction bit (bit Al of |v|),
            kept in the block until its next symbol or, after its last, buffered as BE bits behind
            the pending EOBRUN; runs count only the coefficients still zero, and ZRLs after the last
            newly nonzero one fold into the EOB run
  EOBRUN    emitted as symbol (nbits(EOBRUN) - 1) << 4 and its low bits, then the buffered
            correction bits, when (CAUSES) the next symbol comes, EOBRUN reaches 0x7FFF, BE exceeds
            MAX_CORR_BITS - 64 + 1 = 937 (refinement only), a restart marker comes, or the scan ends
  restart   with an interval every scan is cut into intervals of that many MCUs (blocks, in the AC
            scans); each interval is padded to a byte with 1-bits, RSTn (n from 0 in each scan)
            sits between intervals, and the DC predictors, EOBRUN and BE restart at 0
"""
import numpy as np

from oracle.jpeg import ZIGZAG, _nbits, _pack, huffman_codes, quant_tables
from oracle.jpeg_params import coefficients, optimal_table, resolve

# jpeg_simple_progression for YCbCr: (component indices, Ss, Se, Ah, Al)
SCANS = [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((2,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1),
         ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), ((2,), 1, 63, 1, 0),
         ((1,), 1, 63, 1, 0), ((0,), 1, 63, 1, 0)]
CAUSES = ('next_symbol', 'cap', 'correction_bits', 'restart', 'end_of_scan')
EOBRUN_MAX = 0x7FFF
BE_MAX = 1000 - 64 + 1         # MAX_CORR_BITS - DCTSIZE2 + 1


def _seg(marker, body):
  return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, 'big') + bytes(body)


def _dht(cls_id, table):
  bits, vals = table
  return _seg(0xC4, bytes([cls_id]) + bytes(bits) + bytes(vals))


def _units(blocks, comp, h, w, hs, vs, scan):
  """(the coefficient rows [U, 64] the scan codes, in its order; their components, for the DC
  scans): the interleaved DC scans run over every block of the MCUs, the AC scans over one
  component's blocks in raster order."""
  comps, ss = scan[0], scan[1]
  if ss == 0:
    return blocks, comp
  c = comps[0]
  mr, mc = -(-h // (8 * vs)), -(-w // (8 * hs))
  if c:                                               # chroma: one block per MCU, all of them
    return blocks[comp == c], None
  y = blocks[comp == 0].reshape(mr, mc, vs, hs, 64).transpose(0, 2, 1, 3, 4).reshape(vs * mr, hs * mc, 64)
  return y[:-(-h // 8), :-(-w // 8)].reshape(-1, 64), None


def _scan_items(rows, comp, dummy, per, scan, interval, counts):
  """The scan's coded items per interval: ('s', table, symbol, value, nbits) for a Huffman symbol
  and its extra bits, ('r', value, nbits) for raw bits.  Table 0 / 1 is the DC luma / chroma table
  of an interleaved scan, 0 the AC table of the others."""
  comps, ss, se, ah, al = scan
  n = len(rows)
  per_interval = interval * (per if ss == 0 else 1)
  out = [[]]

  def new_interval(k):
    return per_interval and k and k % per_interval == 0

  if ss == 0:
    dc = rows[:, 0].copy()
    # a dummy block's DC is the last real block's before it (the MCU's first luma block is real)
    real = np.nonzero(~dummy)[0]
    dc[dummy] = dc[real[np.searchsorted(real, np.nonzero(dummy)[0]) - 1]]
    last = [0, 0, 0]
    for k in range(n):
      if new_interval(k):
        out.append([])
        last = [0, 0, 0]
      c = int(comp[k])
      if ah == 0:
        v = int(dc[k]) >> al
        d = v - last[c]
        last[c] = v
        nb = int(_nbits(np.int64(d)))
        out[-1].append(('s', min(c, 1), nb, d - 1 if d < 0 else d, nb))
      else:
        out[-1].append(('r', (int(dc[k]) >> al) & 1, 1))
    return out

  band = rows[:, ss:se + 1]
  eobrun, be = 0, []                                  # be: the buffered correction bits

  def flush(cause):
    nonlocal eobrun, be
    if eobrun:
      nb = eobrun.bit_length() - 1
      out[-1].append(('s', 0, nb << 4, eobrun, nb))
      out[-1].extend(('r', b, 1) for b in be)
      counts[cause] += 1
      eobrun, be = 0, []

  for k in range(n):
    if new_interval(k):
      flush('restart')
      out.append([])
    a = np.abs(band[k]) >> al
    if ah == 0:
      r = 0
      for j in np.nonzero(a)[0] if a.any() else ():
        flush('next_symbol')
        run = j - r
        while run > 15:
          out[-1].append(('s', 0, 0xF0, 0, 0))
          run -= 16
        t = int(a[j])
        nb = t.bit_length()
        out[-1].append(('s', 0, (run << 4) | nb, ~t if band[k, j] < 0 else t, nb))
        r = j + 1
      if r < len(a):
        eobrun += 1
        if eobrun == EOBRUN_MAX:
          flush('cap')
      continue
    ones = np.nonzero(a == 1)[0]
    eob = ones[-1] if len(ones) else -1
    r, br = 0, []
    for j in range(len(a)):
      t = int(a[j])
      if t == 0:
        r += 1
        continue
      while r > 15 and j <= eob:
        flush('next_symbol')
        out[-1].append(('s', 0, 0xF0, 0, 0))
        r -= 16
        out[-1].extend(('r', b, 1) for b in br)
        br = []
      if t > 1:
        br.append(t & 1)
        continue
      flush('next_symbol')
      out[-1].append(('s', 0, (r << 4) | 1, int(band[k, j] >= 0), 1))
      out[-1].extend(('r', b, 1) for b in br)
      br, r = [], 0
    if r or br:
      eobrun += 1
      be += br
      if eobrun == EOBRUN_MAX:
        flush('cap')
      elif len(be) > BE_MAX:
        flush('correction_bits')
  flush('end_of_scan')
  return out


def encode(bgr, quality=95, *, sampling='420', optimize=False, restart_interval=0,
           luma_quality=None, chroma_quality=None, causes=None):
  """The bytes cv2.imencode('.jpg', bgr, cv2_params(..., progressive=True)) writes for a uint8 BGR
  image [h, w, 3].  `causes`, a dict, gets the number of EOBRUN flushes of each of CAUSES added.
  Values cv2 would clamp and sides it refuses raise ValueError."""
  del optimize                                        # progressive tables are always optimal
  bgr = np.asarray(bgr)
  if bgr.dtype != np.uint8 or bgr.ndim != 3 or bgr.shape[2] != 3 or min(bgr.shape[:2]) < 1:
    raise ValueError('need a non-empty uint8 [h, w, 3] image, got %s %r' % (bgr.dtype, bgr.shape))
  h, w = bgr.shape[:2]
  if h > 65500 or w > 65500:
    raise ValueError('JPEG sizes are at most 65500, got %dx%d' % (w, h))
  if not 0 <= restart_interval <= 65535:
    raise ValueError('restart_interval must be in [0, 65535], got %r' % (restart_interval,))
  lq, cq, (hs, vs) = resolve(quality, sampling, luma_quality, chroma_quality)
  blocks, comp, dummy, per = coefficients(bgr, lq, cq, hs, vs)
  counts = dict.fromkeys(CAUSES, 0)

  out = bytes([0xFF, 0xD8]) + _seg(0xE0, b'JFIF\x00' + bytes([1, 1, 0, 0, 1, 0, 1, 0, 0]))
  for i, q in enumerate((quant_tables(lq)[0], quant_tables(cq)[1])):
    out += _seg(0xDB, bytes([i]) + bytes(int(v) for v in q[ZIGZAG]))
  out += _seg(0xC2, bytes([8, h >> 8, h & 255, w >> 8, w & 255, 3, 1, hs << 4 | vs, 0, 2, 0x11, 1,
                           3, 0x11, 1]))
  for si, scan in enumerate(SCANS):
    comps, ss, se, ah, al = scan
    rows, ucomp = _units(blocks, comp, h, w, hs, vs, scan)
    items = _scan_items(rows, ucomp, dummy, per, scan, restart_interval, counts)
    coded = ss != 0 or ah == 0                        # every scan but the DC refinement
    codes = {}
    if coded:
      flat = [it for iv in items for it in iv if it[0] == 's']
      tabs = sorted({it[1] for it in flat})
      for t in tabs:
        freq = {}
        for it in flat:
          if it[1] == t:
            freq[it[2]] = freq.get(it[2], 0) + 1
        table = optimal_table(freq)
        codes[t] = huffman_codes(*table)
        chroma = t == 1 or (ss and comps[0] > 0)
        out += _dht((0x10 if ss else 0x00) | int(chroma), table)
    if si == 0 and restart_interval:
      out += _seg(0xDD, restart_interval.to_bytes(2, 'big'))
    sel = [0 if ss or ah else (0x10 if c else 0) for c in comps]
    if ss:
      sel = [1 if comps[0] else 0]
    body = [len(comps)]
    for c, s in zip(comps, sel):
      body += [c + 1, s]
    out += _seg(0xDA, bytes(body + [ss, se, ah << 4 | al]))
    for i, iv in enumerate(items):
      if i:
        out += bytes([0xFF, 0xD0 + (i - 1) % 8])
      vals, lens = [], []
      for it in iv:
        if it[0] == 's':
          code, clen = codes[it[1]]
          vals.append((int(code[it[2]]) << it[4]) | (it[3] & ((1 << it[4]) - 1)))
          lens.append(int(clen[it[2]]) + it[4])
        else:
          vals.append(it[1])
          lens.append(it[2])
      out += _pack(np.array(vals, np.int64), np.array(lens, np.int64))
  if causes is not None:
    for k, v in counts.items():
      causes[k] = causes.get(k, 0) + v
  return out + bytes([0xFF, 0xD9])
