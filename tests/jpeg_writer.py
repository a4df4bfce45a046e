"""A baseline JPEG writer for the decoder's tests: it writes a file from the quantized coefficients
of another (oracle.jpeg_decode.decode_coefficients), so it transcodes.  The coefficients, the
sampling and the dequantized values stay as they are and only the coding changes, so every file it
writes decodes to the same pixels as its source.  It writes what other encoders write and cv2's
never does: Huffman and quantization tables on any selector, tables built other ways (Annex K,
optimal from the file's own counts, skewed onto 15- and 16-bit codes, all 256 symbols), one
table per segment or all in one, tables defined twice, SOF1, restart intervals of any length with
fill bytes before RSTn markers and 0-bit padding, extra APPn and COM segments, fill bytes between
segments, and the scan's components in another order."""
import numpy as np

from oracle import jpeg as E
from oracle import jpeg_decode as D

# Annex K.3: (bits, vals) of the typical Huffman tables, as the encoder's oracle writes them
DC_LUMA = (E.DC_LUMA_BITS, E.DC_VALS)
DC_CHROMA = (E.DC_CHROMA_BITS, E.DC_VALS)
AC_LUMA = (E.AC_LUMA_BITS, E.AC_LUMA_VALS)
AC_CHROMA = (E.AC_CHROMA_BITS, E.AC_CHROMA_VALS)


def segment(marker, body):
  return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, 'big') + bytes(body)


def source(f):
  """A file -> (Info, coefficient grids) for write()."""
  info = D.parse(f)
  return info, D.decode_coefficients(f, info)


# ---- Huffman tables --------------------------------------------------------------------------------
def optimal_table(freq):
  """jpeg_gen_optimal_table (JPEG Annex K.2, with libjpeg's tie-breaking and reserved all-ones
  code): {symbol: count} -> (bits[16], vals), lengths limited to 16 bits."""
  f = [0] * 257
  for s, c in freq.items():
    f[s] = c
  f[256] = 1
  size, others = [0] * 257, [-1] * 257
  while True:
    c1 = c2 = -1
    v = None
    for i in range(257):
      if f[i] and (v is None or f[i] <= v):
        v, c1 = f[i], i
    v = None
    for i in range(257):
      if f[i] and i != c1 and (v is None or f[i] <= v):
        v, c2 = f[i], i
    if c2 < 0:
      break
    f[c1] += f[c2]
    f[c2] = 0
    size[c1] += 1
    while others[c1] >= 0:
      c1 = others[c1]
      size[c1] += 1
    others[c1] = c2
    size[c2] += 1
    while others[c2] >= 0:
      c2 = others[c2]
      size[c2] += 1
  bits = [0] * 33
  for s in size:
    if s:
      bits[s] += 1
  for i in range(32, 16, -1):
    while bits[i] > 0:
      j = i - 2
      while bits[j] == 0:
        j -= 1
      bits[i] -= 2
      bits[i - 1] += 1
      bits[j + 1] += 2
      bits[j] -= 1
  i = 16
  while bits[i] == 0:
    i -= 1
  bits[i] -= 1                                          # the reserved code
  vals = [s for ln in range(1, 33) for s in range(256) if size[s] == ln]
  return bits[1:17], vals


def lengths_table(lengths):
  """[(symbol, code length)] -> (bits[16], vals) in canonical order."""
  bits = [0] * 16
  for _, ln in lengths:
    bits[ln - 1] += 1
  return bits, [s for s, _ in sorted(lengths, key=lambda e: e[1])]


def skewed_table(freq):
  """A valid table whose 16- and 15-bit codes are the two most used symbols, the rest at one
  length short enough to leave room."""
  used = sorted(freq, key=lambda s: (-freq[s], s))
  rest = used[2:]
  m = max(2, len(rest).bit_length() + 1)
  return lengths_table([(used[0], 16)] + [(s, 15) for s in used[1:2]] + [(s, m) for s in rest])


def full_table(freq, dc):
  """A table listing every symbol a table of its class may hold (DC: 0..15; AC: all 256 byte
  values, the 162 the standard uses and 94 no 8-bit encoder writes), used ones first; AC codes run
  from 7 to 16 bits."""
  order = sorted(range(16 if dc else 256), key=lambda s: (-freq.get(s, 0), s))
  if dc:
    return lengths_table([(s, 4 if k < 8 else 5) for k, s in enumerate(order)])
  ln = (7,) * 64 + (8,) * 64 + (10,) * 64 + (16,) * 64
  return lengths_table(list(zip(order, ln)))


def annexk_table(dc, luma):
  return (DC_LUMA if luma else DC_CHROMA) if dc else (AC_LUMA if luma else AC_CHROMA)


def codes(bits, vals):
  """Canonical Huffman codes: symbol -> (code, length)."""
  out, code, k = {}, 0, 0
  for ln in range(1, 17):
    for _ in range(bits[ln - 1]):
      out[vals[k]] = (code, ln)
      code += 1
      k += 1
    code <<= 1
  return out


# ---- the scan ------------------------------------------------------------------------------------
def _category(v):
  a = abs(int(v))
  return a.bit_length(), (v if v >= 0 else v + (1 << a.bit_length()) - 1)


def block_symbols(blk, pred):
  """[(is_ac, symbol, extra bits, extra length)] of one block (natural order), DC against pred."""
  zz = blk[D.ZIGZAG]
  s, e = _category(int(zz[0]) - pred)
  out = [(0, s, e, s)]
  run = 0
  last = np.flatnonzero(zz[1:])
  last = last[-1] + 1 if len(last) else 0
  for k in range(1, last + 1):
    v = int(zz[k])
    if v == 0:
      run += 1
      continue
    while run > 15:
      out.append((1, 0xF0, 0, 0))
      run -= 16
    s, e = _category(v)
    out.append((1, run << 4 | s, e, s))
    run = 0
  if last < 63:
    out.append((1, 0x00, 0, 0))
  return out


class BitWriter:
  def __init__(self):
    self.acc, self.n, self.out = 0, 0, bytearray()

  def put(self, v, n):
    self.acc = (self.acc << n) | v
    self.n += n
    while self.n >= 8:
      self.n -= 8
      b = (self.acc >> self.n) & 0xFF
      self.out += b'\xff\x00' if b == 0xFF else bytes([b])
    self.acc &= (1 << self.n) - 1

  def pad(self, bit):
    if self.n:
      k = 8 - self.n
      self.put((1 << k) - 1 if bit else 0, k)


def mcu_blocks(info, grids, order):
  """Per MCU, [(component index, block)] in scan order `order` (indices into info.comps)."""
  comps = info.comps
  if len(comps) == 1:
    g = grids[0]
    for my in range(g.shape[0]):
      for mx in range(g.shape[1]):
        yield [(0, g[my, mx])]
    return
  hmax, vmax = max(c.h for c in comps), max(c.v for c in comps)
  mcols = -(-info.width // (8 * hmax))
  mrows = -(-info.height // (8 * vmax))
  for my in range(mrows):
    for mx in range(mcols):
      yield [(ci, grids[ci][my * comps[ci].v + v, mx * comps[ci].h + h])
             for ci in order for v in range(comps[ci].v) for h in range(comps[ci].h)]


def scan_symbols(info, grids, order, restart):
  """Per restart interval, per block: (component index, its symbols)."""
  intervals, cur, pred = [], [], {}
  for m, mcu in enumerate(mcu_blocks(info, grids, order)):
    if restart and m % restart == 0 and m:
      intervals.append(cur)
      cur, pred = [], {}
    for ci, blk in mcu:
      cur.append((ci, block_symbols(blk, pred.get(ci, 0))))
      pred[ci] = int(blk[0])
  intervals.append(cur)
  return intervals


# ---- the file ------------------------------------------------------------------------------------
def exif(orientation=None, little_endian=False, thumbnail=None):
  """An APP1 Exif segment: IFD0 with an Orientation SHORT (None: no entry), and with a thumbnail
  an IFD1 pointing at the JPEG bytes that follow it inside the segment."""
  e = 'little' if little_endian else 'big'
  r = lambda v, n: v.to_bytes(n, e)
  ifd0 = [] if orientation is None else [r(0x0112, 2) + r(3, 2) + r(1, 4) + r(orientation, 2) + bytes(2)]
  ifd1_at = 8 + 2 + 12 * len(ifd0) + 4
  t = (b'II' if little_endian else b'MM') + r(42, 2) + r(8, 4) + r(len(ifd0), 2) + b''.join(ifd0)
  if thumbnail is None:
    return segment(0xE1, b'Exif\x00\x00' + t + r(0, 4))
  data_at = ifd1_at + 2 + 2 * 12 + 4
  ifd1 = r(2, 2) + r(0x0201, 2) + r(4, 2) + r(1, 4) + r(data_at, 4) \
      + r(0x0202, 2) + r(4, 2) + r(1, 4) + r(len(thumbnail), 4) + r(0, 4)
  return segment(0xE1, b'Exif\x00\x00' + t + r(ifd1_at, 4) + ifd1 + bytes(thumbnail))


XMP = segment(0xE1, b'http://ns.adobe.com/xap/1.0/\x00<?xpacket begin=""?><x:xmpmeta '
              b'xmlns:x="adobe:ns:meta/"><tiff:Orientation>6</tiff:Orientation></x:xmpmeta>')
ICC = segment(0xE2, b'ICC_PROFILE\x00\x01\x01' + bytes(range(256)) * 2)
COM = segment(0xFE, b'written by a test encoder \xff\xd9\xff\xd8')


def write(info, grids, huff=None, tables='annexk', quant=None, halve_cr=False, pack='separate',
          redefine=False, sof=0xC0, restart=0, rst_fill=0, pad_bit=1, before=(), after_sof=(),
          fill=0, jfif=True, order=None, sampling=None):
  """A baseline file of `grids` (the quantized coefficients of info's components).

  huff      per component (DC table, AC table) selectors; default: luma 0, chroma 1
  tables    'annexk' (luma tables for those luma uses), 'optimal', 'skewed' or 'full'
  quant     per component quantization table id; a component's table is its source table
  halve_cr  Cr's table holds the source's entries halved where they are even, its coefficients
            doubled there: the same dequantized values from another table
  pack      'separate' (one table per DHT / DQT) or 'joint' (all in one segment)
  redefine  every table is first defined wrongly, then again before SOS
  restart   the restart interval in MCUs (0: none); rst_fill 0xFF fill bytes before every other
            RSTn; pad_bit the bit that pads each interval's last byte
  before    segments after SOI (after the JFIF APP0 when jfif); after_sof segments after SOF
  fill      0xFF fill bytes before each marker of the header
  order     the scan's component order (default: the frame's)
  sampling  per component (h, v) written in SOF, for grids laid out for it"""
  comps = info.comps
  nc = len(comps)
  order = list(range(nc)) if order is None else list(order)
  huff = huff or [(0, 0)] + [(1, 1)] * (nc - 1)
  quant = quant or [c.tq for c in comps]
  sampling = sampling or [(c.h, c.v) for c in comps]
  grids = [g.copy() for g in grids]
  qt = {}
  for ci, c in enumerate(comps):
    q = info.qt[c.tq].astype(np.int64)
    if halve_cr and ci == 2:
      even = (q % 2 == 0) & (q > 0)
      q = np.where(even, q // 2, q)
      grids[ci] = np.where(even, grids[ci] * 2, grids[ci])
    assert quant[ci] not in qt or np.array_equal(qt[quant[ci]], q), 'one id, two tables'
    qt[quant[ci]] = q
  info = D.Info(info.height, info.width,
                [D.Component(c.cid, h, v, quant[ci]) for ci, (c, (h, v)) in enumerate(zip(comps, sampling))],
                info.qt, info.dc, info.ac)
  intervals = scan_symbols(info, grids, order, restart)
  freq = {}
  for iv in intervals:
    for ci, syms in iv:
      for is_ac, s, _, _ in syms:
        key = (is_ac, huff[ci][is_ac])
        freq.setdefault(key, {})
        freq[key][s] = freq[key].get(s, 0) + 1
  tabs = {}
  for (is_ac, tid), fr in sorted(freq.items()):
    if tables == 'annexk':
      tabs[is_ac, tid] = annexk_table(not is_ac, huff[0][is_ac] == tid)
    elif tables == 'optimal':
      tabs[is_ac, tid] = optimal_table(fr)
    elif tables == 'skewed':
      tabs[is_ac, tid] = skewed_table(fr)
    else:
      tabs[is_ac, tid] = full_table(fr, not is_ac)
  enc = {k: codes(*t) for k, t in tabs.items()}
  bw = BitWriter()
  for r, iv in enumerate(intervals):
    for ci, syms in iv:
      for is_ac, s, e, n in syms:
        code, ln = enc[is_ac, huff[ci][is_ac]][s]
        bw.put(code, ln)
        if n:
          bw.put(e, n)
    bw.pad(pad_bit)
    if r + 1 < len(intervals):
      bw.out += b'\xff' * (rst_fill if r % 2 == 0 else 0) + bytes([0xFF, 0xD0 + r % 8])

  def dqt(items):
    return b''.join(bytes([tid]) + bytes(np.asarray(q)[D.ZIGZAG].astype(np.uint8)) for tid, q in items)

  def dht(items):
    return b''.join(bytes([is_ac << 4 | tid]) + bytes(bits) + bytes(vals) for (is_ac, tid), (bits, vals) in items)

  def packed(kind, items):
    make, marker = (dqt, 0xDB) if kind == 'q' else (dht, 0xC4)
    if pack == 'joint':
      return [(marker, make(items))]
    return [(marker, make([it])) for it in items]

  qitems = sorted(qt.items())
  hitems = sorted(tabs.items())
  segs = []
  if jfif:
    segs.append((0xE0, b'JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00'))
  segs += [(None, s) for s in before]
  if redefine:
    segs += packed('q', [(tid, np.full(64, 1 + tid)) for tid, _ in qitems])
    segs += packed('h', [(k, annexk_table(not k[0], False) if tables != 'annexk' else full_table({}, not k[0]))
                         for k, _ in hitems])
  segs += packed('q', qitems)
  body = bytes([8]) + info.height.to_bytes(2, 'big') + info.width.to_bytes(2, 'big') + bytes([nc]) \
      + b''.join(bytes([c.cid, h << 4 | v, quant[ci]]) for ci, (c, (h, v)) in enumerate(zip(comps, sampling)))
  segs.append((sof, body))
  segs += [(None, s) for s in after_sof]
  segs += packed('h', hitems)
  if restart:
    segs.append((0xDD, restart.to_bytes(2, 'big')))
  sos = bytes([nc]) + b''.join(bytes([comps[ci].cid, huff[ci][0] << 4 | huff[ci][1]]) for ci in order) \
      + bytes([0, 63, 0])
  segs.append((0xDA, sos))
  out = bytearray(b'\xff\xd8')
  for m, b in segs:
    out += b'\xff' * fill
    out += b if m is None else segment(m, b)
  return bytes(out + bw.out + b'\xff' * fill + b'\xff\xd9')
