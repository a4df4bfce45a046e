"""CPU restatement of the PNG encoder cv2.imencode('.png', bgr) runs at its defaults (libpng 1.6
with the system zlib 1.2.11) — test infrastructure, like the rest of oracle/.  No zlib call: every
step is written out here, and tests/test_oracle_png.py pins encode() bitwise against the installed
cv2 and the deflate body against zlib.compressobj(1, DEFLATED, 15, 8, Z_RLE).

  chunks    signature, IHDR (8-bit RGB, colour type 2, no interlace), IDAT..., IEND; nothing else
  filter    each row is one filter byte and its 3 w R, G, B bytes (libpng swaps cv2's B, G, R):
            SUB (1), x[i] - x[i - 3] mod 256 with the first pixel unchanged, except for 1-pixel-wide
            images, where libpng drops SUB and writes NONE (0)
  parse     zlib level 1 with strategy Z_RLE is deflate_rle: position p > 0 starts a match when
            bytes p-1 .. p+2 are equal, of the bytes from p equal to byte p-1, at most 258;
            otherwise p is a literal.  Per maximal run of L equal bytes: one literal, then while
            the R = L - 1 bytes left number 3 or more a match of min(R, 258), then R literals
  blocks    a block every 16383 symbols (lit_bufsize - 1 at memLevel 8), flushed non-final; the
            rest, possibly nothing, is the final block
  trees     _tr_flush_block: build_tree (heap with depth tie-break, two codes forced, gen_bitlen's
            repair at 15 bits), scan_tree / build_bl_tree; stored if stored_len + 4 <= opt_lenb
            (opt_lenb the smaller of the dynamic and static sizes), else static if the static size
            is that smaller one, else dynamic
  zlib      header 78 01, its window field lowered for small images (libpng's deflate window choice
            and optimize_cmf), then the deflate body and the big-endian Adler-32 of the filtered
            stream
  IDAT      the zlib stream in 8192-byte chunks, the last one shorter or full: a stream of a
            multiple of 8192 bytes gets no empty IDAT after its last full one

zlib stores a block only while its bytes are in the window (block_start >= 0).  That holds for every
block this parse makes that could be stored, so no window is modelled: a stored block needs
8 (stored_len + 4) <= static_len + 10, and at most 9 bits per literal and 18 per match (8-bit
length code, 5 extra bits, 5-bit distance code) with 8 bits per byte and 3 bytes per match allow
only 6 matches <= literals and so stored_len <= 9/8 * 14043 + 18/8 * 2340 < 21065 bytes, while a
block reaches before the window only once 32507 bytes of it have been read (the 32 KiB window
slides by 32768 when strstart reaches 65274; smaller windows, chosen for images that fit them,
never slide).
"""
import struct

import numpy as np

SIGNATURE = b'\x89PNG\r\n\x1a\n'
BLOCK_SYMBOLS = 16383            # lit_bufsize - 1 at memLevel 8
IDAT_BYTES = 8192                # libpng's zbuffer size
MAX_SIDE = 1000000               # libpng's PNG_USER_WIDTH_MAX / PNG_USER_HEIGHT_MAX
MAX_BITS, MAX_BL_BITS = 15, 7
L_CODES, D_CODES, BL_CODES = 286, 30, 19
END_BLOCK = 256

EXTRA_LBITS = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
BASE_LENGTH = [0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 32, 40, 48, 56, 64, 80, 96,
               112, 128, 160, 192, 224, 255]
EXTRA_DBITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11,
               12, 12, 13, 13]
EXTRA_BLBITS = [0] * 16 + [2, 3, 7]
BL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
REP_3_6, REPZ_3_10, REPZ_11_138 = 16, 17, 18


def length_code(lc):
  """Code index (0..28, symbol 257 + index) of match length lc + 3, as zlib's _length_code."""
  lc = np.asarray(lc, np.int64)
  code = np.searchsorted(np.array(BASE_LENGTH[:28]), lc, side='right') - 1
  return np.where(lc == 255, 28, code)


def bi_reverse(code, n):
  out = 0
  for _ in range(n):
    out = (out << 1) | (code & 1)
    code >>= 1
  return out


def gen_codes(lens):
  """Bit-reversed canonical codes of code lengths `lens` (zlib's gen_codes)."""
  bl_count = [0] * (MAX_BITS + 1)
  for l in lens:
    if l:
      bl_count[l] += 1
  next_code, code = [0] * (MAX_BITS + 1), 0
  for bits in range(1, MAX_BITS + 1):
    code = (code + bl_count[bits - 1]) << 1
    next_code[bits] = code
  codes = [0] * len(lens)
  for n, l in enumerate(lens):
    if l:
      codes[n] = bi_reverse(next_code[l], l)
      next_code[l] += 1
  return codes


STATIC_LLEN = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
STATIC_LCODE = gen_codes(STATIC_LLEN)
STATIC_DLEN = [5] * D_CODES
STATIC_DCODE = [bi_reverse(n, 5) for n in range(D_CODES)]


def build_tree(freq, static_len, extra, base, max_length, info=None):
  """zlib's build_tree + gen_bitlen on symbol frequencies `freq` (a list, changed where codes are
  forced).  -> (lens, max_code, opt_len, static_len); static_len is 0 without a static tree.
  info['repaired'] counts the trees whose lengths gen_bitlen repaired to max_length."""
  elems = len(freq)
  heap_size = 2 * L_CODES + 1
  nodes = 2 * elems + 1
  f = list(freq) + [0] * (nodes - elems)
  depth = [0] * nodes
  dad = [0] * nodes
  heap = [0] * heap_size
  heap_len, heap_max, max_code = 0, heap_size, -1
  opt, stat = 0, 0
  for n in range(elems):
    if f[n]:
      heap_len += 1
      heap[heap_len] = max_code = n
  while heap_len < 2:                       # at least two codes: force a frequency of 1
    if max_code < 2:
      max_code += 1
      node = max_code
    else:
      node = 0
    heap_len += 1
    heap[heap_len] = node
    f[node] = 1
    opt -= 1
    if static_len:
      stat -= static_len[node]

  def smaller(n, m):
    return f[n] < f[m] or (f[n] == f[m] and depth[n] <= depth[m])

  def down(k):
    v = heap[k]
    j = k << 1
    while j <= heap_len:
      if j < heap_len and smaller(heap[j + 1], heap[j]):
        j += 1
      if smaller(v, heap[j]):
        break
      heap[k] = heap[j]
      k = j
      j <<= 1
    heap[k] = v

  for k in range(heap_len // 2, 0, -1):
    down(k)
  node = elems
  while True:
    n = heap[1]
    heap[1] = heap[heap_len]
    heap_len -= 1
    down(1)
    m = heap[1]
    heap_max -= 1
    heap[heap_max] = n
    heap_max -= 1
    heap[heap_max] = m
    f[node] = f[n] + f[m]
    depth[node] = max(depth[n], depth[m]) + 1
    dad[n] = dad[m] = node
    heap[1] = node
    node += 1
    down(1)
    if heap_len < 2:
      break
  heap_max -= 1
  heap[heap_max] = heap[1]

  # gen_bitlen
  ln = [0] * nodes
  bl_count = [0] * (MAX_BITS + 1)
  overflow = 0
  ln[heap[heap_max]] = 0
  for h in range(heap_max + 1, heap_size):
    n = heap[h]
    bits = ln[dad[n]] + 1
    if bits > max_length:
      bits = max_length
      overflow += 1
    ln[n] = bits
    if n > max_code:
      continue
    bl_count[bits] += 1
    xbits = extra[n - base] if n >= base else 0
    opt += f[n] * (bits + xbits)
    if static_len:
      stat += f[n] * (static_len[n] + xbits)
  if overflow:
    if info is not None:
      info['repaired'] = info.get('repaired', 0) + 1
    while overflow > 0:
      bits = max_length - 1
      while bl_count[bits] == 0:
        bits -= 1
      bl_count[bits] -= 1
      bl_count[bits + 1] += 2
      bl_count[max_length] -= 1
      overflow -= 2
    h = heap_size
    for bits in range(max_length, 0, -1):
      n = bl_count[bits]
      while n:
        h -= 1
        m = heap[h]
        if m > max_code:
          continue
        if ln[m] != bits:
          opt += (bits - ln[m]) * f[m]
          ln[m] = bits
        n -= 1
  lens = [ln[n] if n <= max_code and f[n] else 0 for n in range(elems)]
  return lens, max_code, opt, stat


def _tree_runs(lens, max_code):
  """scan_tree / send_tree's walk of code lengths lens[0..max_code]: a list of (bl symbol, extra
  value, extra bits)."""
  out = []
  prevlen, nextlen, count = -1, lens[0], 0
  max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
  for n in range(max_code + 1):
    curlen = nextlen
    nextlen = lens[n + 1] if n + 1 <= max_code else -1      # the 0xffff guard
    count += 1
    if count < max_count and curlen == nextlen:
      continue
    if count < min_count:
      out += [(curlen, 0, 0)] * count
    elif curlen != 0:
      if curlen != prevlen:
        out.append((curlen, 0, 0))
        count -= 1
      out.append((REP_3_6, count - 3, 2))
    elif count <= 10:
      out.append((REPZ_3_10, count - 3, 3))
    else:
      out.append((REPZ_11_138, count - 11, 7))
    count, prevlen = 0, curlen
    if nextlen == 0:
      max_count, min_count = 138, 3
    elif curlen == nextlen:
      max_count, min_count = 6, 3
    else:
      max_count, min_count = 7, 4
  return out


def filter_rows(bgr):
  """The filtered stream of a uint8 BGR [h, w, 3] image: per row the filter byte, then SUB of its
  R, G, B bytes (NONE for w == 1)."""
  h, w = bgr.shape[:2]
  rgb = np.ascontiguousarray(bgr[:, :, ::-1]).reshape(h, 3 * w)
  out = np.empty((h, 3 * w + 1), np.uint8)
  out[:, 0] = 1 if w > 1 else 0
  out[:, 1:4] = rgb[:, :3]
  out[:, 4:] = rgb[:, 3:] - rgb[:, :-3]
  return out.reshape(-1)


def parse(data):
  """deflate_rle's symbols of `data` (uint8): (pos, length) int64 arrays, length 1 for a literal
  and 3..258 for a distance-1 match starting at pos."""
  d = np.asarray(data, np.uint8)
  n = len(d)
  brk = np.ones(n, bool)
  brk[1:] = d[1:] != d[:-1]
  starts = np.flatnonzero(brk)
  ends = np.append(starts[1:], n)
  run = np.repeat(np.arange(len(starts)), ends - starts)
  p = np.arange(n, dtype=np.int64)
  o = p - starts[run]                       # offset in the run
  e = ends[run] - p                         # bytes from p to the run's end
  q = np.where(o > 0, (o - 1) % 258, 0)
  lit = (o == 0) | (e + q < 3)
  first = lit | (q == 0)
  pos = p[first]
  length = np.where(lit[first], 1, np.minimum(e[first], 258))
  return pos, length


def _flush_block(data, pos, length, start, end, last, out, bitpos, info):
  """_tr_flush_block of the symbols (pos, length) covering data[start:end]; appends (value, bits)
  pairs to out.  -> (bitpos after the block, kind) with kind 'stored', 'static' or 'dynamic'."""
  lit = length == 1
  lcode = np.where(lit, data[pos].astype(np.int64), 257 + length_code(length - 3))
  lfreq = np.bincount(lcode, minlength=L_CODES)[:L_CODES].tolist()
  lfreq[END_BLOCK] += 1
  dfreq = [int((~lit).sum())] + [0] * (D_CODES - 1)
  llen, lmax, lopt, lstat = build_tree(lfreq, STATIC_LLEN, EXTRA_LBITS, 257, MAX_BITS, info)
  dlen, dmax, dopt, dstat = build_tree(dfreq, STATIC_DLEN, EXTRA_DBITS, 0, MAX_BITS)
  runs = _tree_runs(llen, lmax) + _tree_runs(dlen, dmax)
  blfreq = np.bincount([r[0] for r in runs], minlength=BL_CODES).tolist()
  bllen, _, blopt, _ = build_tree(blfreq, None, EXTRA_BLBITS, 0, MAX_BL_BITS)
  max_blindex = BL_CODES - 1
  while max_blindex >= 3 and bllen[BL_ORDER[max_blindex]] == 0:
    max_blindex -= 1
  opt_len = lopt + dopt + blopt + 3 * (max_blindex + 1) + 14
  static_len = lstat + dstat
  opt_lenb, static_lenb = (opt_len + 3 + 7) >> 3, (static_len + 3 + 7) >> 3
  opt_lenb = min(opt_lenb, static_lenb)
  stored_len = end - start
  if stored_len + 4 <= opt_lenb:
    pad = (-(bitpos + 3)) % 8
    out.append(([last, 0, stored_len, stored_len ^ 0xFFFF], [3, pad, 16, 16]))
    out.append((data[start:end].astype(np.int64), np.full(stored_len, 8)))
    return bitpos + 3 + pad + 32 + 8 * stored_len, 'stored'
  if static_lenb == opt_lenb:
    lc, ll, dc, dl = STATIC_LCODE, STATIC_LLEN, STATIC_DCODE, STATIC_DLEN
    out.append(([2 + last], [3]))
    kind = 'static'
  else:
    lc, ll, dc, dl = gen_codes(llen), llen, gen_codes(dlen), dlen
    blc = gen_codes(bllen)
    vals = [4 + last, lmax + 1 - 257, dmax + 1 - 1, max_blindex + 1 - 4]
    bits = [3, 5, 5, 4]
    for r in range(max_blindex + 1):
      vals.append(bllen[BL_ORDER[r]])
      bits.append(3)
    for sym, xv, xb in runs:
      vals += [blc[sym], xv]
      bits += [bllen[sym], xb]
    out.append((vals, bits))
    kind = 'dynamic'
  lc, ll = np.array(lc, np.int64), np.array(ll, np.int64)
  # per symbol: its literal/length code, then a match's extra length bits and distance code
  code = lcode - 257
  xb = np.where(lit, 0, np.array(EXTRA_LBITS)[np.maximum(code, 0)])
  xv = np.where(lit, 0, length - 3 - np.array(BASE_LENGTH)[np.maximum(code, 0)])
  v = lc[lcode] | (xv << ll[lcode]) | np.where(lit, 0, dc[0] << (ll[lcode] + xb))
  b = ll[lcode] + xb + np.where(lit, 0, dl[0])
  out.append((np.append(v, lc[END_BLOCK]), np.append(b, ll[END_BLOCK])))
  return bitpos + 3 + (static_len if kind == 'static' else opt_len), kind


def _pack(pieces):
  """(value, bits) pairs, LSB first -> bytes, the last byte padded with zero bits."""
  vals = np.concatenate([np.asarray(v, np.int64) for v, _ in pieces])
  bits = np.concatenate([np.asarray(b, np.int64) for _, b in pieces])
  keep = bits > 0
  vals, bits = vals[keep], bits[keep]
  k = np.arange(32)
  mask = k[None, :] < bits[:, None]
  stream = ((vals[:, None] >> k[None, :]) & 1)[mask].astype(np.uint8)
  return np.packbits(stream, bitorder='little').tobytes()


def deflate_rle(data, info=None):
  """The raw deflate body zlib 1.2.11 writes for `data` at level 1 with Z_RLE (memLevel 8) in one
  Z_FINISH.  `info`, a dict, gets 'blocks' (each block's kind), 'symbols', 'matches',
  'repaired' (literal/length trees repaired at 15 bits) and 'parse' (parse's (pos, length))."""
  data = np.asarray(data, np.uint8)
  pos, length = parse(data)
  nsym = len(pos)
  ends = np.append(pos, len(data))
  out, bitpos, kinds = [], 0, []
  if info is not None:
    info['repaired'] = 0
  nblocks = nsym // BLOCK_SYMBOLS + 1
  for b in range(nblocks):
    s0, s1 = b * BLOCK_SYMBOLS, min((b + 1) * BLOCK_SYMBOLS, nsym)
    bitpos, kind = _flush_block(data, pos[s0:s1], length[s0:s1], int(ends[s0]), int(ends[s1]),
                                int(b == nblocks - 1), out, bitpos, info)
    kinds.append(kind)
  if info is not None:
    info['blocks'] = kinds
    info['symbols'] = nsym
    info['matches'] = int((length > 1).sum())
    info['parse'] = (pos, length)
  return _pack(out)


def adler32(data):
  d = np.asarray(data, np.uint8).astype(np.int64)
  n = len(d)
  a = (1 + int(d.sum())) % 65521
  b = (n + int((((n - np.arange(n)) % 65521) * d % 65521).sum())) % 65521
  return (b << 16) | a


def zlib_header(size):
  """The 2-byte zlib header libpng leaves for `size` bytes of filtered image data: zlib's header of
  the window libpng asks for (15 bits, less while size + 262 fits half of it; zlib takes 8 as 9),
  level 1 (FLEVEL 0), then optimize_cmf's lower window field where size fits it."""
  wbits = 15
  if size <= 16384:
    half = 1 << (wbits - 1)
    while size + 262 <= half:
      half >>= 1
      wbits -= 1
  wbits = max(wbits, 9)
  cmf = 8 | ((wbits - 8) << 4)
  flg = 31 - (cmf << 8) % 31
  if size <= 16384:
    cinfo = cmf >> 4
    half = 1 << (cinfo + 7)
    if size <= half:
      while True:
        half >>= 1
        cinfo -= 1
        if not (cinfo > 0 and size <= half):
          break
      cmf = 8 | (cinfo << 4)
      flg = (flg & 0xe0) + 31 - ((cmf << 8) + (flg & 0xe0)) % 31
  return bytes([cmf, flg])


def _crc_table():
  t = []
  for i in range(256):
    c = i
    for _ in range(8):
      c = (c >> 1) ^ (0xEDB88320 & -(c & 1))
    t.append(c)
  return t


_CRC_TABLE = _crc_table()


def crc32(data):
  c = 0xFFFFFFFF
  for byte in bytes(data):
    c = _CRC_TABLE[(c ^ byte) & 0xFF] ^ (c >> 8)
  return c ^ 0xFFFFFFFF


def chunk(kind, body):
  return struct.pack('>I', len(body)) + kind + body + struct.pack('>I', crc32(kind + body))


def check_size(h, w):
  if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
    raise ValueError('a PNG is 1 to %d pixels wide and high, got %dx%d' % (MAX_SIDE, w, h))


def encode(bgr, info=None):
  """The bytes of cv2.imencode('.png', bgr) for a uint8 BGR [h, w, 3] image.  `info`, a dict, gets
  deflate_rle's 'blocks' and 'symbols', 'zlib_bytes' and 'idat' (the IDAT lengths)."""
  bgr = np.asarray(bgr, np.uint8)
  h, w = bgr.shape[:2]
  check_size(h, w)
  data = filter_rows(bgr)
  z = zlib_header(len(data)) + deflate_rle(data, info) + struct.pack('>I', adler32(data))
  idat = [z[i:i + IDAT_BYTES] for i in range(0, len(z), IDAT_BYTES)]
  if info is not None:
    info['zlib_bytes'] = len(z)
    info['idat'] = [len(c) for c in idat]
  ihdr = struct.pack('>IIBBBBB', w, h, 8, 2, 0, 0, 0)
  return (SIGNATURE + chunk(b'IHDR', ihdr) + b''.join(chunk(b'IDAT', c) for c in idat) +
          chunk(b'IEND', b''))
