"""CPU restatement of cv2.imencode('.jpg', ...) with its other IMWRITE_JPEG_* parameters: sampling
factors, optimized Huffman tables, restart intervals and separate luma and chroma quality (libjpeg-
turbo's integer pipeline, as oracle/jpeg.py, whose colour conversion, DCT and quantization this
reuses).  PINNED bitwise against the installed cv2 (tests/test_oracle_jpeg_params.py).

encode(bgr, quality, sampling=..., optimize=..., restart_interval=..., luma_quality=...,
chroma_quality=...) is what cv2 writes for the matching parameters:

  sampling  the luma factors h x v of '411' (4x1), '420' (2x2, the default), '422' (2x1), '440'
            (1x2) or '444' (1x1); Cb and Cr are 1x1.  An MCU is 8 h x 8 v pixels: h v luma blocks
            (row-major), then Cb, Cr
  edges     the full-size planes' last row is repeated to a multiple of v rows and their last column
            to the component's width_in_blocks * 8 * (its downsampling); luma rows and the
            downsampled chroma rows to whole MCU rows.  Luma blocks right of or below the image's
            ceil(w / 8) x ceil(h / 8) blocks are dummies (all zero, the DC of the block before)
  chroma    h2v2: (sum of 2x2 + 1, 2, 1, 2, ...) >> 2; h2v1: (sum of 2 + 0, 1, 0, 1, ...) >> 1;
            4x1 and 1x2 (int_downsample): (sum + 2) // 4 and (sum + 1) // 2
  quality   luma_quality alone replaces quality; chroma_quality alone is ignored; both set scale
            the luma and chroma tables separately, and when they differ the file is 4:4:4 whatever
            `sampling` says
  optimize  the four tables (DC and AC of luma and chroma) are jpeg_gen_optimal_table of the
            symbol counts of the whole scan, dummy blocks included
  restart   a DRI segment (after the DHTs) when the interval (in MCUs) is above 0; the DC
            predictors reset at each interval, each interval is padded to a byte with 1-bits and
            stuffed on its own, and RSTn (n = 0..7 in turn) sits between intervals, unstuffed
"""
import numpy as np

from oracle.jpeg import (AC_CHROMA_BITS, AC_CHROMA_VALS, AC_LUMA_BITS, AC_LUMA_VALS, DC_CHROMA_BITS,
                         DC_LUMA_BITS, DC_VALS, ZIGZAG, _nbits, _pack, _pad_to, fdct_islow,
                         huffman_codes, quant_tables, quantize, rgb_to_ycc)

# luma (h, v) sampling factors and cv2's IMWRITE_JPEG_SAMPLING_FACTOR value of each sampling
SAMPLING_FACTORS = {'411': (4, 1), '420': (2, 2), '422': (2, 1), '440': (1, 2), '444': (1, 1)}
CV2_SAMPLING = {'411': 0x411111, '420': 0x221111, '422': 0x211111, '440': 0x121111, '444': 0x111111}
STD_TABLES = [(DC_LUMA_BITS, DC_VALS), (AC_LUMA_BITS, AC_LUMA_VALS),
              (DC_CHROMA_BITS, DC_VALS), (AC_CHROMA_BITS, AC_CHROMA_VALS)]


def cv2_params(quality=95, sampling='420', optimize=False, restart_interval=0, luma_quality=None,
               chroma_quality=None):
  """The cv2.imencode parameter list of these settings (IMWRITE_JPEG_* only where set)."""
  import cv2
  p = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, CV2_SAMPLING[sampling]]
  if optimize:
    p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
  if restart_interval:
    p += [cv2.IMWRITE_JPEG_RST_INTERVAL, restart_interval]
  if luma_quality is not None:
    p += [cv2.IMWRITE_JPEG_LUMA_QUALITY, luma_quality]
  if chroma_quality is not None:
    p += [cv2.IMWRITE_JPEG_CHROMA_QUALITY, chroma_quality]
  return p


def resolve(quality=95, sampling='420', luma_quality=None, chroma_quality=None):
  """(luma quality, chroma quality, (h, v) luma sampling factors) cv2 encodes with."""
  for name, q in (('quality', quality), ('luma_quality', luma_quality),
                  ('chroma_quality', chroma_quality)):
    if q is not None and not 1 <= q <= 100:
      raise ValueError('%s must be in [1, 100], got %r' % (name, q))
  if sampling not in SAMPLING_FACTORS:
    raise ValueError('sampling must be one of %s, got %r' % (', '.join(SAMPLING_FACTORS), sampling))
  if luma_quality is None:
    return quality, quality, SAMPLING_FACTORS[sampling]
  cq = luma_quality if chroma_quality is None else chroma_quality
  return luma_quality, cq, (1, 1) if cq != luma_quality else SAMPLING_FACTORS[sampling]


def downsample(p, hs, vs):
  """A full-size chroma plane (already edge-expanded to multiples of hs columns and vs rows)
  downsampled by hs x vs as libjpeg-turbo's jcsample.c does for a 1x1 component."""
  if (hs, vs) == (1, 1):
    return p
  if (hs, vs) == (2, 1):
    bias = np.tile(np.array([0, 1], np.int64), p.shape[1] // 4 + 1)[:p.shape[1] // 2]
    return (p[:, 0::2] + p[:, 1::2] + bias) >> 1
  if (hs, vs) == (2, 2):
    bias = np.tile(np.array([1, 2], np.int64), p.shape[1] // 4 + 1)[:p.shape[1] // 2]
    return (p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2] + bias) >> 2
  s = sum(p[i::vs, j::hs] for i in range(vs) for j in range(hs))
  return (s + hs * vs // 2) // (hs * vs)


def coefficients(bgr, lq, cq, hs, vs):
  """(blocks [N, 64] quantized zigzag coefficients in stream order, component [N], dummy [N],
  blocks per MCU) of the whole scan; dummy blocks are zero."""
  h, w = bgr.shape[:2]
  mr, mc = -(-h // (8 * vs)), -(-w // (8 * hs))
  hib, wib = -(-h // 8), -(-w // 8)
  qy, qc = quant_tables(lq)[0], quant_tables(cq)[1]
  y, cb, cr = rgb_to_ycc(bgr)

  def coef(plane, q):
    r, c = plane.shape
    blk = plane.reshape(r // 8, 8, c // 8, 8).swapaxes(1, 2) - 128
    return quantize(fdct_islow(blk).reshape(r // 8, c // 8, 64), q * 8)[..., ZIGZAG]

  yb = np.zeros((vs * mr, hs * mc, 64), np.int64)
  yb[:hib, :wib] = coef(_pad_to(y, 8 * hib, 8 * wib), qy)
  dummy_y = np.ones((vs * mr, hs * mc), bool)
  dummy_y[:hib, :wib] = False
  chroma = []
  for p in (cb, cr):
    p = _pad_to(p, vs * -(-h // vs), 8 * hs * mc)
    chroma.append(coef(_pad_to(downsample(p, hs, vs), 8 * mr, 8 * mc), qc))
  per = hs * vs + 2
  yq = yb.reshape(mr, vs, mc, hs, 64).transpose(0, 2, 1, 3, 4).reshape(mr, mc, hs * vs, 64)
  blocks = np.concatenate([yq, chroma[0][:, :, None], chroma[1][:, :, None]], axis=2).reshape(-1, 64)
  dy = dummy_y.reshape(mr, vs, mc, hs).transpose(0, 2, 1, 3).reshape(mr, mc, hs * vs)
  dummy = np.concatenate([dy, np.zeros((mr, mc, 2), bool)], axis=2).reshape(-1)
  comp = np.tile(np.array([0] * (hs * vs) + [1, 2]), mr * mc)
  return blocks, comp, dummy, per


def symbols(blocks, comp, dummy, per, restart_interval):
  """(table [S] 0..3 = DC luma, AC luma, DC chroma, AC chroma, symbol [S], extra bits [S], their
  length [S], block [S]) of every Huffman symbol of the scan, in stream order."""
  n = len(blocks)
  interval = np.arange(n) // per // restart_interval if restart_interval else np.zeros(n, np.int64)
  dc = blocks[:, 0]
  diff = np.zeros(n, np.int64)
  for c in range(3):
    idx = np.nonzero(comp == c)[0]
    real = ~dummy[idx]
    # a dummy block stands for the last real block before it (the MCU's first luma block is real)
    eff = dc[idx][np.maximum.accumulate(np.where(real, np.arange(len(idx)), -1))]
    prev = np.concatenate([[0], eff[:-1]])
    first = np.concatenate([[True], interval[idx][1:] != interval[idx][:-1]])
    diff[idx] = np.where(real, eff - np.where(first, 0, prev), 0)
  chroma = (comp > 0).astype(np.int64)
  ac = np.where(dummy[:, None], 0, blocks[:, 1:])

  keys, tabs, syms, extra, enb = [], [], [], [], []

  def add(key, tab, sym, val, nb):
    keys.append(key)
    tabs.append(tab)
    syms.append(sym)
    extra.append(np.where(val < 0, val - 1, val) & ((np.int64(1) << nb) - 1))
    enb.append(nb)

  nb = _nbits(diff)
  add(np.arange(n) * 256, 2 * chroma, nb, diff, nb)
  bi, ki = np.nonzero(ac)
  k = ki + 1
  first = np.ones(len(bi), bool)
  first[1:] = bi[1:] != bi[:-1]
  run = k - np.where(first, 0, np.concatenate([[0], k[:-1]])) - 1
  v = ac[bi, ki]
  nb = _nbits(v)
  t = 2 * chroma[bi] + 1
  add(bi * 256 + k * 4 + 3, t, ((run & 15) << 4) | nb, v, nb)
  for j in range(3):                                  # ZRLs before the run's symbol
    m = (run >> 4) > j
    add(bi[m] * 256 + k[m] * 4 + j, t[m], np.full(m.sum(), 0xF0), np.zeros(m.sum(), np.int64),
        np.zeros(m.sum(), np.int64))
  lastk = np.zeros(n, np.int64)
  np.maximum.at(lastk, bi, k)
  e = np.nonzero(lastk < 63)[0]                        # EOB unless coefficient 63 is nonzero
  add(e * 256 + 255, 2 * chroma[e] + 1, np.zeros(len(e), np.int64), np.zeros(len(e), np.int64),
      np.zeros(len(e), np.int64))
  keys, tabs, syms, extra, enb = (np.concatenate(a).astype(np.int64) for a in (keys, tabs, syms, extra, enb))
  order = np.argsort(keys, kind='stable')
  return tabs[order], syms[order], extra[order], enb[order], keys[order] // 256


def optimal_table(freq):
  """jpeg_gen_optimal_table (JPEG Annex K.2, with libjpeg's tie-breaking and reserved all-ones
  code): {symbol: count} -> (bits[16], vals), lengths limited to 16 bits."""
  f = [0] * 257
  for s, c in freq.items():
    f[s] = c
  f[256] = 1
  size, others = [0] * 257, [-1] * 257
  while True:
    # the smallest nonzero count (ties: the larger symbol), then the next smallest
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
  for i in range(32, 16, -1):                         # lengths above 16 moved up the tree
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
  bits[i] -= 1                                        # the reserved symbol 256's code
  vals = [s for length in range(1, 33) for s in range(256) if size[s] == length]
  return bits[1:17], vals


def header(h, w, lq, cq, hs, vs, tables, restart_interval):
  """The bytes before the entropy-coded segment: SOI, JFIF APP0, DQT x 2, SOF0, DHT x 4 (`tables`:
  (bits, vals) of DC luma, AC luma, DC chroma, AC chroma), DRI when restart_interval > 0, SOS."""
  def seg(marker, body):
    return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, 'big') + bytes(body)

  out = bytes([0xFF, 0xD8]) + seg(0xE0, b'JFIF\x00' + bytes([1, 1, 0, 0, 1, 0, 1, 0, 0]))
  for i, q in enumerate((quant_tables(lq)[0], quant_tables(cq)[1])):
    out += seg(0xDB, bytes([i]) + bytes(int(v) for v in q[ZIGZAG]))
  out += seg(0xC0, bytes([8, h >> 8, h & 255, w >> 8, w & 255, 3, 1, hs << 4 | vs, 0, 2, 0x11, 1,
                          3, 0x11, 1]))
  for cls_id, (bits, vals) in zip((0x00, 0x10, 0x01, 0x11), tables):
    out += seg(0xC4, bytes([cls_id]) + bytes(bits) + bytes(vals))
  if restart_interval:
    out += seg(0xDD, restart_interval.to_bytes(2, 'big'))
  return out + seg(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))


def encode(bgr, quality=95, *, sampling='420', optimize=False, restart_interval=0,
           luma_quality=None, chroma_quality=None):
  """The bytes cv2.imencode('.jpg', bgr, cv2_params(...)) writes for a uint8 BGR image [h, w, 3].
  Values cv2 would clamp (qualities outside 1..100, restart intervals outside 0..65535) and
  sizes it refuses (sides above 65500) raise ValueError."""
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
  tab, sym, extra, enb, blk = symbols(blocks, comp, dummy, per, restart_interval)
  tables = STD_TABLES
  if optimize:
    tables = []
    for t in range(4):
      counts = np.bincount(sym[tab == t], minlength=256)
      tables.append(optimal_table({s: int(c) for s, c in enumerate(counts) if c}))
  codes = [huffman_codes(*tb) for tb in tables]
  code = np.stack([c[0] for c in codes])[tab, sym]
  clen = np.stack([c[1] for c in codes])[tab, sym]
  vals, lens = (code << enb) | extra, clen + enb
  # each restart interval is packed (padded and stuffed) on its own, RSTn between them
  interval = blk // per // restart_interval if restart_interval else np.zeros(len(blk), np.int64)
  bounds = np.searchsorted(interval, np.arange(interval[-1] + 2))
  body = b''
  for i in range(len(bounds) - 1):
    if i:
      body += bytes([0xFF, 0xD0 + (i - 1) % 8])
    body += _pack(vals[bounds[i]:bounds[i + 1]], lens[bounds[i]:bounds[i + 1]])
  return header(h, w, lq, cq, hs, vs, tables, restart_interval) + body + bytes([0xFF, 0xD9])
