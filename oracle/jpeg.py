"""CPU restatement of the baseline JPEG encoder cv2.imencode('.jpg', ...) runs (libjpeg-turbo's
integer pipeline with its defaults) — test infrastructure, like the rest of oracle/.

encode(bgr, quality) returns the bytes of cv2.imencode('.jpg', bgr, [IMWRITE_JPEG_QUALITY, quality]),
PINNED bitwise against the installed cv2 (tests/test_oracle_jpeg.py):

  header    SOI, JFIF APP0 1.01 (density 1:1, no unit), one DQT per table, SOF0 with Y 2x2 and
            Cb, Cr 1x1 (4:2:0), one DHT per table (Annex K's DC, AC luminance and chrominance
            tables), SOS over the three components, no restart interval
  colour    RGB -> YCbCr in 16-bit fixed point; Cb and Cr round with ONE_HALF - 1
  edges     the last row is repeated to a 2-row group, each component's last column to its
            width_in_blocks * 8 samples (the chroma before its 2x2 downsampling), and the last
            downsampled row to a whole 16-row MCU row
  chroma    2x2 box sum plus the bias 1, 2, 1, 2, ... along a row, >> 2
  DCT       jpeg_fdct_islow (13 fraction bits, 2 pass bits) on samples - 128
  quantize  each coefficient x by d = 8 q: sign(x) * ((|x| + c) * m >> s), the reciprocal
            (m, c, s) of d built for 16-bit coefficients (quant_reciprocal); for every |x| < 2^15
            that is |x| / d rounded half away from zero
  MCUs      Y0 Y1 Y2 Y3 Cb Cr; a luma block right of or below the image's blocks (a dummy block)
            is all zero with the DC of the block before it, so it codes as DC difference 0 + EOB
  entropy   DC differences per component, AC run/size codes with ZRL and EOB, 0xFF bytes
            followed by 0x00, the last byte padded with 1-bits, then EOI
"""
import numpy as np

# ---- tables (ITU T.81 Annex K) ------------------------------------------------------------------
STD_LUMA_QT = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
    14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
STD_CHROMA_QT = np.full(64, 99, np.int64)
STD_CHROMA_QT[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66,
                                                                24, 26, 56, 47, 66]

# ZIGZAG[k] is the natural (row-major) index of the k-th coefficient in zigzag order
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5,
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)

DC_LUMA_BITS = [0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0]
DC_CHROMA_BITS = [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0]
DC_VALS = list(range(12))
AC_LUMA_BITS = [0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d]
AC_CHROMA_BITS = [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77]
AC_LUMA_VALS = [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5,
    0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
    0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa]
AC_CHROMA_VALS = [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
    0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0,
    0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26,
    0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5,
    0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
    0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa]
assert len(AC_LUMA_VALS) == sum(AC_LUMA_BITS) == 162
assert len(AC_CHROMA_VALS) == sum(AC_CHROMA_BITS) == 162


def huffman_codes(bits, vals):
  """(code [256], length [256]) of the canonical Huffman code with `bits[l - 1]` codes of length l
  for the symbols `vals` in order (length 0: not in the table)."""
  code = np.zeros(256, np.int64)
  size = np.zeros(256, np.int64)
  c, k = 0, 0
  for length in range(1, 17):
    for _ in range(bits[length - 1]):
      code[vals[k]] = c
      size[vals[k]] = length
      c += 1
      k += 1
    c <<= 1
  return code, size


# (DC code, DC length, AC code, AC length) of luma (0) and chroma (1)
HUFF = [huffman_codes(DC_LUMA_BITS, DC_VALS) + huffman_codes(AC_LUMA_BITS, AC_LUMA_VALS),
        huffman_codes(DC_CHROMA_BITS, DC_VALS) + huffman_codes(AC_CHROMA_BITS, AC_CHROMA_VALS)]


def quant_tables(quality):
  """The luma and chroma quantization tables (natural order) of `quality` in 1..100: the standard
  tables scaled by jpeg_quality_scaling, rounded, clamped to 1..255 (baseline)."""
  if not 1 <= quality <= 100:
    raise ValueError('quality must be in [1, 100], got %r' % (quality,))
  scale = 5000 // quality if quality < 50 else 200 - 2 * quality
  return [np.clip((t * scale + 50) // 100, 1, 255) for t in (STD_LUMA_QT, STD_CHROMA_QT)]


def quant_reciprocal(d):
  """(m, c, s) with q = (|x| + c) * m >> s for a divisor d = 8 q >= 8: the reciprocal
  libjpeg-turbo builds for 16-bit coefficients (compute_reciprocal)."""
  d = np.asarray(d, np.int64)
  b = np.floor(np.log2(d)).astype(np.int64)
  r = 16 + b
  fq = (np.int64(1) << r) // d
  fr = (np.int64(1) << r) % d
  c = d // 2
  pow2 = fr == 0
  fq = np.where(pow2, fq >> 1, np.where(fr > d // 2, fq + 1, fq))
  r = np.where(pow2, r - 1, r)
  c = np.where(~pow2 & (fr <= d // 2), c + 1, c)
  return fq, c, r


def quantize(x, d):
  """x (DCT output) divided by d = 8 q as libjpeg-turbo's quantize does."""
  m, c, s = quant_reciprocal(d)
  a = np.abs(x)
  q = ((a + c) * m) >> s
  return np.where(x < 0, -q, q)


# ---- pixel pipeline ---------------------------------------------------------------------------
def _fix(x):
  return int(x * 65536 + 0.5)


def rgb_to_ycc(bgr):
  """Y, Cb, Cr planes (int64) of a uint8 BGR image, as libjpeg-turbo's rgb_ycc_convert."""
  b, g, r = (bgr[..., i].astype(np.int64) for i in range(3))
  half, off = 1 << 15, 128 << 16
  y = (_fix(0.29900) * r + _fix(0.58700) * g + _fix(0.11400) * b + half) >> 16
  cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + off + half - 1) >> 16
  cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + off + half - 1) >> 16
  return y, cb, cr


def _pad_to(a, rows, cols):
  """a with its last row and column repeated to rows x cols."""
  return np.pad(a, ((0, rows - a.shape[0]), (0, cols - a.shape[1])), mode='edge')


def planes_420(bgr):
  """The Y (16 * mcu_rows x 8 * ceil(w / 8)) and Cb, Cr (8 * mcu_rows x 8 * ceil(w / 16)) sample
  planes the DCT reads, edges replicated and chroma downsampled as libjpeg-turbo does."""
  h, w = bgr.shape[:2]
  mcu_rows = -(-h // 16)
  y, cb, cr = rgb_to_ycc(bgr)
  ycols, ccols = 8 * -(-w // 8), 8 * -(-w // 16)
  Y = _pad_to(y, 16 * mcu_rows, ycols)
  out = [Y]
  for p in (cb, cr):
    p = _pad_to(p, 2 * -(-h // 2), 2 * ccols)          # row group, then width_in_blocks * 16
    s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
    bias = np.tile(np.array([1, 2], np.int64), ccols // 2 + 1)[:ccols]
    out.append(_pad_to((s + bias) >> 2, 8 * mcu_rows, ccols))
  return out


def fdct_islow(blocks):
  """jpeg_fdct_islow of int64 blocks [..., 8, 8] of samples - 128 (output scaled by 8)."""
  CB, PB = 13, 2
  F = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299,
           c1847=15137, c1961=16069, c2053=16819, c2562=20995, c3072=25172)

  def desc(x, n):
    return (x + (1 << (n - 1))) >> n

  def one_pass(d, first):
    d = [d[..., i] for i in range(8)]
    t0, t7 = d[0] + d[7], d[0] - d[7]
    t1, t6 = d[1] + d[6], d[1] - d[6]
    t2, t5 = d[2] + d[5], d[2] - d[5]
    t3, t4 = d[3] + d[4], d[3] - d[4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = [None] * 8
    sh = CB - PB if first else CB + PB
    o[0] = (t10 + t11) << PB if first else desc(t10 + t11, PB)
    o[4] = (t10 - t11) << PB if first else desc(t10 - t11, PB)
    z1 = (t12 + t13) * F['c0541']
    o[2] = desc(z1 + t13 * F['c0765'], sh)
    o[6] = desc(z1 - t12 * F['c1847'], sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * F['c1175']
    t4, t5, t6, t7 = t4 * F['c0298'], t5 * F['c2053'], t6 * F['c3072'], t7 * F['c1501']
    z1, z2 = z1 * -F['c0899'], z2 * -F['c2562']
    z3, z4 = z3 * -F['c1961'] + z5, z4 * -F['c0390'] + z5
    o[7] = desc(t4 + z1 + z3, sh)
    o[5] = desc(t5 + z2 + z4, sh)
    o[3] = desc(t6 + z2 + z3, sh)
    o[1] = desc(t7 + z1 + z4, sh)
    return np.stack(o, axis=-1)

  rows = one_pass(blocks, True)
  return np.swapaxes(one_pass(np.swapaxes(rows, -1, -2), False), -1, -2)


def _blocks(plane):
  """[rows / 8, cols / 8, 64] of a sample plane's 8x8 blocks (natural order)."""
  r, c = plane.shape
  return plane.reshape(r // 8, 8, c // 8, 8).swapaxes(1, 2).reshape(r // 8, c // 8, 64)


def coefficients(bgr, quality):
  """(Y [mcu_rows, mcu_cols, 4, 64], Cb, Cr [mcu_rows, mcu_cols, 64]) quantized zigzag
  coefficients of every MCU, dummy luma blocks zero (their DC is resolved by the entropy coder)."""
  h, w = bgr.shape[:2]
  qy, qc = quant_tables(quality)
  mr, mc = -(-h // 16), -(-w // 16)
  Y, Cb, Cr = planes_420(bgr)

  def coef(plane, q):
    blk = _blocks(plane)
    d = fdct_islow(blk.reshape(blk.shape[:2] + (8, 8)) - 128).reshape(blk.shape)
    return quantize(d, q * 8)[..., ZIGZAG]

  yb = coef(Y, qy)                                    # [2 mr, ceil(w / 8), 64]
  full = np.zeros((2 * mr, 2 * mc, 64), np.int64)
  full[:, :yb.shape[1]] = yb
  hib = -(-h // 8)
  full[hib:] = 0
  yq = full.reshape(mr, 2, mc, 2, 64).transpose(0, 2, 1, 3, 4).reshape(mr, mc, 4, 64)
  return yq, coef(Cb, qc), coef(Cr, qc)


# ---- entropy coding ----------------------------------------------------------------------------
def _nbits(a):
  """Bit length of |a| (0 for 0)."""
  a = np.abs(a)
  out = np.zeros(a.shape, np.int64)
  nz = a > 0
  out[nz] = np.floor(np.log2(a[nz])).astype(np.int64) + 1
  return out


def _scan_symbols(h, w, yq, cb, cr):
  """The coded (value, length) pairs of the whole scan, in stream order."""
  mr, mc = yq.shape[:2]
  hib, wib = -(-h // 8), -(-w // 8)
  # block stream order: per MCU, Y0 Y1 Y2 Y3 Cb Cr
  blocks = np.concatenate([yq, cb[:, :, None], cr[:, :, None]], axis=2).reshape(-1, 64)
  comp = np.tile(np.array([0, 0, 0, 0, 1, 2]), mr * mc)
  by = (np.arange(mr)[:, None, None] * 2 + np.array([0, 0, 1, 1])[None, None, :])
  bx = (np.arange(mc)[None, :, None] * 2 + np.array([0, 1, 0, 1])[None, None, :])
  dummy_y = ((by >= hib) | (bx >= wib)).reshape(mr, mc, 4)
  dummy = np.concatenate([dummy_y, np.zeros((mr, mc, 2), bool)], axis=2).reshape(-1)
  # DC differences per component; a dummy block repeats the previous block's DC
  dc = blocks[:, 0].copy()
  diff = np.zeros(len(blocks), np.int64)
  for c in range(3):
    idx = np.nonzero(comp == c)[0]
    v = dc[idx]
    real = ~dummy[idx]
    # effective DC: the last real block's DC at or before each position
    last_real = np.maximum.accumulate(np.where(real, np.arange(len(idx)), -1))
    eff = v[last_real]
    prev = np.concatenate([[0], eff[:-1]])
    diff[idx] = np.where(real, eff - prev, 0)
  blocks[dummy] = 0
  table = np.where(comp == 0, 0, 1)

  keys, vals, lens = [], [], []
  # DC
  nb = _nbits(diff)
  vbits = np.where(diff < 0, diff - 1, diff) & ((np.int64(1) << nb) - 1)
  dcode = np.where(table == 0, HUFF[0][0][nb], HUFF[1][0][nb])
  dlen = np.where(table == 0, HUFF[0][1][nb], HUFF[1][1][nb])
  keys.append(np.arange(len(blocks)) * 256)
  vals.append((dcode << nb) | vbits)
  lens.append(dlen + nb)
  # AC
  ac = blocks[:, 1:]
  bi, ki = np.nonzero(ac)
  k = ki + 1
  first = np.ones(len(bi), bool)
  first[1:] = bi[1:] != bi[:-1]
  prevk = np.where(first, 0, np.concatenate([[0], k[:-1]]))
  run = k - prevk - 1
  v = ac[bi, ki]
  nb = _nbits(v)
  vbits = np.where(v < 0, v - 1, v) & ((np.int64(1) << nb) - 1)
  sym = ((run & 15) << 4) | nb
  t = table[bi]
  code = np.where(t == 0, HUFF[0][2][sym], HUFF[1][2][sym])
  clen = np.where(t == 0, HUFF[0][3][sym], HUFF[1][3][sym])
  keys.append(bi * 256 + k * 4 + 3)
  vals.append((code << nb) | vbits)
  lens.append(clen + nb)
  for j in range(3):                                  # ZRLs before the run's symbol
    m = (run >> 4) > j
    zc = np.where(t[m] == 0, HUFF[0][2][0xF0], HUFF[1][2][0xF0])
    zl = np.where(t[m] == 0, HUFF[0][3][0xF0], HUFF[1][3][0xF0])
    keys.append(bi[m] * 256 + k[m] * 4 + j)
    vals.append(zc)
    lens.append(zl)
  # EOB after the last nonzero coefficient, unless it is coefficient 63
  lastk = np.zeros(len(blocks), np.int64)
  np.maximum.at(lastk, bi, k)
  e = np.nonzero(lastk < 63)[0]
  te = table[e]
  keys.append(e * 256 + 255)
  vals.append(np.where(te == 0, HUFF[0][2][0], HUFF[1][2][0]))
  lens.append(np.where(te == 0, HUFF[0][3][0], HUFF[1][3][0]))
  keys, vals, lens = (np.concatenate(a) for a in (keys, vals, lens))
  order = np.argsort(keys, kind='stable')
  return vals[order], lens[order]


def _pack(vals, lens):
  """The entropy-coded segment: the codes MSB first, 1-bit padded, 0xFF stuffed with 0x00."""
  total = int(lens.sum())
  pad = -total % 8
  vals = np.append(vals, (1 << pad) - 1)
  lens = np.append(lens, pad)
  starts = np.cumsum(lens) - lens
  ev = np.repeat(np.arange(len(lens)), lens)
  pos = np.arange(total + pad) - starts[ev]
  bits = ((vals[ev] >> (lens[ev] - 1 - pos)) & 1).astype(np.uint8)
  data = np.packbits(bits)
  ff = np.nonzero(data == 0xFF)[0]
  return np.insert(data, ff + 1, 0).tobytes()


def header(h, w, quality):
  """The bytes before the entropy-coded segment of an h x w image at `quality`."""
  def seg(marker, body):
    return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, 'big') + bytes(body)

  qy, qc = quant_tables(quality)
  out = bytes([0xFF, 0xD8])
  out += seg(0xE0, b'JFIF\x00' + bytes([1, 1, 0, 0, 1, 0, 1, 0, 0]))
  for i, q in enumerate((qy, qc)):
    out += seg(0xDB, bytes([i]) + bytes(int(v) for v in q[ZIGZAG]))
  out += seg(0xC0, bytes([8, h >> 8, h & 255, w >> 8, w & 255, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
  for cls_id, bits, vals in ((0x00, DC_LUMA_BITS, DC_VALS), (0x10, AC_LUMA_BITS, AC_LUMA_VALS),
                             (0x01, DC_CHROMA_BITS, DC_VALS), (0x11, AC_CHROMA_BITS, AC_CHROMA_VALS)):
    out += seg(0xC4, bytes([cls_id]) + bytes(bits) + bytes(vals))
  out += seg(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))
  return out


def encode(bgr, quality=95):
  """The bytes cv2.imencode('.jpg', bgr, [cv2.IMWRITE_JPEG_QUALITY, quality]) writes for a uint8
  BGR image [h, w, 3].  Sides above 65500 (libjpeg's JPEG_MAX_DIMENSION) raise ValueError where
  cv2.imencode fails."""
  bgr = np.asarray(bgr)
  if bgr.dtype != np.uint8 or bgr.ndim != 3 or bgr.shape[2] != 3 or min(bgr.shape[:2]) < 1:
    raise ValueError('need a non-empty uint8 [h, w, 3] image, got %s %r' % (bgr.dtype, bgr.shape))
  h, w = bgr.shape[:2]
  if h > 65500 or w > 65500:
    raise ValueError('JPEG sizes are at most 65500, got %dx%d' % (w, h))
  yq, cb, cr = coefficients(bgr, quality)
  vals, lens = _scan_symbols(h, w, yq, cb, cr)
  return header(h, w, quality) + _pack(vals, lens) + bytes([0xFF, 0xD9])
