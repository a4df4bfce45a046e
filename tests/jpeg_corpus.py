"""JPEG files for the decoder's tests, made by cv2.imencode from seeded content: the content kinds
of test_gpu_jpeg (noise, gradients, flat, checkerboards of pixels and of 8x8 blocks, dots) plus a
smooth picture, over sizes, qualities, samplings, restart intervals, optimized Huffman tables,
separate luma and chroma qualities, grayscale and EXIF orientations.  foreign() rewrites such
files with tests/jpeg_writer.py into what other encoders write; camera() is at camera sizes;
exif_variants() and refused() pin how cv2 reads EXIF and what the decoder refuses."""
import cv2
import numpy as np

from oracle import jpeg_decode as D
from oracle.jpeg_decode import with_orientation

import jpeg_writer as W

KINDS = ('noise', 'grad', 'flat', 'check', 'blocks', 'dots', 'smooth')
SAMPLINGS = (0x111111, 0x211111, 0x121111, 0x221111, 0x411111)
SIZES = [(1, 1), (1, 2), (2, 1), (2, 3), (3, 5), (5, 4), (7, 9), (8, 8), (9, 17), (15, 31),
         (16, 16), (17, 23), (31, 33), (61, 97)]


def content(kind, h, w, c, rng):
  """uint8 [h, w, c]."""
  if kind == 'noise':
    return rng.integers(0, 256, (h, w, c), dtype=np.uint8)
  y, x = np.mgrid[:h, :w]
  if kind == 'grad':
    return ((y[..., None] * 3 + x[..., None] * 5 + np.arange(c) * 40) % 256).astype(np.uint8)
  if kind == 'flat':
    return np.full((h, w, c), 77, np.uint8)
  if kind in ('check', 'blocks'):
    cell = (y + x) % 2 if kind == 'check' else (y // 8 + x // 8) % 2
    return np.repeat((cell * 255).astype(np.uint8)[..., None], c, axis=2)
  if kind == 'smooth':
    ph = rng.uniform(0, 6, c)
    v = 128 + 90 * np.sin(y[..., None] / 37.0 + ph) * np.cos(x[..., None] / 53.0 + 2 * ph)
    return np.clip(v + rng.normal(0, 3, (h, w, c)), 0, 255).astype(np.uint8)
  img = np.full((h, w, c), 128, np.uint8)
  img[(y % 8 == 7) & (x % 8 == 7)] = 255
  return img


def encode(img, *params):
  ok, buf = cv2.imencode('.jpg', img, list(params))
  assert ok
  return buf.tobytes()


def corpus(seed=0, big=True):
  """[(name, file bytes)] covering every case the decoder supports."""
  rng = np.random.default_rng(seed)
  out = []
  for si, samp in enumerate(SAMPLINGS):
    for zi, (h, w) in enumerate(SIZES):
      kind = KINDS[(si + zi) % len(KINDS)]
      q = (1, 5, 25, 50, 75, 90, 95, 100)[(si * 3 + zi) % 8]
      out.append(('%s %dx%d s%06x q%d' % (kind, h, w, samp, q),
                  encode(content(kind, h, w, 3, rng), cv2.IMWRITE_JPEG_QUALITY, q,
                         cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)))
  for kind in KINDS:
    img = content(kind, 45, 70, 3, rng)
    for samp in SAMPLINGS:
      out.append(('%s 45x70 s%06x rst2' % (kind, samp),
                  encode(img, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp, cv2.IMWRITE_JPEG_RST_INTERVAL, 2)))
    out.append(('%s 45x70 optimize' % kind, encode(img, cv2.IMWRITE_JPEG_OPTIMIZE, 1)))
    out.append(('%s 45x70 luma20 chroma90' % kind,
                encode(img, cv2.IMWRITE_JPEG_LUMA_QUALITY, 20, cv2.IMWRITE_JPEG_CHROMA_QUALITY, 90)))
    out.append(('%s 45x70 gray' % kind, encode(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY),
                                              cv2.IMWRITE_JPEG_QUALITY, 85)))
  for q in (1, 10, 50, 100):
    out.append(('noise 33x47 gray q%d rst1' % q,
                encode(content('noise', 33, 47, 1, rng)[..., 0], cv2.IMWRITE_JPEG_QUALITY, q,
                       cv2.IMWRITE_JPEG_RST_INTERVAL, 1)))
  base = content('smooth', 37, 58, 3, rng)
  for o in range(1, 9):
    for samp in (0x221111, 0x211111):
      out.append(('exif %d s%06x' % (o, samp),
                  with_orientation(encode(base, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp), o, o % 2 == 0)))
  if big:
    for (h, w), samp in (((375, 1242), 0x221111), ((1080, 1920), 0x221111), ((1080, 1920), 0x111111)):
      out.append(('smooth %dx%d s%06x q95' % (h, w, samp),
                  encode(content('smooth', h, w, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 95,
                         cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)))
  return out


def imdecode(f):
  return cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)


# ---- hand-made variants of cv2's files: what other encoders write ---------------------------------
def segments(f):
  """[(marker, body)] of the header up to and including SOS, and the bytes after it."""
  i, out = 2, []
  while True:
    m, n = f[i + 1], int.from_bytes(f[i + 2:i + 4], 'big')
    out.append((m, bytes(f[i + 4:i + 2 + n])))
    i += 2 + n
    if m == 0xDA:
      return out, bytes(f[i:])


def assemble(segs, rest):
  return b'\xff\xd8' + b''.join(bytes([0xFF, m]) + (len(b) + 2).to_bytes(2, 'big') + b
                                for m, b in segs) + rest


def sixteen_bit_tables(f, scale=1, sof=0xC1):
  """f with 16-bit DQT entries scaled by `scale` (capped at 65535) and SOF marker `sof`."""
  segs, rest = segments(f)
  out = []
  for m, b in segs:
    if m == 0xDB:
      nb, j = bytearray(), 0
      while j < len(b):
        nb += bytes([0x10 | (b[j] & 15)]) + b''.join(min(v * scale, 65535).to_bytes(2, 'big')
                                                     for v in b[j + 1:j + 65])
        j += 65
      b = bytes(nb)
    out.append((sof if m == 0xC0 else m, b))
  return assemble(out, rest)


def component_ids(f, ids, jfif=True, adobe=None):
  """f with component ids `ids` in SOF and SOS, its JFIF APP0 kept or dropped, and an Adobe APP14
  with transform `adobe` added (None: none)."""
  segs, rest = segments(f)
  out = [] if adobe is None else [(0xEE, b'Adobe' + bytes([0, 100, 0, 0, 0, 0, adobe]))]
  for m, b in segs:
    b = bytearray(b)
    if m == 0xE0 and not jfif:
      continue
    if m == 0xC0:
      for k, c in enumerate(ids):
        b[6 + 3 * k] = c
    if m == 0xDA:
      for k, c in enumerate(ids):
        b[1 + 2 * k] = c
    out.append((m, bytes(b)))
  return assemble(out, rest)


def bad_huffman(f, kind):
  """f with its first DC table over-subscribed ('over') or given a symbol above 15 ('dc16')."""
  segs, rest = segments(f)
  out = []
  for m, b in segs:
    if m == 0xC4 and b[0] == 0x00:
      b = bytearray(b)
      if kind == 'over':
        b[1 + 1] += 3                   # three more 2-bit codes than there is room for
        b[17 + sum(b[1:17]) - 3:17 + sum(b[1:17]) - 3] = bytes(3)
      else:
        b[17] = 16
      b = bytes(b)
    out.append((m, b))
  return assemble(out, rest)


def extra_rst_data(f):
  """f (with restart markers) with two bytes of data before its first RST and an RST after its
  last interval: libjpeg skips both."""
  k = f.index(b'\xff\xd0', len(f) - len(segments(f)[1]))
  f = f[:k] + b'\x5a\xa5' + f[k:]
  return f[:-2] + b'\xff\xd7\xff\xd9'


def handmade(seed=0):
  """[(name, file bytes)] of decodable files cv2 does not write itself: SOF1 with 16-bit tables
  (scaled so dequantized values overflow 16 bits), colour-space markers libjpeg reads as YCbCr,
  and data and RSTs libjpeg skips."""
  rng = np.random.default_rng(seed)
  f = encode(content('smooth', 40, 56, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90)
  g = encode(content('noise', 33, 47, 1, rng)[..., 0], cv2.IMWRITE_JPEG_QUALITY, 50)
  out = [('sof1 16-bit x%d' % s, sixteen_bit_tables(f, s)) for s in (1, 16, 256, 4096)]
  out.append(('sof1 16-bit gray x64', sixteen_bit_tables(g, 64)))
  out += [('ids 1,2,3 no JFIF', component_ids(f, (1, 2, 3), jfif=False)),
          ('ids R,G,B with JFIF', component_ids(f, (82, 71, 66))),
          ('JFIF and Adobe 0', component_ids(f, (1, 2, 3), adobe=0)),
          ('Adobe 1 no JFIF', component_ids(f, (1, 2, 3), jfif=False, adobe=1)),
          ('extra data and RST', extra_rst_data(encode(content('smooth', 40, 56, 3, rng),
                                                       cv2.IMWRITE_JPEG_RST_INTERVAL, 2)))]
  return out


# ---- files other encoders write, camera sizes, EXIF as cv2 reads it, and refusals ------------------
def _foreign_sources(rng):
  """(name, cv2 file) covering every sampling, odd sizes, grayscale and q50-100."""
  out = []
  for kind, (h, w), samp, q in (('noise', (37, 53), 0x111111, 100), ('check', (45, 70), 0x211111, 90),
                                ('smooth', (61, 97), 0x121111, 75), ('noise', (33, 47), 0x221111, 50),
                                ('smooth', (29, 83), 0x411111, 95), ('check', (26, 35), 0x221111, 100)):
    out.append(('%s %dx%d s%06x q%d' % (kind, h, w, samp, q),
                encode(content(kind, h, w, 3, rng), cv2.IMWRITE_JPEG_QUALITY, q,
                       cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)))
  for kind, (h, w), q in (('check', (23, 41), 60), ('smooth', (50, 38), 85)):
    out.append(('%s %dx%d gray q%d' % (kind, h, w, q),
                encode(content(kind, h, w, 1, rng)[..., 0], cv2.IMWRITE_JPEG_QUALITY, q)))
  return out


def _variants(nc, mcols, mcus, thumb):
  """name -> write() settings for a source of nc components and mcols x (mcus / mcols) MCUs."""
  odd = next(r for r in range(3, 64) if mcols % r and r % mcols)
  v = {
      'tables 0 for all': dict(huff=[(0, 0)] * nc),
      'luma on 3,2': dict(huff=[(3, 2)] + [(1, 1)] * (nc - 1)),
      'optimal': dict(tables='optimal'),
      'skewed': dict(tables='skewed'),
      'full 256': dict(tables='full'),
      'joint segments': dict(pack='joint', tables='optimal'),
      'redefined tables': dict(redefine=True),
      'sof1': dict(sof=0xC1),
      'rst 1': dict(restart=1),
      'rst %d (not a row)' % odd: dict(restart=odd, tables='optimal'),
      'rst past the end': dict(restart=mcus + 7),
      'rst 2 fill bytes': dict(restart=2, rst_fill=3),
      'rst 1 0-padded': dict(restart=1, pad_bit=0, tables='skewed'),
      '0-padded': dict(pad_bit=0),
      'COM APP2 XMP': dict(before=(W.COM, W.ICC, W.XMP), after_sof=(W.COM,)),
      'EXIF thumbnail': dict(before=(W.exif(1, True, thumb),), jfif=False),
      'fill between segments': dict(fill=2, redefine=True),
      'everything': dict(huff=[(3, 1), (1, 2), (2, 0)][:nc], tables='skewed', pack='joint',
                         redefine=True, sof=0xC1, restart=odd, rst_fill=1, pad_bit=0,
                         before=(W.COM, W.exif(1, False, thumb), W.XMP), fill=1, jfif=False,
                         quant=[3, 0, 2][:nc], halve_cr=nc == 3),
  }
  if nc == 3:
    v.update({
        'chroma on 2,3': dict(huff=[(0, 0), (2, 3), (2, 3)]),
        'Cb, Cr apart': dict(huff=[(3, 1), (1, 2), (2, 0)], tables='optimal'),
        'Cr on quant 2': dict(quant=[0, 1, 2]),
        'quant 3, 0, 2': dict(quant=[3, 0, 2], tables='full'),
        'Cr quant halved': dict(quant=[0, 1, 2], halve_cr=True),
    })
  return v


def foreign(seed=0):
  """[(name, file bytes, source file)]: cv2 files of every sampling, odd sizes, grayscale, noise, checkerboard
  and smooth content at q50-100, transcoded by tests/jpeg_writer.py into what other encoders
  write.  Each decodes (in cv2) to its source's pixels."""
  rng = np.random.default_rng(seed)
  thumb = encode(content('smooth', 12, 16, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 70)
  out = []
  for sname, f in _foreign_sources(rng):
    info, grids = W.source(f)
    _, mcols, mrows = D.mcu_geometry(info)
    for vname, kw in _variants(len(info.comps), mcols, mcols * mrows, thumb).items():
      out.append(('%s, %s' % (sname, vname), W.write(info, grids, **kw), f))
  return out


def _tiff_entry(tag, typ, count, value4, e):
  return tag.to_bytes(2, e) + typ.to_bytes(2, e) + count.to_bytes(4, e) + value4


def _exif_body(entries, e, ifd1=None):
  """'Exif\\0\\0' and a TIFF header in byte order e with IFD0 `entries` (and IFD1 `ifd1`)."""
  r = lambda v, n: v.to_bytes(n, e)
  t = (b'II' if e == 'little' else b'MM') + r(42, 2) + r(8, 4) + r(len(entries), 2) + b''.join(entries)
  if ifd1 is None:
    return b'Exif\x00\x00' + t + r(0, 4)
  return b'Exif\x00\x00' + t + r(len(t) + 4, 4) + r(len(ifd1), 2) + b''.join(ifd1) + r(0, 4)


def exif_variants(seed=0):
  """[(name, file bytes, the orientation cv2 applies)]: Orientation entries of every type, count,
  byte order and placement, on a 13x21 noise file at q100 4:4:4 whose eight orientations all
  differ."""
  rng = np.random.default_rng(seed)
  f = encode(content('noise', 13, 21, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 100,
             cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x111111)
  B, L = 'big', 'little'
  o = lambda typ, cnt, v4, e=B: _tiff_entry(0x0112, typ, cnt, v4, e)
  short = lambda v, e=B: v.to_bytes(2, e) + b'\x00\x00'
  rows = [
      ('SHORT 6 big-endian', _exif_body([o(3, 1, short(6))], B), 6),
      ('SHORT 6 little-endian', _exif_body([o(3, 1, short(6, L), L)], L), 6),
      ('LONG 6 little-endian', _exif_body([o(4, 1, (6).to_bytes(4, L), L)], L), 6),
      ('type 0, 6 in the first two bytes', _exif_body([o(0, 1, short(6))], B), 6),
      ('ends after the value\'s first two bytes', _exif_body([o(3, 1, short(6))], B)[:6 + 8 + 2 + 10], 6),
      ('LONG 6 big-endian', _exif_body([o(4, 1, (6).to_bytes(4, B))], B), 1),
      ('BYTE 6 big-endian', _exif_body([o(1, 1, b'\x06\x00\x00\x00')], B), 1),
      ('SHORT 6 count 0', _exif_body([o(3, 0, short(6))], B), 6),
      ('SHORT 6 count 2', _exif_body([o(3, 2, short(6))], B), 6),
      ('6 then 3', _exif_body([o(3, 1, short(6)), o(3, 1, short(3))], B), 6),
      ('only in IFD1', _exif_body([_tiff_entry(0x010F, 2, 4, b'abc\x00', B)], B, [o(3, 1, short(6))]), 1),
      ('value 0', _exif_body([o(3, 1, short(0))], B), 1),
      ('value 9', _exif_body([o(3, 1, short(9))], B), 1),
      ('SHORT 8 little-endian', _exif_body([o(3, 1, short(8, L), L)], L), 8),
  ]
  out = [(name, f[:2] + W.segment(0xE1, body) + f[2:], want) for name, body, want in rows]
  out.append(('XMP before the Exif', f[:2] + W.XMP + W.segment(0xE1, rows[0][1]) + f[2:], 6))
  return out


def camera(seed=0):
  """[(name, file bytes)] at camera sizes, none a multiple of 16 in both sides: 12 MP smooth 4:2:0
  with EXIF orientation 6 and a thumbnail, 12 MP 4:2:2 at orientation 8 with a restart interval of
  one MCU row, a 4032x3024 noise file at q100 4:4:4 (about 50 MB), and 1x8191 and 8191x1."""
  rng = np.random.default_rng(seed)
  thumb = encode(content('smooth', 120, 160, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 80)
  a = encode(content('smooth', 3000, 4000, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 92)
  b = encode(content('smooth', 4000, 3000, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 95,
             cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x211111, cv2.IMWRITE_JPEG_RST_INTERVAL, 3000 // 16 + 1)
  return [('4000x3000 q92 s221111 exif 6', a[:2] + W.exif(6, True, thumb) + a[2:]),
          ('3000x4000 q95 s211111 rst row exif 8', with_orientation(b, 8)),
          ('4032x3024 noise q100 s111111', encode(content('noise', 3024, 4032, 3, rng),
                                                  cv2.IMWRITE_JPEG_QUALITY, 100,
                                                  cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x111111)),
          ('1x8191', encode(content('smooth', 1, 8191, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90)),
          ('8191x1', encode(content('smooth', 8191, 1, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90))]


def refused(seed=0):
  """[(name, file bytes, reason, whether cv2 decodes it)]: files the decoder refuses by design.
  libjpeg-turbo refuses a scan whose components are in another order than the frame's (its
  component lookup skips an id already placed at the same index), so cv2 returns None for those."""
  rng = np.random.default_rng(seed)
  f = encode(content('smooth', 30, 44, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90,
             cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x111111)
  g = encode(content('smooth', 30, 44, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90)
  info, grids = W.source(f)
  info2, grids2 = W.source(g)
  return [('SOS order Y, Cr, Cb', W.write(info, grids, order=(0, 2, 1)), D.SAMPLING, False),
          ('SOS order Cb, Y, Cr', W.write(info, grids, order=(1, 0, 2)), D.SAMPLING, False),
          ('Y and Cb 2x2, Cr 1x1', W.write(info2, [grids2[0], grids2[0], grids2[2]],
                                           sampling=[(2, 2), (2, 2), (1, 1)]), D.SAMPLING, True),
          ('bytes before a marker', W.write(info, grids, before=(b'\x00\x5a',)), D.MALFORMED, True)]
