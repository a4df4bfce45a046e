"""JPEG files for the decoder's tests, all made by cv2.imencode from seeded content: the content
kinds of test_gpu_jpeg (noise, gradients, flat, checkerboards of pixels and of 8x8 blocks, dots)
plus a smooth picture, over sizes, qualities, samplings, restart intervals, optimized Huffman
tables, separate luma and chroma qualities, grayscale and EXIF orientations."""
import cv2
import numpy as np

from oracle.jpeg_decode import with_orientation

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
