"""Progressive files of foreign scan scripts: a baseline file's coefficients (oracle.jpeg_decode)
rewritten as SOF2 with any list of scans, as other encoders (jpegtran, mozjpeg) write them.

write(f, script, ...) -> bytes.  A scan is (components, Ss, Se, Ah, Al) with frame component
indices; each coded scan carries its own optimal tables (DHT before its SOS), coded as
oracle.jpeg_progressive codes cv2's scans (EOBRUN up to 0x7FFF, correction bits buffered behind
it).  `restarts` gives a scan's restart interval (a DRI before it whenever it changes), and
`dqt_after` redefines every quantization table with junk after that scan, which must not change
the pixels of components already scanned.  For every complete script cv2 decodes the file to the
baseline file's pixels."""
import numpy as np

from oracle import jpeg_decode as D
from oracle import jpeg_decode_progressive as P
from oracle.jpeg import _pack, huffman_codes
from oracle.jpeg_params import optimal_table
from oracle.jpeg_progressive import CAUSES, _dht, _scan_items, _seg

# scripts of complete files (every coefficient of every component down to bit 0)
SPECTRAL = [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 5, 0, 0), ((0,), 6, 63, 0, 0), ((2,), 1, 63, 0, 0),
            ((1,), 1, 63, 0, 0)]
DEEP = ([((0, 1, 2), 0, 0, 0, 13)] + [((c,), 1, 63, 0, 13) for c in (0, 1, 2)]
        + [s for a in range(12, -1, -1)
           for s in [((0, 1, 2), 0, 0, a + 1, a)] + [((c,), 1, 63, a + 1, a) for c in (0, 1, 2)]])
PER_COEF = [((0, 1, 2), 0, 0, 0, 0)] + [((c,), k, k, 0, 0) for c in (0, 1, 2) for k in range(1, 64)]
DC_CHAINS = ([((c,), 0, 0, 0, 3) for c in (2, 0, 1)] + [((c,), 0, 0, a + 1, a) for a in (2, 1, 0)
                                                        for c in (0, 1, 2)]
             + [((c,), 1, 63, 0, 1) for c in (0, 1, 2)] + [((c,), 1, 63, 1, 0) for c in (1, 0, 2)])
DC_SUBSETS = [((0, 1), 0, 0, 0, 1), ((2,), 0, 0, 0, 1), ((1, 2), 0, 0, 1, 0), ((0,), 0, 0, 1, 0),
              ((0,), 1, 9, 0, 2), ((0,), 10, 63, 0, 0), ((0,), 1, 9, 2, 1), ((1,), 1, 63, 0, 0),
              ((2,), 1, 63, 0, 0), ((0,), 1, 9, 1, 0)]
GRAY_DEEP = [((0,), 0, 0, 0, 4), ((0,), 1, 2, 0, 3), ((0,), 3, 63, 0, 2), ((0,), 0, 0, 4, 3),
             ((0,), 0, 0, 3, 2), ((0,), 0, 0, 2, 1), ((0,), 0, 0, 1, 0), ((0,), 1, 2, 3, 2),
             ((0,), 1, 63, 2, 1), ((0,), 1, 63, 1, 0)]
COMPLETE = {'spectral': SPECTRAL, 'deep': DEEP, 'per coefficient': PER_COEF,
            'dc chains': DC_CHAINS, 'dc subsets': DC_SUBSETS}
# incomplete scripts libjpeg does not smooth: refinement missing above coefficient 9, and Cr
# never coded (no DC scan)
UNSMOOTHED = {'no refinement above 9': [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 9, 0, 0),
                                        ((0,), 10, 63, 0, 2), ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0)],
              'no Cr': [((0, 1), 0, 0, 0, 0), ((0,), 1, 63, 0, 0), ((1,), 1, 63, 0, 0)]}
SMOOTHED = {'no AC refinement': [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 63, 0, 1), ((1,), 1, 63, 0, 0),
                                 ((2,), 1, 63, 0, 0)],
            'DC only': [((0, 1, 2), 0, 0, 0, 0)]}
BAD = {'AC over two components': [((0, 1, 2), 0, 0, 0, 0), ((0, 1), 1, 63, 0, 0)],
       'Al 14': [((0, 1, 2), 0, 0, 0, 14)],
       'Ah 2 Al 0': [((0, 1, 2), 0, 0, 0, 2), ((0, 1, 2), 0, 0, 2, 0)],
       'DC with Se 5': [((0, 1, 2), 0, 5, 0, 0)],
       'Ss above Se': [((0, 1, 2), 0, 0, 0, 0), ((0,), 9, 3, 0, 0)]}
BOGUS = {'AC before DC': [((0,), 1, 63, 0, 0), ((0, 1, 2), 0, 0, 0, 0), ((1,), 1, 63, 0, 0),
                          ((2,), 1, 63, 0, 0)],
         'Ah not the last Al': [((0, 1, 2), 0, 0, 0, 2), ((0, 1, 2), 0, 0, 1, 0)] +
                               [((c,), 1, 63, 0, 0) for c in (0, 1, 2)],
         # libjpeg does not warn on a second first scan of a coefficient whose last Al was 0: it
         # overwrites the coefficients, which the device decoder's parallel first scans cannot
         'first scan twice': [((0, 1, 2), 0, 0, 0, 0)] + [((c,), 1, 63, 0, 0) for c in (0, 1, 2)] +
                             [((0,), 1, 5, 0, 0)]}


def source(f):
  """(Info, per-component coefficient grids) of a baseline file."""
  info = D.parse(f)
  return info, D.decode_coefficients(f, info)


def write(f, script, restarts=None, dqt_after=None):
  info, grids = source(f)
  comps = info.comps
  nc = len(comps)
  shapes = P.grid_shapes(info)
  out = bytearray(b'\xff\xd8' + _seg(0xE0, b'JFIF\x00' + bytes([1, 1, 0, 0, 1, 0, 1, 0, 0])))
  for t, q in sorted(info.qt.items()):
    out += _seg(0xDB, bytes([t]) + bytes(int(v) for v in q[D.ZIGZAG]))
  sof = bytes([8, info.height >> 8, info.height & 255, info.width >> 8, info.width & 255, nc])
  for c in comps:
    sof += bytes([c.cid, c.h << 4 | c.v, c.tq])
  out += _seg(0xC2, sof)
  counts = dict.fromkeys(CAUSES, 0)
  restart = 0
  for si, scan in enumerate(script):
    sc, ss, se, ah, al = scan
    sc = tuple(c for c in sc if c < nc)
    units = P._units(info, P.Scan(list(sc), ss, se, ah, al, [], 0, 0, 0), shapes)
    rows = np.array([grids[ci][by, bx][D.ZIGZAG] for u in units for ci, by, bx in u], np.int64)
    ucomp = np.array([ci for u in units for ci, _, _ in u])
    per = len(units[0])
    want = (restarts or {}).get(si, restart)
    if want != restart:
      out += _seg(0xDD, want.to_bytes(2, 'big'))
      restart = want
    items = _scan_items(rows, ucomp, np.zeros(len(rows), bool), per, (sc, ss, se, ah, al), restart,
                        counts)
    codes = {}
    if ss or ah == 0:
      flat = [it for iv in items for it in iv if it[0] == 's']
      for t in sorted({it[1] for it in flat}):
        freq = {}
        for it in flat:
          if it[1] == t:
            freq[it[2]] = freq.get(it[2], 0) + 1
        table = optimal_table(freq)
        codes[t] = huffman_codes(*table)
        out += _dht((0x10 if ss else 0) | (int(sc[0] > 0) if ss else t), table)
    body = [len(sc)]
    for c in sc:
      body += [comps[c].cid, (int(c > 0) if ss else (0x10 if c else 0)) if ss == 0 else int(c > 0)]
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
    if dqt_after == si:
      for t in sorted(info.qt):
        out += _seg(0xDB, bytes([t]) + bytes(range(1, 65)))
  return bytes(out + b'\xff\xd9')


def scan_data_end(f, index):
  """The offset of the marker that ends the entropy-coded data of scan `index`."""
  at = [i for i in range(len(f) - 1) if f[i] == 0xFF and f[i + 1] == 0xDA][index]
  return P._data_end(f, at + 2 + int.from_bytes(f[at + 2:at + 4], 'big'))


def with_trailing_rst(f, index=0, count=1):
  """f with `count` RSTn markers after scan `index`'s last interval, which libjpeg skips."""
  k = scan_data_end(f, index)
  return f[:k] + b''.join(bytes([0xFF, 0xD0 + i % 8]) for i in range(count)) + f[k:]


def with_dri(f, interval):
  """f with a DRI segment after SOI: every scan then needs RSTn markers it does not have."""
  return f[:2] + _seg(0xDD, interval.to_bytes(2, 'big')) + f[2:]
