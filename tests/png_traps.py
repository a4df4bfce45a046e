"""Images that drive cv2's PNG writer (libpng + zlib Z_RLE) into each of its corner cases, shared by
the oracle tests and the device tests.  Each is paired with a check of the oracle's `info` that the
case really occurs."""
import numpy as np

from oracle import png as opng


def from_filtered(payload):
  """The BGR image (w > 1) whose filtered rows are `payload` [h, 3 w] after the SUB filter byte."""
  payload = np.asarray(payload, np.uint8)
  h, n = payload.shape
  rgb = np.cumsum(payload.reshape(h, n // 3, 3).astype(np.int64), axis=1) % 256
  return np.ascontiguousarray(rgb[:, :, ::-1].astype(np.uint8))


def _runs_payload():
  """Runs of every length class: 1..6, 258 + 1 .. 258 + 4 (the remainder after a full match of 0,
  1, 2 or 3 bytes), 516 + 1 .. + 4, separated by other bytes, and a run that ends a row and
  continues through the next row's filter byte 0x01."""
  parts, v = [], 10
  for L in list(range(1, 7)) + [259, 260, 261, 262, 263, 517, 518, 519, 520]:
    parts.append(np.full(L, v, np.uint8))
    parts.append(np.array([v + 1], np.uint8))
    v = (v + 7) % 250 + 2
  row = np.concatenate(parts)
  w = -(-len(row) // 3)
  row = np.concatenate([row, np.full(3 * w - len(row), 1, np.uint8)])   # ends in 0x01s
  return np.stack([row, np.roll(row, 5), np.full(3 * w, 1, np.uint8), row])


def _fibonacci_payload():
  """One row whose literal counts follow the Fibonacci numbers, with the end-of-block code and the
  filter byte as the two 1s: a Huffman tree 18 deep, repaired to 15.  No byte repeats 4 times in a
  row, so there are no matches to disturb the counts."""
  fib = [1, 1]
  while len(fib) < 19:
    fib.append(fib[-1] + fib[-2])
  left = fib[2:]
  left[-1] += 1                                          # 10944 bytes: 3648 pixels
  vals = np.arange(17) * 13 + 3
  out = []
  while sum(left):
    for k in sorted(range(17), key=lambda k: -left[k]):
      if left[k] and not (len(out) >= 3 and out[-1] == out[-2] == out[-3] == vals[k]):
        out.append(vals[k])
        left[k] -= 1
        break
  return np.array(out, np.uint8)[None, :]


def _small_alphabet(h, w, seed):
  """Bytes 0..7 with no run of 4, so no match: a dynamic block with two forced distance codes."""
  rng = np.random.default_rng(seed)
  p = rng.integers(0, 8, (h, 3 * w)).astype(np.uint8)
  flat = p.reshape(-1)
  for i in range(3, len(flat)):
    if flat[i] == flat[i - 1] == flat[i - 2] == flat[i - 3]:
      flat[i] = (flat[i] + 1) % 8
  return p


def _idat_multiple():
  img = np.random.default_rng(2).integers(0, 256, (60, 100, 3), dtype=np.uint8)
  img.reshape(-1, 3)[6000 - 582:] = 0
  return img


def runs_of(data):
  """(start, length) of every maximal run of equal bytes in `data`."""
  d = np.asarray(data, np.uint8)
  starts = np.flatnonzero(np.append(True, d[1:] != d[:-1]))
  return list(zip(starts.tolist(), np.diff(np.append(starts, len(d))).tolist()))


def run_symbols(L):
  """The (offset, length) symbols deflate_rle codes a run of L equal bytes as: one literal, matches
  of min(258, R) while the R bytes left are 3 or more, then R literals."""
  out, o, r = [(0, 1)], 1, L - 1
  while r >= 3:
    m = min(258, r)
    out.append((o, m))
    o, r = o + m, r - m
  return out + [(o + k, 1) for k in range(r)]


def check_runs(img, info):
  """Every run of 259 bytes or more is parsed as run_symbols says, the bytes left after its full
  258-byte matches number 0, 1, 2 and 3 or more in some run each, and a match covers a row's filter
  byte in the middle of a run that crosses into that row."""
  data = opng.filter_rows(img)
  pos, length = info['parse']
  sym = dict(zip(pos.tolist(), length.tolist()))
  classes = set()
  for a, L in runs_of(data):
    if L < 259:
      continue
    got = [(p - a, sym[p]) for p in range(a, a + L) if p in sym]
    if got != run_symbols(L):
      return False
    classes.add(min((L - 1) % 258, 3))
  row = 3 * img.shape[1] + 1
  crossing = any(ln > 1 and p % row and (p // row + 1) * row < p + ln
                 for p, ln in zip(pos.tolist(), length.tolist()))
  return classes == {0, 1, 2, 3} and crossing


def check_one_literal(info, data):
  pos, length = info['parse']
  return len(set(data[pos[length == 1]].tolist())) == 1 and info['matches'] > 0


# name -> (image, check of encode's info)
def traps():
  noise = np.random.default_rng(0)
  runs = from_filtered(_runs_payload())
  one = np.tile(np.arange(1, 301, dtype=np.uint8)[None, :, None], (50, 1, 3))
  return {
      'stored_then_empty_final': (noise.integers(0, 256, (3, 1820, 3), dtype=np.uint8),
                                  lambda i: i['symbols'] == 16383 and i['blocks'] == ['stored', 'static']),
      'two_stored_then_empty_final': (np.random.default_rng(1).integers(0, 256, (6, 1820, 3), dtype=np.uint8),
                                      lambda i: i['symbols'] == 2 * 16383 and
                                      i['blocks'] == ['stored', 'stored', 'static']),
      'dynamic_then_empty_final': (from_filtered(_small_alphabet(3, 1820, 5)),
                                   lambda i: i['symbols'] == 16383 and i['blocks'] == ['dynamic', 'static']),
      'no_matches': (from_filtered(_small_alphabet(40, 60, 6)),
                     lambda i: i['matches'] == 0 and i['blocks'] == ['dynamic']),
      'runs': (runs, lambda i: check_runs(runs, i)),
      'one_literal_value': (one, lambda i: check_one_literal(i, opng.filter_rows(one))),
      'repaired_at_15_bits': (from_filtered(_fibonacci_payload()),
                              lambda i: i['repaired'] >= 1 and i['blocks'] == ['dynamic']),
      'idat_multiple_of_8192': (_idat_multiple(),
                                lambda i: i['zlib_bytes'] == 16384 and i['idat'] == [8192, 8192]),
      'stored_blocks': (noise.integers(0, 256, (100, 300, 3), dtype=np.uint8),
                        lambda i: 'stored' in i['blocks']),
      'flat_rows': (np.full((40, 700, 3), 9, np.uint8), lambda i: i['blocks'] == ['dynamic']),
  }


def header_widths():
  """One-row widths around every filtered-data size where libpng's zlib window or optimize_cmf's
  window field changes (sizes 2^k - 262 and 2^k for k = 8 .. 14): every header byte pair."""
  ws = set()
  for k in range(8, 15):
    for edge in (2 ** k - 262, 2 ** k):
      base = (edge - 1) // 3
      ws.update(w for w in range(base - 1, base + 3) if w >= 1)
  return sorted(ws | {1, 2, 3})
