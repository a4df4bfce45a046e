#!/usr/bin/env python
"""Recovers OpenCV's FONT_HERSHEY_SIMPLEX strokes for ASCII 32..126 from the installed cv2 and
writes them as squeezedet_b200/csrc/hershey_simplex.inc, the table sqdet_draw_dets' kernel and
oracle.draw render labels from.

    python -m oracle.make_hershey            # rewrites the header
    python -m oracle.make_hershey --check    # exits 1 when the header differs from a fresh run

putText places every glyph vertex at pen + (u, v) * hscale in 16.16 fixed point, u and v integer
font units, and joins vertices with 1-px lines.  At an integer font scale S every vertex therefore
lands on the pixel lattice org + S * (u, v) and every stroke is the integer line between two lattice
points.  For each glyph:
  1. render it alone at scale S (`raster`);
  2. keep the pairs of set lattice points whose cv2.line lies inside the raster, and of those the
     maximal ones (a pair on a longer kept pair's segment is part of that stroke);
  3. check that the kept lines reproduce the raster exactly, at two scales;
  4. orient each segment as putText draws it.  cv2.clipLine moves an endpoint outside the canvas
     by an intercept truncated toward zero from the *first* endpoint, so a segment cut by the
     canvas edge can draw different pixels in its two directions; the direction whose pixels
     stay inside cv2's render on small canvases cut through the segment at fractional scales is
     the one kept (segments whose two directions never differ keep either);
  5. take the advance from getTextSize (thickness 0 adds nothing) and check it against the
     offset of a second glyph in a two-glyph string;
  6. check the whole table against cv2.putText through oracle.draw, in and across the canvas
     edges, at fractional scales."""
import argparse
import itertools
import os
import sys

import numpy as np

FONT_SCALES = (13, 17)        # two integer scales; lattice pairs must agree at both
ORG = (16, 40)                # pen position in font units from the canvas' top-left corner
SIZE = (64, 72)               # canvas height, width in font units: every glyph fits inside
ORIENT_SCALES = (0.3, 0.5, 1.0, 1.7, 2.3, 3.0, 5.0, 7.3)
ORIENT_TRIALS = 240           # small cut canvases per segment
CHECK_TRIALS = 400            # random clipped renders per glyph in the final check


def _render(cv2, text, scale, org, shape):
  img = np.zeros(shape, np.uint8)
  cv2.putText(img, text, org, cv2.FONT_HERSHEY_SIMPLEX, scale, 255, 1, cv2.LINE_8)
  return img


def _segments_at(cv2, ch, S):
  """The glyph's maximal lattice segments at integer scale S, in font units."""
  shape = (SIZE[0] * S + 1, SIZE[1] * S + 1)
  org = (ORG[0] * S, ORG[1] * S)
  raster = _render(cv2, ch, S, org, shape)
  ys, xs = np.nonzero(raster)
  if len(xs) == 0:
    return raster, org, []
  if xs.min() == 0 or ys.min() == 0 or xs.max() == shape[1] - 1 or ys.max() == shape[0] - 1:
    raise RuntimeError('glyph %r reaches the edge of its canvas' % ch)
  pts = sorted({((x - org[0]) // S, (y - org[1]) // S) for x, y in zip(xs, ys)
                if (x - org[0]) % S == 0 and (y - org[1]) % S == 0})
  x0, x1, y0, y1 = xs.min(), xs.max() + 1, ys.min(), ys.max() + 1
  inside = raster[y0:y1, x0:x1] > 0
  cand = []
  scratch = np.zeros_like(inside, np.uint8)
  for a, b in itertools.combinations(pts, 2):
    scratch[:] = 0
    cv2.line(scratch, (org[0] + a[0] * S - x0, org[1] + a[1] * S - y0),
             (org[0] + b[0] * S - x0, org[1] + b[1] * S - y0), 1, 1, cv2.LINE_8)
    on = scratch > 0
    if not (on & ~inside).any():
      cand.append((a, b))

  def covers(big, small):
    (ax, ay), (bx, by) = big
    for px, py in small:
      if (bx - ax) * (py - ay) - (by - ay) * (px - ax) != 0:
        return False
      if not (min(ax, bx) <= px <= max(ax, bx) and min(ay, by) <= py <= max(ay, by)):
        return False
    return True

  keep = [s for s in cand if not any(t != s and covers(t, s) for t in cand)]
  return raster, org, sorted(keep)


def _draw_segments(cv2, segs, S, org, shape):
  img = np.zeros(shape, np.uint8)
  for (ax, ay), (bx, by) in segs:
    cv2.line(img, (org[0] + ax * S, org[1] + ay * S), (org[0] + bx * S, org[1] + by * S), 255, 1,
             cv2.LINE_8)
  return img


def _pixels(draw, seg, org, hs, h, w):
  """oracle.draw's pixels of one glyph segment at pen position `org`."""
  x0, y0, x1, y1 = seg
  vx, vy = org[0] << 16, org[1] << 16
  r = lambda v: draw._i32((v + 0x8000) >> 16)  # noqa: E731
  return draw.line_pixels(w, h, r(vx + x0 * hs), r(vy + y0 * hs), r(vx + x1 * hs), r(vy + y1 * hs))


def _orient(cv2, ch, segs, rng):
  """Each segment in the direction putText draws it (step 4)."""
  from oracle import draw
  out = []
  for s in segs:
    both = (s, (s[2], s[3], s[0], s[1]))
    bad = [0, 0]
    for _ in range(ORIENT_TRIALS):
      sc = rng.choice(ORIENT_SCALES)
      hs = draw.hscale(sc)
      h, w, t = rng.randint(1, 8), rng.randint(1, 8), rng.random()
      px = (s[0] + t * (s[2] - s[0])) * hs / 65536.0
      py = (s[1] + t * (s[3] - s[1])) * hs / 65536.0
      org = (int(round(-px)) + rng.randrange(w), int(round(-py)) + rng.randrange(h))
      inside = _render(cv2, ch, sc, org, (h, w)) > 0
      for d, seg in enumerate(both):
        bad[d] += any(not inside[y, x] for x, y in _pixels(draw, seg, org, hs, h, w))
    if bad[0] and bad[1]:
      raise RuntimeError('glyph %r: segment %s fits neither direction' % (ch, s))
    out.append(both[1] if bad[0] else s)
  return out


def _check(cv2, ch, segs, rng):
  """Step 6 for one glyph: random canvases, origins and scales, most of them clipping."""
  from oracle import draw
  for _ in range(CHECK_TRIALS):
    sc = rng.choice(ORIENT_SCALES)
    hs = draw.hscale(sc)
    h, w = rng.randint(1, 40), rng.randint(1, 40)
    org = (rng.randint(int(-25 * sc) - 2, w + 2), rng.randint(-2, h + int(25 * sc) + 2))
    want = _render(cv2, ch, sc, org, (h, w)) > 0
    got = np.zeros((h, w), bool)
    for seg in segs:
      for x, y in _pixels(draw, seg, org, hs, h, w):
        got[y, x] = True
    if not np.array_equal(got, want):
      raise RuntimeError('glyph %r differs from cv2.putText at scale %g, origin %s on %dx%d'
                         % (ch, sc, org, w, h))


def recover(cv2):
  """[(advance, [(x0, y0, x1, y1), ...])] for ASCII 32..126."""
  import random
  font = cv2.FONT_HERSHEY_SIMPLEX
  rng = random.Random(2024)
  out = []
  for code in range(32, 127):
    ch = chr(code)
    found = []
    for S in FONT_SCALES:
      raster, org, segs = _segments_at(cv2, ch, S)
      if not np.array_equal(_draw_segments(cv2, segs, S, org, raster.shape), raster):
        raise RuntimeError('glyph %r: the recovered strokes do not reproduce the raster at scale %d'
                           % (ch, S))
      found.append(segs)
    if found[0] != found[1]:
      raise RuntimeError('glyph %r: different strokes at scales %s' % (ch, FONT_SCALES))
    (adv, _), _ = cv2.getTextSize(ch, font, 1.0, 0)
    # cross-check: the second glyph of ch + '|' starts `adv` font units right of where '|' alone does
    S = FONT_SCALES[0]
    shape, org = (SIZE[0] * S + 1, SIZE[1] * S + 1), (ORG[0] * S, ORG[1] * S)
    bar = np.nonzero(_render(cv2, '|', S, org, shape).any(axis=0))[0].min()
    two = _render(cv2, ch + '|', S, org, shape) - _render(cv2, ch, S, org, shape)
    if np.nonzero(two.any(axis=0))[0].min() != bar + adv * S:
      raise RuntimeError('glyph %r: advance %d disagrees with a two-glyph render' % (ch, adv))
    segs = _orient(cv2, ch, [(a[0], a[1], b[0], b[1]) for a, b in found[0]], rng)
    _check(cv2, ch, segs, rng)
    out.append((adv, segs))
  return out


def header(glyphs):
  lines = ['/* FONT_HERSHEY_SIMPLEX strokes for ASCII 32..126, recovered from OpenCV\'s putText by',
           ' * oracle/make_hershey.py.  Generated: do not edit.',
           ' *',
           ' * A glyph at pen position (px, py) (16.16 fixed point, py the text origin\'s row) with',
           ' * hscale = cvRound(font_scale * 65536) draws each segment (x0, y0, x1, y1) from',
           ' * (px + x0 * hscale, py + y0 * hscale) to (px + x1 * hscale, py + y1 * hscale), then moves',
           ' * the pen by advance * hscale.  y grows downwards, as in the image. */',
           '#ifndef SQDET_HERSHEY_SPACE',
           '#define SQDET_HERSHEY_SPACE  /* a CUDA source defines it as __constant__ */',
           '#endif',
           '#define SQDET_HERSHEY_SEGMENTS %d' % sum(len(s) for _, s in glyphs),
           '/* per character: { advance, first segment, segment count } */',
           'static SQDET_HERSHEY_SPACE const short kHersheyGlyphs[95][3] = {']
  first = 0
  for code, (adv, segs) in zip(range(32, 127), glyphs):
    shown = chr(code) if chr(code) not in '*/\\' else '0x%02x' % code
    lines.append('  {%d, %d, %d}, /* glyph %d %s */' % (adv, first, len(segs), code, shown))
    first += len(segs)
  lines.append('};')
  lines.append('/* { x0, y0, x1, y1 } in font units */')
  lines.append('static SQDET_HERSHEY_SPACE const signed char '
               'kHersheySegments[SQDET_HERSHEY_SEGMENTS][4] = {')
  for segs in (s for _, s in glyphs):
    for x0, y0, x1, y1 in segs:
      lines.append('  {%d, %d, %d, %d},' % (x0, y0, x1, y1))
  lines.append('};')
  return '\n'.join(lines) + '\n'


def main(argv=None):
  ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  ap.add_argument('--check', action='store_true', help='compare with the committed header only')
  args = ap.parse_args(argv)
  import cv2
  from oracle import draw
  text = header(recover(cv2))
  if args.check:
    with open(draw.INC_PATH) as f:
      same = f.read() == text
    print('hershey_simplex.inc is %s' % ('up to date' if same else 'STALE'))
    return 0 if same else 1
  with open(draw.INC_PATH, 'w') as f:
    f.write(text)
  print('wrote', os.path.normpath(draw.INC_PATH))
  return 0


if __name__ == '__main__':
  sys.exit(main())
