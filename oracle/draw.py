"""CPU restatement of the detection drawing of sqdet_draw_dets — test infrastructure, like the rest
of oracle/.

The reference draws each kept detection with ``cv2.rectangle`` + ``cv2.putText`` (src/train.py:51-72
``_draw_box``, called by src/demo.py's ``draw_detections``; this package's ``utils.viz.draw_box``).
On a uint8 canvas with thickness 1 and LINE_8, OpenCV 4.13 draws both from one primitive, restated
here operation for operation and PINNED bitwise against the installed cv2
(tests/test_oracle_draw.py):

  line        the 8-connected integer line of cv2.LineIterator (left to right), after cv2.clipLine
              against the canvas: Cohen-Sutherland in int64 with double-precision intercepts;
  rectangle   the four edges (x1,y1)-(x2,y1)-(x2,y2)-(x1,y2)-(x1,y1) as lines;
  putText     FONT_HERSHEY_SIMPLEX: each glyph's segments at 16.16 fixed-point positions, pen
              advance and glyph offsets in units of hscale = cvRound(font_scale * 65536); each
              segment's endpoints are rounded to pixels ((v + 0x8000) >> 16, as int32) and drawn
              as a line.  The strokes come from squeezedet_b200/csrc/hershey_simplex.inc, which
              oracle/make_hershey.py recovers from the installed cv2.

Every pixel a record draws gets its colour, so a record is a mask (record_mask) and later records
overwrite earlier ones.  For 4:2:0 frames, which cv2 cannot draw on, the rule is this module's own
(draw_frame): luma takes the colour's Y on the mask; a chroma sample takes (U, V) when its 2x2
luma block, in frame coordinates, holds a mask pixel.  (Y, U, V) is cv2.cvtColor of a solid BGR
patch with COLOR_BGR2YUV_I420 (yuv_of_bgr, OpenCV's BT.601 fixed-point constants)."""
import math
import os
import re

import numpy as np

INC_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'squeezedet_b200', 'csrc',
                        'hershey_simplex.inc')
_FONT = None


def font():
  """{char: (advance, [(x0, y0, x1, y1), ...])} for ASCII 32..126, in font units relative to the
  pen position on the text origin's row, parsed from the generated header."""
  global _FONT
  if _FONT is None:
    with open(INC_PATH) as f:
      src = f.read()
    glyphs = [tuple(int(v) for v in m) for m in
              re.findall(r'\{\s*(-?\d+),\s*(-?\d+),\s*(-?\d+)\s*\},\s*/\* glyph', src)]
    segs = [tuple(int(v) for v in m) for m in
            re.findall(r'\{\s*(-?\d+),\s*(-?\d+),\s*(-?\d+),\s*(-?\d+)\s*\}', src)]
    assert len(glyphs) == 95, len(glyphs)
    _FONT = {chr(32 + i): (adv, segs[first:first + count])
             for i, (adv, first, count) in enumerate(glyphs)}
  return _FONT


def _i32(v):
  """C's (int) of an int64 that cv2 narrows to a Point."""
  return ((v + 2 ** 31) % 2 ** 32) - 2 ** 31


def clip_line(w, h, x1, y1, x2, y2):
  """cv2.clipLine(Size2l(w, h), pt1, pt2) -> (inside, x1, y1, x2, y2)."""
  if w <= 0 or h <= 0:
    return False, x1, y1, x2, y2
  right, bottom = w - 1, h - 1
  c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
  c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
  if (c1 & c2) == 0 and (c1 | c2) != 0:
    # float(a) * float(b) / float(c) is the C double expression; int() truncates toward zero
    if c1 & 12:
      a = 0 if c1 < 8 else bottom
      x1 += int(float(a - y1) * float(x2 - x1) / float(y2 - y1))
      y1 = a
      c1 = (x1 < 0) + (x1 > right) * 2
    if c2 & 12:
      a = 0 if c2 < 8 else bottom
      x2 += int(float(a - y2) * float(x2 - x1) / float(y2 - y1))
      y2 = a
      c2 = (x2 < 0) + (x2 > right) * 2
    if (c1 & c2) == 0 and (c1 | c2) != 0:
      if c1:
        a = 0 if c1 == 1 else right
        y1 += int(float(a - x1) * float(y2 - y1) / float(x2 - x1))
        x1 = a
        c1 = 0
      if c2:
        a = 0 if c2 == 1 else right
        y2 += int(float(a - x2) * float(y2 - y1) / float(x2 - x1))
        x2 = a
        c2 = 0
  return (c1 | c2) == 0, x1, y1, x2, y2


def line_pixels(w, h, x1, y1, x2, y2):
  """The (x, y) pixels cv2.line(canvas, (x1, y1), (x2, y2), c, 1, LINE_8) sets on an h x w canvas
  (int32 endpoints)."""
  if not (0 <= x1 < w and 0 <= x2 < w and 0 <= y1 < h and 0 <= y2 < h):
    inside, x1, y1, x2, y2 = clip_line(w, h, x1, y1, x2, y2)
    if not inside:
      return []
  dx, dy = x2 - x1, y2 - y1
  if dx < 0:                                   # leftToRight
    dx, dy, x1, y1 = -dx, -dy, x2, y2
  sy = -1 if dy < 0 else 1
  dy = abs(dy)
  vert = dy > dx
  if vert:
    dx, dy = dy, dx
  err, plus, minus = dx - 2 * dy, 2 * dx, -2 * dy
  x, y, out = x1, y1, []
  for _ in range(dx + 1):
    out.append((x, y))
    step = err < 0
    err += minus + (plus if step else 0)
    if vert:
      y += sy
      x += step
    else:
      x += 1
      y += sy if step else 0
  return out


def hscale(font_scale):
  """cvRound(font_scale * XY_ONE) of the float32 font scale (round half to even)."""
  return int(round(float(np.float32(font_scale)) * 65536.0))


def text_segments(text, org, hs):
  """putText's segments of `text` at integer origin `org`, each as rounded pixel endpoints."""
  table = font()
  view_x, view_y = org[0] << 16, org[1] << 16
  out = []
  for ch in text:
    adv, segs = table[ch]
    for x0, y0, x1, y1 in segs:
      out.append(tuple(_i32((v + 0x8000) >> 16) for v in
                       (view_x + x0 * hs, view_y + y0 * hs, view_x + x1 * hs, view_y + y1 * hs)))
    view_x += adv * hs
  return out


def _mark(mask, pixels):
  for x, y in pixels:
    mask[y, x] = True


def put_text_mask(mask, text, org, font_scale):
  """cv2.putText(canvas, text, org, FONT_HERSHEY_SIMPLEX, font_scale, c, 1) as pixels on `mask`."""
  h, w = mask.shape
  for s in text_segments(text, org, hscale(font_scale)):
    _mark(mask, line_pixels(w, h, *s))


def rectangle_mask(mask, x1, y1, x2, y2):
  """cv2.rectangle(canvas, (x1, y1), (x2, y2), c, 1) as pixels on `mask`."""
  h, w = mask.shape
  for a, b in (((x1, y1), (x2, y1)), ((x2, y1), (x2, y2)), ((x2, y2), (x1, y2)),
               ((x1, y2), (x1, y1))):
    _mark(mask, line_pixels(w, h, a[0], a[1], b[0], b[1]))


def prob_label(prob):
  """'%.2f' % prob for a float32 prob, restated in the integers the kernel uses: the exact value
  times 100, rounded half to even.  None outside [0, 1] (no label is drawn)."""
  p = np.float32(prob)
  if not (0.0 <= p <= 1.0):
    return None
  bits = int(p.view(np.uint32))
  sign, e, m = bits >> 31, (bits >> 23) & 255, bits & 0x7FFFFF
  if e:
    m |= 0x800000
  k = 150 - max(e, 1)          # p == m / 2**k
  q = 0
  if k < 32:                   # otherwise p * 100 < 2**31 / 2**32: rounds to 0
    num = m * 100
    q, r = num >> k, num & ((1 << k) - 1)
    half = 1 << (k - 1) if k > 0 else 0
    if k > 0 and (r > half or (r == half and q & 1)):
      q += 1
  return ('-' if sign else '') + '%d.%d%d' % (q // 100, q // 10 % 10, q % 10)


def box_corners(cx, cy, w, h):
  """int() of bbox_transform([cx, cy, w, h]) in float32, or None when a corner is non-finite or
  at least 2**31 in magnitude (the record is skipped)."""
  cx, cy, w, h = (np.float32(v) for v in (cx, cy, w, h))
  with np.errstate(all='ignore'):
    hw, hh = w / np.float32(2), h / np.float32(2)
    corners = [cx - hw, cy - hh, cx + hw, cy + hh]
  if not all(math.isfinite(v) and abs(float(v)) < 2.0 ** 31 for v in corners):
    return None
  return [int(v) for v in corners]


def record_mask(shape, det, names, thresh, font_scale):
  """The bool mask [h, w] one record draws on an h x w canvas, or None when it draws nothing."""
  if not np.float32(det['prob']) > np.float32(thresh):
    return None
  cls = int(det['cls'])
  if not 0 <= cls < len(names):
    return None
  c = box_corners(det['cx'], det['cy'], det['w'], det['h'])
  if c is None:
    return None
  mask = np.zeros(shape, bool)
  rectangle_mask(mask, c[0], c[1], c[2], c[3])
  label = prob_label(det['prob'])
  if label is not None:
    put_text_mask(mask, names[cls] + ': (' + label + ')', (c[0], c[3]), font_scale)
  return mask


def masks(shape, dets, count, names, class_bgr, thresh, font_scale):
  """[(mask, (b, g, r))] of one canvas's records, in drawing order."""
  if count < 0:
    return []
  out = []
  for d in dets[:count]:
    m = record_mask(shape, d, names, thresh, font_scale)
    if m is not None:
      out.append((m, tuple(int(v) for v in class_bgr[int(d['cls'])])))
  return out


def draw_bgr(canvas, dets, count, names, class_bgr, thresh, font_scale):
  """sqdet_draw_dets on a uint8 BGR canvas [h, w, 3], in place (a numpy view of a crop works)."""
  for m, bgr in masks(canvas.shape[:2], dets, count, names, class_bgr, thresh, font_scale):
    canvas[m] = bgr
  return canvas


def yuv_of_bgr(b, g, r):
  """(Y, U, V) of cv2.cvtColor(solid 2x2 BGR patch, COLOR_BGR2YUV_I420): OpenCV's BT.601
  limited-range coefficients with 20 fraction bits.  Works on ints or int arrays."""
  b, g, r = (np.asarray(v, np.int64) for v in (b, g, r))
  half = 1 << 19
  y = (269484 * r + 528482 * g + 102760 * b + (16 << 20) + half) >> 20
  u = (-155188 * r - 305135 * g + 460324 * b + (128 << 20) + half) >> 20
  v = (460324 * r - 385875 * g - 74448 * b + (128 << 20) + half) >> 20
  return y, u, v


def draw_yuv420(luma, chroma_u, chroma_v, crop, dets, count, names, class_bgr, thresh, font_scale):
  """sqdet_draw_dets on a 4:2:0 frame, in place: luma [H, W], chroma_u / chroma_v [H/2, W/2]
  (views of NV12's interleaved plane work), canvas = the crop (x, y, w, h) of the frame."""
  x, y, w, h = crop
  H, W = luma.shape
  for m, (b, g, r) in masks((h, w), dets, count, names, class_bgr, thresh, font_scale):
    Y, U, V = (int(v) for v in yuv_of_bgr(b, g, r))
    full = np.zeros((H, W), bool)
    full[y:y + h, x:x + w] = m
    luma[full] = Y
    block = full.reshape(H // 2, 2, W // 2, 2).any(axis=(1, 3))
    chroma_u[block] = U
    chroma_v[block] = V
