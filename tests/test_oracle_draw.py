"""Pins oracle.draw, the restatement sqdet_draw_dets follows, bitwise against the installed cv2:
putText glyph by glyph, draw_box on random records (every clip side and corner, canvases down to
1x1, crop views, overlapping records), the '%.2f' label digits and the YUV colour of every BGR
colour."""
import numpy as np
import pytest

from oracle import draw

cv2 = pytest.importorskip('cv2')
from squeezedet_b200.utils.viz import draw_box  # noqa: E402

FONT = cv2.FONT_HERSHEY_SIMPLEX
NAMES = ('car', 'pedestrian', 'cyclist')
BGR = np.array([(255, 191, 0), (255, 0, 191), (0, 191, 255)], np.uint8)
PRINTABLE = ''.join(chr(c) for c in range(32, 127))


def records(rng, n, h, w, spread=1.5):
  d = np.zeros(n, draw_dets_dtype())
  d['cls'] = rng.integers(0, 3, n)
  d['prob'] = rng.uniform(0, 1, n).astype(np.float32)
  d['cx'] = rng.uniform(-spread * 0.25 * w, spread * w, n)
  d['cy'] = rng.uniform(-spread * 0.25 * h, spread * h, n)
  d['w'] = rng.uniform(0, 0.8 * w + 4, n)
  d['h'] = rng.uniform(0, 0.8 * h + 4, n)
  return d


def draw_dets_dtype():
  from squeezedet_b200 import _lib
  return _lib.DET_DTYPE


def cv2_draw(canvas, dets, count, thresh=0.4):
  """demo.draw_detections' selection + viz.draw_box, on the records as records_to_lists gives them."""
  keep = [r for r in dets[:max(count, 0)] if np.float32(r['prob']) > thresh]
  boxes = [np.array([r['cx'], r['cy'], r['w'], r['h']], np.float32) for r in keep]
  labels = [NAMES[int(r['cls'])] + ': (%.2f)' % np.float32(r['prob']) for r in keep]
  cdict = {n: tuple(int(v) for v in c) for n, c in zip(NAMES, BGR)}
  return draw_box(canvas, boxes, labels, cdict=cdict)


@pytest.mark.parametrize('scale', [0.3, 0.5, 1.0])
def test_every_glyph_bitwise_puttext(scale):
  for ch in PRINTABLE:
    for org in [(3, 20), (4, 25), (-2, 9), (7, 2)]:
      want = np.zeros((36, 30), np.uint8)
      cv2.putText(want, ch, org, FONT, scale, 255, 1)
      got = np.zeros((36, 30), bool)
      draw.put_text_mask(got, ch, org, scale)
      assert np.array_equal(got, want > 0), (ch, org, scale)


@pytest.mark.parametrize('scale', [0.3, 0.5, 1.0])
def test_random_labels_bitwise_puttext(scale):
  rng = np.random.default_rng(int(scale * 10))
  for _ in range(400):
    h, w = (int(v) for v in rng.integers(1, 60, 2))
    text = ''.join(rng.choice(list(PRINTABLE), int(rng.integers(1, 16))))
    org = (int(rng.integers(-int(80 * scale) - 20, w + 10)), int(rng.integers(-10, h + int(40 * scale))))
    want = np.zeros((h, w), np.uint8)
    cv2.putText(want, text, org, FONT, scale, 255, 1)
    got = np.zeros((h, w), bool)
    draw.put_text_mask(got, text, org, scale)
    assert np.array_equal(got, want > 0), (text, org, scale, h, w)


def test_line_bitwise_cv2_line():
  rng = np.random.default_rng(3)
  for _ in range(3000):
    h, w = (int(v) for v in rng.integers(1, 40, 2))
    r = int(rng.choice([5, 60, 1000, 10 ** 6]))
    p = [int(v) for v in rng.integers(-r, r + 40, 4)]
    want = np.zeros((h, w), np.uint8)
    cv2.line(want, tuple(p[:2]), tuple(p[2:]), 255, 1, cv2.LINE_8)
    got = np.zeros((h, w), bool)
    for x, y in draw.line_pixels(w, h, *p):
      got[y, x] = True
    assert np.array_equal(got, want > 0), (p, h, w)


@pytest.mark.parametrize('h,w', [(1, 1), (1, 7), (5, 1), (3, 4), (24, 40), (375, 1242)])
def test_draw_box_bitwise(h, w):
  """Random records over small and KITTI-size canvases: boxes and labels past every side and
  corner, overlaps of different colours."""
  rng = np.random.default_rng(h * 1000 + w)
  for trial in range(40 if h * w < 5000 else 8):
    dets = records(rng, int(rng.integers(1, 12)), h, w)
    base = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    want = cv2_draw(base.copy(), dets, len(dets))
    got = draw.draw_bgr(base.copy(), dets, len(dets), NAMES, BGR, 0.4, 0.3)
    np.testing.assert_array_equal(got, want, err_msg='trial %d' % trial)


def test_crop_view_bitwise():
  """Drawing on a crop is cv2 drawing on the numpy view of it."""
  rng = np.random.default_rng(11)
  for _ in range(30):
    H, W = (int(v) for v in rng.integers(8, 90, 2))
    x, y = (int(v) for v in rng.integers(0, 6, 2))
    w, h = int(rng.integers(1, W - x + 1)), int(rng.integers(1, H - y + 1))
    dets = records(rng, 6, h, w)
    frame = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    want = frame.copy()
    cv2_draw(want[y:y + h, x:x + w], dets, len(dets))
    got = frame.copy()
    draw.draw_bgr(got[y:y + h, x:x + w], dets, len(dets), NAMES, BGR, 0.4, 0.3)
    np.testing.assert_array_equal(got, want)


def test_counts_and_skips():
  rng = np.random.default_rng(5)
  dets = records(rng, 4, 50, 80)
  dets['prob'] = 0.9
  canvas = np.zeros((50, 80, 3), np.uint8)
  assert not draw.draw_bgr(canvas.copy(), dets, -1, NAMES, BGR, 0.4, 0.3).any()
  assert not draw.draw_bgr(canvas.copy(), dets, 0, NAMES, BGR, 0.4, 0.3).any()
  bad = dets.copy()
  bad['cls'] = [-1, 3, 0, 0]
  bad['cx'][2] = np.nan
  bad['w'][3] = np.inf
  assert not draw.draw_bgr(canvas.copy(), bad, 4, NAMES, BGR, 0.4, 0.3).any()
  big = dets[:1].copy()
  big['cx'] = 3e9                   # a corner at or past 2^31: skipped
  assert not draw.draw_bgr(canvas.copy(), big, 1, NAMES, BGR, 0.4, 0.3).any()
  odd = dets[:1].copy()
  odd['prob'] = 1.5                 # kept, rectangle only
  want = canvas.copy()
  c = draw.box_corners(odd['cx'][0], odd['cy'][0], odd['w'][0], odd['h'][0])
  cv2.rectangle(want, (c[0], c[1]), (c[2], c[3]), tuple(int(v) for v in BGR[odd['cls'][0]]), 1)
  np.testing.assert_array_equal(draw.draw_bgr(canvas.copy(), odd, 1, NAMES, BGR, 0.4, 0.3), want)


def test_prob_label_is_python_format():
  """'%.2f' of every float32 on a dense grid of [0, 1], every k/8 tie, and both neighbours of
  every rounding boundary (2j + 1) / 200."""
  grid = np.linspace(0, 1, 200001, dtype=np.float32)
  bounds = np.array([(2 * j + 1) / 200 for j in range(100)], np.float32)
  near = np.concatenate([bounds, np.nextafter(bounds, np.float32(0)), np.nextafter(bounds, np.float32(1))])
  ties = np.array([k / 8 for k in range(9)], np.float32)
  tiny = np.array([0, 1e-45, 1e-38, 1e-10, 0.004999, 0.005, 0.995, 1.0], np.float32)
  for p in np.concatenate([grid, near, ties, tiny]):
    assert draw.prob_label(p) == '%.2f' % p, p
  assert draw.prob_label(np.float32(0.125)) == '0.12'
  assert draw.prob_label(np.float32(-0.0)) == '-0.00' == '%.2f' % np.float32(-0.0)
  assert draw.prob_label(np.float32(1.0000001)) is None
  assert draw.prob_label(np.float32(np.nan)) is None


def test_yuv_of_every_bgr_colour():
  """cv2.cvtColor(COLOR_BGR2YUV_I420) of all 256^3 colours as 2x2 patches, 65536 at a time."""
  c = np.arange(65536)
  for r in range(256):
    bgr = np.stack([c & 255, c >> 8, np.full_like(c, r)], axis=-1).astype(np.uint8)
    im = np.ascontiguousarray(np.repeat(np.repeat(bgr[None], 2, 0), 2, 1))
    out = cv2.cvtColor(im, cv2.COLOR_BGR2YUV_I420)
    y, u, v = draw.yuv_of_bgr(bgr[:, 0], bgr[:, 1], bgr[:, 2])
    np.testing.assert_array_equal(out[0, 0::2], y)
    np.testing.assert_array_equal(out[0, 1::2], y)
    np.testing.assert_array_equal(out[2, :65536], u)
    np.testing.assert_array_equal(out[2, 65536:], v)


def test_yuv420_rule():
  """Luma takes Y on the BGR mask; a chroma sample takes (U, V) when its 2x2 block (frame
  coordinates, odd crop origins included) holds a mask pixel."""
  rng = np.random.default_rng(8)
  H, W = 40, 60
  for x, y in [(0, 0), (1, 1), (3, 2), (5, 7)]:
    w, h = W - x - 1, H - y - 2
    dets = records(rng, 5, h, w)
    dets['prob'] = 0.9
    luma = rng.integers(0, 256, (H, W), dtype=np.uint8)
    uv = rng.integers(0, 256, (H // 2, W), dtype=np.uint8)
    got_y, got_uv = luma.copy(), uv.copy()
    draw.draw_yuv420(got_y, got_uv[:, 0::2], got_uv[:, 1::2], (x, y, w, h), dets, 5, NAMES, BGR,
                     0.4, 0.3)
    want_y, want_uv = luma.copy(), uv.copy()
    for m, (b, g, r) in draw.masks((h, w), dets, 5, NAMES, BGR, 0.4, 0.3):
      Y, U, V = (int(v) for v in draw.yuv_of_bgr(b, g, r))
      for cy, cx in np.argwhere(m):
        want_y[y + cy, x + cx] = Y
        want_uv[(y + cy) // 2, 2 * ((x + cx) // 2)] = U
        want_uv[(y + cy) // 2, 2 * ((x + cx) // 2) + 1] = V
    np.testing.assert_array_equal(got_y, want_y)
    np.testing.assert_array_equal(got_uv, want_uv)
