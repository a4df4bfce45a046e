"""oracle.jpeg_progressive is cv2.imencode('.jpg', ...) with IMWRITE_JPEG_PROGRESSIVE byte for byte:
every sampling at every MCU-edge remainder, qualities, restart intervals and luma/chroma quality,
and its EOBRUN flushes reach every cause.  cv2.imdecode of each file equals that of the baseline
file of the same settings."""
import cv2
import numpy as np
import pytest

from jpeg_corpus import KINDS, content
from oracle import jpeg_params, jpeg_progressive
from progressive_inputs import CORRECTION_QUALITY, cap_frame, correction_frame, requantized

SAMPLINGS = tuple(jpeg_params.SAMPLING_FACTORS)
# rotated through the edge sizes, so that each sampling meets each of them at several remainders
ROTATION = [dict(), dict(restart_interval=1), dict(quality=50, restart_interval=3),
            dict(quality=100, restart_interval=7), dict(quality=1, restart_interval=65535),
            dict(luma_quality=90, chroma_quality=40), dict(luma_quality=60, chroma_quality=60)]


def cv2_encode(img, progressive=True, **kw):
  params = jpeg_params.cv2_params(**kw) + ([cv2.IMWRITE_JPEG_PROGRESSIVE, 1] if progressive else [])
  ok, buf = cv2.imencode('.jpg', img, params)
  assert ok
  return buf.tobytes()


def decoded(f):
  return cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)


def check(img, causes=None, **kw):
  f = jpeg_progressive.encode(img, causes=causes, **kw)
  assert f == cv2_encode(img, **kw), (img.shape, kw)
  assert np.array_equal(decoded(f), decoded(cv2_encode(img, progressive=False, **kw)))
  return f


def edge_sizes(sampling):
  """(h, w) with every height remainder modulo the MCU height and every width remainder modulo its
  width, plus 1 x 1 and 61 x 97."""
  hs, vs = jpeg_params.SAMPLING_FACTORS[sampling]
  mw, mh = 8 * hs, 8 * vs
  n = max(mw, mh)
  return [(mh + 1 + i % mh, mw + 1 + i % mw) for i in range(n)] + [(1, 1), (61, 97)]


@pytest.mark.parametrize('sampling', SAMPLINGS)
def test_edges(sampling):
  rng = np.random.default_rng(1)
  for i, (h, w) in enumerate(edge_sizes(sampling)):
    check(content(KINDS[i % len(KINDS)], h, w, 3, rng), **ROTATION[i % len(ROTATION)], sampling=sampling)


@pytest.mark.parametrize('sampling', SAMPLINGS)
def test_qualities_and_intervals(sampling):
  rng = np.random.default_rng(2)
  for q in (1, 50, 95, 100):
    for r in (0, 1, 3, 7, 65535):
      check(content(('noise', 'smooth', 'check')[r % 3], 37, 53, 3, rng), quality=q, restart_interval=r,
            sampling=sampling)


@pytest.mark.parametrize('sampling', SAMPLINGS)
def test_luma_chroma_quality(sampling):
  rng = np.random.default_rng(3)
  img = content('noise', 29, 45, 3, rng)
  for lq, cq in ((75, 75), (95, 95), (90, 40), (40, 90), (1, 100), (100, 1), (75, None), (None, 30)):
    f = check(img, sampling=sampling, luma_quality=lq, chroma_quality=cq, quality=60)
    if lq is not None and cq is not None and cq != lq:      # 4:4:4, whatever the sampling
      assert f == jpeg_progressive.encode(img, sampling='444', luma_quality=lq, chroma_quality=cq)


def test_optimize_has_no_effect():
  img = content('noise', 40, 56, 3, np.random.default_rng(4))
  for r in (0, 2):
    assert cv2_encode(img, optimize=True, restart_interval=r) == cv2_encode(img, restart_interval=r)
    assert jpeg_progressive.encode(img, optimize=True, restart_interval=r) == \
        jpeg_progressive.encode(img, restart_interval=r)


def test_scan_script():
  """SOF2, ten SOS with cv2's (Ss, Se, Ah, Al), DHTs before every scan but the DC refinement (two
  before the first), one DRI before the first SOS."""
  f = check(content('noise', 33, 47, 3, np.random.default_rng(5)), restart_interval=2)
  i, scans, dhts, dri = 2, [], [0], []
  while f[i + 1] != 0xD9:
    marker, n = f[i + 1], int.from_bytes(f[i + 2:i + 4], 'big')
    if marker == 0xC2:
      assert f[i + 9] == 3
    if marker == 0xC4:
      dhts[-1] += 1
    if marker == 0xDD:
      dri.append(len(scans))
    if marker == 0xDA:
      k = f[i + 4]
      scans.append((tuple(f[i + 5:i + 5 + 2 * k:2]),) + tuple(f[i + 5 + 2 * k:i + 7 + 2 * k]) +
                   (f[i + 7 + 2 * k] >> 4, f[i + 7 + 2 * k] & 15))
      dhts.append(0)
      i += 2 + n
      while not (f[i] == 0xFF and f[i + 1] not in (0x00,) and not 0xD0 <= f[i + 1] <= 0xD7):
        i += 1
      continue
    i += 2 + n
  assert [(tuple(c + 1 for c in comps), ss, se, ah, al)
          for comps, ss, se, ah, al in jpeg_progressive.SCANS] == scans
  assert dhts[:10] == [2, 1, 1, 1, 1, 1, 0, 1, 1, 1] and dri == [0]


def test_every_flush_cause():
  """The corpus reaches each EOBRUN flush cause: natural content the next symbol, restarts and the
  scan's end; a flat frame of 33 024 luma blocks the 0x7FFF cap; a frame whose luma AC
  coefficients are 0 or at least 4 in magnitude the correction-bit overflow."""
  causes = {}
  rng = np.random.default_rng(6)
  for kind in ('noise', 'smooth', 'grad'):
    check(content(kind, 64, 96, 3, rng), restart_interval=5, causes=causes)
  assert causes['next_symbol'] and causes['restart'] and causes['end_of_scan']
  cap = {}
  check(cap_frame(), causes=cap)
  assert cap['cap'] == 4                              # scans 2, 5, 6 and 10 of the luma blocks
  img, z = correction_frame()
  assert np.array_equal(requantized(img), z) and (np.abs(z[:, 1:13]) >= 4).mean() > 0.9
  corr = {}
  check(img, quality=CORRECTION_QUALITY, sampling='444', causes=corr)
  assert corr['correction_bits'] > 0
  natural = {}
  for kind in ('noise', 'smooth'):
    for q in (50, 95, 100):
      check(content(kind, 96, 128, 3, rng), quality=q, causes=natural)
  assert natural['correction_bits'] == 0 and natural['cap'] == 0


def test_refusals():
  img = np.zeros((8, 8, 3), np.uint8)
  for kw in (dict(quality=0), dict(quality=101), dict(luma_quality=0), dict(chroma_quality=101),
             dict(sampling='421'), dict(restart_interval=-1), dict(restart_interval=65536)):
    with pytest.raises(ValueError):
      jpeg_progressive.encode(img, **kw)
