"""oracle.jpeg_params is cv2.imencode('.jpg', ...) byte for byte with cv2's other JPEG parameters:
every sampling at every MCU-edge remainder, qualities, separate luma and chroma quality, optimized
tables and restart intervals, over the content kinds of jpeg_corpus."""
import cv2
import numpy as np
import pytest

from jpeg_corpus import KINDS, content
from oracle import jpeg, jpeg_params

SAMPLINGS = tuple(jpeg_params.SAMPLING_FACTORS)
# rotated through the edge sizes, so that each sampling meets each of them at several remainders
ROTATION = [dict(), dict(optimize=True), dict(restart_interval=1), dict(restart_interval=2, optimize=True),
            dict(luma_quality=90, chroma_quality=40), dict(quality=50, restart_interval=3),
            dict(quality=100, optimize=True, restart_interval=7)]


def cv2_encode(img, **kw):
  ok, buf = cv2.imencode('.jpg', img, jpeg_params.cv2_params(**kw))
  assert ok
  return buf.tobytes()


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
    img = content(KINDS[i % len(KINDS)], h, w, 3, rng)
    kw = dict(ROTATION[i % len(ROTATION)], sampling=sampling)
    assert jpeg_params.encode(img, **kw) == cv2_encode(img, **kw), (h, w, kw)


@pytest.mark.parametrize('sampling', SAMPLINGS)
@pytest.mark.parametrize('optimize', [False, True])
def test_qualities(sampling, optimize):
  rng = np.random.default_rng(2)
  for q in (1, 50, 75, 95, 100):
    for kind in ('noise', 'smooth', 'check'):
      img = content(kind, 37, 53, 3, rng)
      kw = dict(quality=q, sampling=sampling, optimize=optimize)
      assert jpeg_params.encode(img, **kw) == cv2_encode(img, **kw), (q, kind)


@pytest.mark.parametrize('sampling', SAMPLINGS)
def test_luma_chroma_quality(sampling):
  rng = np.random.default_rng(3)
  img = content('noise', 29, 45, 3, rng)
  for lq, cq in ((75, 75), (95, 95), (90, 40), (40, 90), (1, 100), (100, 1), (75, None), (None, 30)):
    kw = dict(sampling=sampling, luma_quality=lq, chroma_quality=cq, quality=60)
    f = jpeg_params.encode(img, **kw)
    assert f == cv2_encode(img, **kw), (lq, cq)
    if lq is None:                                    # chroma quality alone is ignored
      assert f == jpeg_params.encode(img, 60, sampling=sampling)
    elif cq is None or cq == lq:                      # the same as quality = luma quality
      assert f == jpeg_params.encode(img, lq, sampling=sampling)
    else:                                             # 4:4:4, whatever the sampling
      assert f == jpeg_params.encode(img, sampling='444', luma_quality=lq, chroma_quality=cq)
      assert jpeg_params.resolve(60, sampling, lq, cq)[2] == (1, 1)


@pytest.mark.parametrize('sampling', SAMPLINGS)
@pytest.mark.parametrize('optimize', [False, True])
def test_restart_intervals(sampling, optimize):
  rng = np.random.default_rng(4)
  for h, w in ((61, 97), (9, 17), (1, 1)):
    img = content('noise', h, w, 3, rng)
    for r in (0, 1, 2, 3, 7, 1000, 65535):
      kw = dict(sampling=sampling, optimize=optimize, restart_interval=r)
      f = jpeg_params.encode(img, **kw)
      assert f == cv2_encode(img, **kw), (h, w, r)
      assert (b'\xff\xdd' in f[:f.index(b'\xff\xda')]) == (r > 0)


@pytest.mark.parametrize('sampling', SAMPLINGS)
@pytest.mark.parametrize('kind', KINDS)
def test_optimize_contents(sampling, kind):
  rng = np.random.default_rng(5)
  for h, w, q in ((1, 1, 95), (23, 41, 100), (64, 64, 30)):
    img = content(kind, h, w, 3, rng)
    kw = dict(quality=q, sampling=sampling, optimize=True)
    f = jpeg_params.encode(img, **kw)
    assert f == cv2_encode(img, **kw), (h, w, q)


def test_optimize_code_lengths_reach_16():
  """Noise at quality 100 gives codes of the longest length, 16 bits, and a flat image one symbol
  per DC table."""
  img = content('noise', 256, 256, 3, np.random.default_rng(6))
  tables = []
  f = jpeg_params.encode(img, 100, sampling='444', optimize=True)
  assert f == cv2_encode(img, quality=100, sampling='444', optimize=True)
  i = 2
  while f[i:i + 2] != b'\xff\xda':
    n = int.from_bytes(f[i + 2:i + 4], 'big')
    if f[i + 1] == 0xC4:
      tables.append(list(f[i + 5:i + 21]))
    i += 2 + n
  assert max(max(l for l in range(16) if t[l]) for t in tables) == 15
  flat = content('flat', 16, 16, 3, None)
  g = jpeg_params.encode(flat, sampling='444', optimize=True)
  assert g == cv2_encode(flat, sampling='444', optimize=True)


def test_defaults_match_the_baseline_oracle():
  img = content('noise', 33, 47, 3, np.random.default_rng(7))
  for q in (1, 75, 95, 100):
    assert jpeg_params.encode(img, q) == jpeg.encode(img, q)


def test_refusals():
  img = np.zeros((8, 8, 3), np.uint8)
  for kw in (dict(quality=0), dict(quality=101), dict(luma_quality=0), dict(chroma_quality=101),
             dict(sampling='421'), dict(restart_interval=-1), dict(restart_interval=65536)):
    with pytest.raises(ValueError):
      jpeg_params.encode(img, **kw)
