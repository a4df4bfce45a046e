"""oracle.jpeg_decode_progressive is cv2.imdecode bitwise on progressive files: cv2's over the
corpus kinds, sizes, samplings, qualities, restart intervals, grayscale and EXIF orientations,
oracle.jpeg_progressive's, and foreign scan scripts (tests/progressive_writer.py).  Complete
scripts decode to the baseline source's pixels; refused scripts are pinned to what cv2 does."""
import cv2
import numpy as np
import pytest

from oracle import jpeg_decode as D
from oracle import jpeg_decode_progressive as P
from oracle import jpeg_progressive

import jpeg_corpus as J
import progressive_writer as W
from progressive_inputs import correction_frame, CORRECTION_QUALITY

PROG = cv2.IMWRITE_JPEG_PROGRESSIVE


def same(f):
  want = J.imdecode(f)
  got = P.decode(f)
  assert want is not None and np.array_equal(got, want)


@pytest.mark.parametrize('samp', J.SAMPLINGS)
def test_cv2_files(samp):
  rng = np.random.default_rng(samp & 0xFFFF)
  for zi, (h, w) in enumerate(J.SIZES[::2]):
    q = (1, 25, 75, 95, 100)[zi % 5]
    rst = (0, 1, 3, 7)[zi % 4]
    same(J.encode(J.content(J.KINDS[zi % len(J.KINDS)], h, w, 3, rng), PROG, 1,
                  cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp,
                  cv2.IMWRITE_JPEG_RST_INTERVAL, rst))


def test_gray_and_orientation():
  rng = np.random.default_rng(1)
  for q, rst in ((10, 0), (90, 2)):
    same(J.encode(J.content('noise', 33, 47, 1, rng)[..., 0], PROG, 1, cv2.IMWRITE_JPEG_QUALITY, q,
                  cv2.IMWRITE_JPEG_RST_INTERVAL, rst))
  base = J.encode(J.content('smooth', 21, 34, 3, rng), PROG, 1)
  for o in range(1, 9):
    same(D.with_orientation(base, o, o % 2 == 1))


def test_oracle_encoder_files():
  rng = np.random.default_rng(2)
  same(jpeg_progressive.encode(J.content('noise', 29, 45, 3, rng), 90, sampling='422', restart_interval=3))
  img, _ = correction_frame()
  same(jpeg_progressive.encode(img[:64, :64], CORRECTION_QUALITY, sampling='444'))


@pytest.fixture(scope='module')
def sources():
  rng = np.random.default_rng(3)
  return [J.encode(J.content('smooth', 37, 58, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90,
                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp) for samp in (0x221111, 0x111111, 0x411111)]


@pytest.mark.parametrize('name', sorted(W.COMPLETE))
def test_complete_scripts(sources, name):
  for f in sources:
    g = W.write(f, W.COMPLETE[name])
    assert np.array_equal(J.imdecode(g), J.imdecode(f))          # the writer's self-check
    same(g)


def test_restarts_tables_and_dqt(sources):
  for f in sources:
    for g in (W.write(f, W.SPECTRAL, restarts={1: 2, 3: 0, 4: 5}),
              W.write(f, W.DC_SUBSETS, dqt_after=1), W.write(f, W.DEEP, restarts={0: 1, 20: 3})):
      assert np.array_equal(J.imdecode(g), J.imdecode(f))
      same(g)
  rng = np.random.default_rng(4)
  gray = J.encode(J.content('noise', 37, 58, 1, rng)[..., 0])
  g = W.write(gray, W.GRAY_DEEP, restarts={0: 3, 4: 1, 8: 0})
  assert np.array_equal(J.imdecode(g), J.imdecode(gray))
  same(g)


def test_incomplete_unsmoothed(sources):
  for f in sources:
    for script in W.UNSMOOTHED.values():
      same(W.write(f, script))


def reason(g):
  with pytest.raises(P.Unsupported) as e:
    P.parse(g)
  return e.value.reason


def test_refused_scripts(sources):
  f = sources[0]
  for script in W.BAD.values():
    g = W.write(f, script)
    assert reason(g) == P.BAD_PROGRESSION and J.imdecode(g) is None
  for script in W.BOGUS.values():
    g = W.write(f, script)
    assert reason(g) == P.BOGUS_PROGRESSION and J.imdecode(g) is not None
  differs = 0
  for script in W.SMOOTHED.values():
    g = W.write(f, script)
    assert reason(g) == P.SMOOTHED and J.imdecode(g) is not None
    differs += unsmoothed_differs(g)
  assert differs >= 1


def unsmoothed_differs(g):
  """Whether cv2's (smoothed) pixels differ from the plain decode of the same coefficients."""
  smoothed = P.smoothed
  try:
    P.smoothed = lambda *a: False
    plain = P.decode(g)
  finally:
    P.smoothed = smoothed
  return not np.array_equal(plain, J.imdecode(g))


def scans(g):
  return sum(1 for i in range(len(g) - 1) if g[i:i + 2] == b'\xff\xda')


def test_scan_cap(sources):
  dc = [((0, 1, 2), 0, 0, 0, 13)] + [((0, 1, 2), 0, 0, a + 1, a) for a in range(12, -1, -1)]
  many = W.write(sources[0], dc + [((c,), k, k, 0, 0) for c in (0, 1, 2) for k in range(1, 64)])
  assert scans(many) == 203
  same(many)
  over = W.write(sources[0], dc + [((c,), k, k, 0, 1) for c in (0, 1, 2) for k in range(1, 64)] +
                 [((c,), k, k, 1, 0) for c in (0, 1, 2) for k in range(1, 22)])
  assert scans(over) > P.MAX_SCANS
  assert reason(over) == P.TOO_MANY_SCANS and J.imdecode(over) is not None
