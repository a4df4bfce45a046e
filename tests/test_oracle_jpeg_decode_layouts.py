"""oracle.jpeg_decode_layouts is bitwise cv2.imdecode (IMREAD_COLOR and IMREAD_REDUCED_COLOR_2/4/8)
on CMYK, YCCK and RGB-coded files and on samplings cv2's encoder never writes, sequential and
progressive; cv2 returns None for every file it refuses as BAD_SAMPLING or COMPONENTS; and the
other oracles keep refusing these files."""
import cv2
import numpy as np
import pytest

from oracle import jpeg_decode as D
from oracle import jpeg_decode_layouts as L
from oracle import jpeg_decode_progressive as P

import jpeg_layouts as JL

FLAGS = {1: cv2.IMREAD_COLOR, 2: cv2.IMREAD_REDUCED_COLOR_2, 4: cv2.IMREAD_REDUCED_COLOR_4,
         8: cv2.IMREAD_REDUCED_COLOR_8}
CORPUS = JL.corpus()


def imdecode(f, s):
  return cv2.imdecode(np.frombuffer(f, np.uint8), FLAGS[s])


def check(f, s, name):
  want = imdecode(f, s)
  assert want is not None, name
  got = L.decode(f, s, progressive=True)
  assert got.shape == want.shape and np.array_equal(got, want), (name, s)


@pytest.mark.parametrize('s', (1, 2, 4, 8))
@pytest.mark.parametrize('name', [n for n, _ in CORPUS])
def test_corpus(name, s):
  check(dict(CORPUS)[name], s, name)


@pytest.mark.parametrize('s', (1, 2, 4, 8))
@pytest.mark.parametrize('sampling', ([(4, 2), (1, 1), (1, 1)], [(2, 1), (1, 4), (1, 2), (1, 1)]))
def test_every_side_remainder(sampling, s):
  markers = [JL.JFIF] if len(sampling) == 3 else []
  for name, f in JL.remainders(sampling, markers, seed=len(sampling)):
    check(f, s, name)


@pytest.mark.parametrize('o', range(1, 9))
def test_orientations(o):
  for f in (JL.make(21, 34, [(2, 2), (1, 1), (1, 1), (2, 1)], markers=[JL.adobe(2)], seed=o),
            JL.make(22, 31, [(1, 1), (3, 1), (1, 1)], markers=[JL.adobe(0)], seed=o, script=())):
    for s in (1, 4):
      check(D.with_orientation(f, o, little_endian=o % 2 == 0), s, o)


def test_pillow_cmyk_is_adobe_inverted():
  # Pillow stores CMYK inverted under an Adobe transform 0 and cv2 does not invert it back: ink
  # (0, 0, 0, 40) is stored as (255, 255, 255, 215), and B = K - ((255 - Y) * K >> 8) = 215
  img = np.zeros((16, 16, 4), np.uint8)
  img[..., 3] = 40
  f = JL.pillow(img, 'CMYK', quality=100)
  assert (imdecode(f, 1) == 215).all() and (L.decode(f) == 215).all()


@pytest.mark.parametrize('name', [n for n, _, _ in JL.refused()])
def test_refused_files_cv2_returns_none(name):
  f, reason = {n: (f, r) for n, f, r in JL.refused()}[name]
  with pytest.raises(L.Unsupported) as e:
    L.parse(f, 1, progressive=True)
  assert e.value.reason == reason and str(e.value) == L.REASONS[reason]
  for s in FLAGS:
    assert imdecode(f, s) is None, s


def test_other_oracles_refuse_or_agree():
  # every file here but those YCbCr ones the plain decoder reads is refused by the other oracles
  plain = 0
  for name, f in CORPUS:
    try:
      P.parse(f)
    except D.Unsupported as e:
      assert e.reason in (D.COMPONENTS, D.COLOR_TRANSFORM, D.SAMPLING), name
      continue
    plain += 1
    assert np.array_equal(P.decode(f), L.decode(f, progressive=True)), name
  assert plain == 5


def test_wide_progressive_frame_goes_to_cv2():
  f = JL.wide_progressive()
  with pytest.raises(L.Unsupported) as e:
    L.parse(f, 1, progressive=True)
  assert e.value.reason == D.SAMPLING
  assert imdecode(f, 1) is not None
