"""oracle.jpeg_decode is bitwise cv2.imdecode(buf, cv2.IMREAD_COLOR) over the decoder's corpus:
sizes from 1x1 to 1080p, qualities 1-100, every supported sampling, restart intervals, optimized
Huffman tables, separate luma and chroma qualities, grayscale and all eight EXIF orientations."""
import cv2
import numpy as np
import pytest

from oracle import jpeg_decode as D

import jpeg_corpus as J


@pytest.fixture(scope='module')
def corpus():
  return J.corpus(seed=1)


def test_corpus_is_cv2(corpus):
  for name, f in corpus:
    want = J.imdecode(f)
    got = D.decode(f)
    assert got.shape == want.shape and np.array_equal(got, want), name


@pytest.mark.parametrize('o', range(1, 9))
def test_orientation_index_maps(o):
  rng = np.random.default_rng(o)
  img = J.content('noise', 13, 21, 3, rng)
  f = J.encode(img, cv2.IMWRITE_JPEG_QUALITY, 100, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x111111)
  plain = J.imdecode(f)
  for le in (False, True):
    g = D.with_orientation(f, o, le)
    assert np.array_equal(J.imdecode(g), D.orient(plain, o))
    assert np.array_equal(D.decode(g), D.orient(plain, o))
  if o == 6:
    assert np.array_equal(D.orient(plain, 6), cv2.rotate(plain, cv2.ROTATE_90_CLOCKWISE))


@pytest.mark.parametrize('samp', J.SAMPLINGS)
@pytest.mark.parametrize('w', [1, 2, 3, 4, 5, 6, 9, 16, 17])
def test_narrow_upsampling(samp, w):
  # fancy h2v1 / h2v2 upsampling only runs on chroma wider than 2 samples; h1v2 always
  rng = np.random.default_rng(w)
  for h in (1, 2, 3, 7, 18):
    f = J.encode(J.content('noise', h, w, 3, rng), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)
    assert np.array_equal(D.decode(f), J.imdecode(f)), (h, w)


def test_refusals():
  rng = np.random.default_rng(2)
  img = J.content('smooth', 20, 24, 3, rng)
  prog = J.encode(img, cv2.IMWRITE_JPEG_PROGRESSIVE, 1)
  with pytest.raises(D.Unsupported) as e:
    D.parse(prog)
  assert e.value.reason == D.PROGRESSIVE
  with pytest.raises(D.Unsupported) as e:
    D.parse(prog[:100])
  assert e.value.reason in (D.MALFORMED, D.PROGRESSIVE)


def test_handmade_files_are_cv2():
  # SOF1 and 16-bit tables, scaled until dequantized coefficients overflow 16 bits, where cv2's
  # SIMD islow wraps and saturates; and colour-space markers libjpeg reads as YCbCr
  for name, f in J.handmade():
    assert np.array_equal(D.decode(f), J.imdecode(f)), name


def test_rgb_coded_and_bad_tables_refused():
  rng = np.random.default_rng(4)
  f = J.encode(J.content('smooth', 40, 56, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90)
  for g in (J.component_ids(f, (82, 71, 66), jfif=False), J.component_ids(f, (1, 2, 3), jfif=False, adobe=0)):
    with pytest.raises(D.Unsupported) as e:
      D.parse(g)
    assert e.value.reason == D.COLOR_TRANSFORM
    assert not np.array_equal(J.imdecode(g), J.imdecode(f))     # cv2 decodes them as RGB
  for kind in ('over', 'dc16'):
    g = J.bad_huffman(f, kind)
    assert J.imdecode(g) is None
    with pytest.raises(D.Unsupported) as e:
      D.parse(g)
    assert e.value.reason == D.MALFORMED
