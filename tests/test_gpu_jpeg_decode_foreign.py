"""decode_jpeg_device on files other encoders write and on camera-size files: every frame is
bitwise cv2.imdecode's, in mixed batches, through the synchronisation paths of the parallel
Huffman decode, with EXIF orientation read as cv2 reads it; a corrupt camera file fails alone."""
import numpy as np
import pytest
import torch

from oracle import jpeg_decode as D
from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import decode_jpeg_device

import jpeg_corpus as J

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def foreign():
  return [(n, f) for n, f, _ in J.foreign()] + [(n, f) for n, f, _ in J.exif_variants()]


@pytest.fixture(scope='module')
def camera():
  """[(name, file, cv2's frame)]."""
  return [(n, f, J.imdecode(f)) for n, f in J.camera()]


@pytest.fixture
def sub_bits():
  """Sets the subsequence size of the parallel Huffman decode for one test."""
  lib = _lib.load()
  yield lambda bits: _lib.check(lib.sqdet_jpeg_decode_set_subsequence_bits(bits))
  _lib.check(lib.sqdet_jpeg_decode_set_subsequence_bits(0))


def check_batch(named, wants=None):
  files = [f for _, f in named]
  frames, status = decode_jpeg_device(files, DEV)
  st = status.cpu().numpy()
  for k, ((name, f), fr, s) in enumerate(zip(named, frames, st)):
    want = J.imdecode(f) if wants is None else wants[k]
    assert s == 0, '%s: status %d' % (name, s)
    got = fr.cpu().numpy()
    assert got.shape == want.shape, name
    assert np.array_equal(got, want), '%s: %d pixels differ' % (name, int((got != want).any(2).sum()))


def batches(items, sizes=(1, 7, 32, 19, 3)):
  i, k = 0, 0
  while i < len(items):
    n = sizes[k % len(sizes)]
    yield items[i:i + n]
    i += n
    k += 1


@pytest.mark.parametrize('bits', [0, 32, 64])
def test_foreign_and_exif_mixed_batches(foreign, sub_bits, bits):
  sub_bits(bits)
  order = np.random.default_rng(bits).permutation(len(foreign))
  for b in batches([foreign[i] for i in order]):
    check_batch(b)


def test_camera_files_alone_then_together(camera):
  for name, f, want in camera:
    check_batch([(name, f)], [want])
  check_batch([(n, f) for n, f, _ in camera], [w for _, _, w in camera])


def test_noise_file_among_127_foreign(foreign, camera):
  name, f, want = camera[2]
  small = foreign[:127]
  named = small[:60] + [(name, f)] + small[60:]
  check_batch(named, [J.imdecode(g) for _, g in small[:60]] + [want] + [J.imdecode(g) for _, g in small[60:]])


def test_small_subsequences_on_a_camera_file(camera, sub_bits):
  # 32-bit subsequences: the 2 MB file has about half a million of them, so sync_chain_kernel walks
  # thousands of tiles
  sub_bits(32)
  name, f, want = camera[0]
  check_batch([(name, f)], [want])


def test_refused_files_raise():
  for name, f, reason, _ in J.refused():
    with pytest.raises(ValueError, match=D.REASONS[reason]):
      decode_jpeg_device([J.encode(J.content('flat', 8, 8, 3, np.random.default_rng(0))), f], DEV)


def test_corrupt_camera_file_fails_alone(camera):
  (na, a, wa), (nb, b, wb), (nn, noise, wn), (n1, one, w1), (n2, two, w2) = camera
  bad_b = bytearray(b)                       # all-ones bits inside a restart interval past the middle
  k = bytes(bad_b).index(b'\xff\xd7', D.parse(b).scan + len(b) // 2) + 200
  bad_b[k:k + 40] = b'\xff\x00' * 20
  scan = D.parse(noise).scan
  bad_noise = noise[:scan + (len(noise) - scan) // 2]
  for files, wants, bad in (([a, bytes(bad_b), noise, one], [wa, None, wn, w1], 1),
                            ([a, b, bad_noise, two], [wa, wb, None, w2], 2)):
    frames, status = decode_jpeg_device(files, DEV)
    st = status.cpu().tolist()
    assert st[bad] < 0, st
    for i, (fr, w) in enumerate(zip(frames, wants)):
      if i != bad:
        assert st[i] == 0, st
        assert np.array_equal(fr.cpu().numpy(), w), i
