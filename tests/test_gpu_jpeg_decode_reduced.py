"""decode_jpeg_device(reduce=s) / sqdet_decode_jpeg_params: frames bitwise
cv2.imdecode(f, IMREAD_REDUCED_COLOR_s) for s in 2, 4, 8, over mixed sequential and progressive
batches of every sampling, size remainder, quality, restart interval and orientation, the handmade
16-bit-table files and other encoders' files; with short subsequences; at camera sizes with EXIF
orientation 6.  A corrupt file fails alone, and reduced frames give the forward's records of
cv2's reduced frames."""
import cv2
import numpy as np
import pytest
import torch

from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import decode_jpeg_device

from oracle.jpeg_decode import with_orientation

import jpeg_corpus as J
import progressive_writer as W
from gpu_util import fetch_results

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
PROG = cv2.IMWRITE_JPEG_PROGRESSIVE
FLAGS = {2: cv2.IMREAD_REDUCED_COLOR_2, 4: cv2.IMREAD_REDUCED_COLOR_4, 8: cv2.IMREAD_REDUCED_COLOR_8}


def imdecode(f, s):
  return cv2.imdecode(np.frombuffer(f, np.uint8), FLAGS[s])


def reduced_corpus(seed=0):
  """[(name, file)]: cv2's sequential corpus, progressive files over samplings, remainders,
  qualities and restart intervals, foreign scan scripts, the handmade files and a third of the
  foreign encoders' files."""
  rng = np.random.default_rng(seed)
  out = list(J.corpus(seed=seed, big=False))
  for si, samp in enumerate(J.SAMPLINGS):
    for k in range(8):
      h, w = 1 + (k * 13 + si * 5) % 67, 1 + (k * 29 + si * 11) % 131
      q = (1, 50, 95, 100)[k % 4]
      out.append(('prog %dx%d s%06x q%d' % (h, w, samp, q),
                  J.encode(J.content(J.KINDS[k % len(J.KINDS)], h, w, 3, rng), PROG, 1,
                           cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp,
                           cv2.IMWRITE_JPEG_RST_INTERVAL, k % 3)))
  base = J.encode(J.content('smooth', 37, 58, 3, rng), PROG, 1, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x211111)
  out += [('prog exif %d' % o, with_orientation(base, o)) for o in range(1, 9)]
  f = J.encode(J.content('smooth', 45, 70, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90)
  out += [(name, W.write(f, script)) for name, script in W.COMPLETE.items()]
  out += J.handmade(seed)
  out += [(name, g) for name, g, _ in J.foreign(seed)[::3]]
  return out


@pytest.fixture(scope='module')
def mixed():
  items = reduced_corpus()
  rng = np.random.default_rng(5)
  return [items[i] for i in rng.permutation(len(items))]


@pytest.fixture
def sub_bits():
  lib = _lib.load()
  yield lambda bits: _lib.check(lib.sqdet_jpeg_decode_set_subsequence_bits(bits))
  _lib.check(lib.sqdet_jpeg_decode_set_subsequence_bits(0))


def check_batch(named, s):
  frames, status = decode_jpeg_device([f for _, f in named], DEV, progressive=True, reduce=s)
  st = status.cpu().numpy()
  for (name, f), fr, code in zip(named, frames, st):
    want = imdecode(f, s)
    assert code == 0, '%s 1/%d: status %d' % (name, s, code)
    got = fr.cpu().numpy()
    assert got.shape == want.shape, (name, s)
    assert np.array_equal(got, want), '%s 1/%d: %d pixels differ' % (name, s, int((got != want).any(2).sum()))


def batches(items, sizes=(1, 7, 32, 19, 3, 64)):
  i, k = 0, 0
  while i < len(items):
    n = sizes[k % len(sizes)]
    yield items[i:i + n]
    i += n
    k += 1


@pytest.mark.parametrize('s', (2, 4, 8))
def test_mixed_batches(mixed, s):
  for b in batches(mixed):
    check_batch(b, s)


@pytest.mark.parametrize('s', (2, 4, 8))
def test_batch_of_128(mixed, s):
  check_batch(mixed[-128:], s)


@pytest.mark.parametrize('s', (2, 8))
def test_small_subsequences(mixed, sub_bits, s):
  sub_bits(32)
  for b in batches(mixed, sizes=(32, 17)):
    check_batch(b, s)


def test_camera_sizes_orientation_6():
  cam = J.camera()
  files = [('4000x3000 s221111 exif 6', cam[0][1]),
           ('4032x3024 noise q100 s111111 exif 6', with_orientation(cam[2][1], 6)),
           ('3000x4000 s211111 rst exif 6', with_orientation(cam[1][1], 6))]
  files.append(('4000x3000 progressive exif 6',
                with_orientation(J.encode(J.imdecode(cam[0][1]), PROG, 1, cv2.IMWRITE_JPEG_QUALITY, 90), 6)))
  for s in (2, 4, 8):
    check_batch(files, s)


def test_corrupt_file_fails_alone():
  rng = np.random.default_rng(13)
  good = [J.encode(J.content('smooth', 64, 96, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90),
          J.encode(J.content('smooth', 64, 96, 3, rng), PROG, 1)]
  junk = bytearray(J.encode(J.content('smooth', 64, 96, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90))
  k = junk.index(b'\xff\xda')
  junk[k + 40:k + 80] = b'\xff\x00' * 20
  for s in (2, 4, 8):
    frames, status = decode_jpeg_device([good[0], bytes(junk), good[1]], DEV, progressive=True, reduce=s)
    st = status.cpu().tolist()
    assert st[1] < 0 and st[0] == st[2] == 0, st
    for i, f in ((0, good[0]), (2, good[1])):
      assert np.array_equal(frames[i].cpu().numpy(), imdecode(f, s))


def test_forward_on_reduced_frames():
  from squeezedet_b200.bench_device_frames import make_model
  rng = np.random.default_rng(17)
  files = [J.encode(J.content('smooth', 1500, 4968, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 95),
           J.encode(J.content('smooth', 1536, 2048, 3, rng), PROG, 1, cv2.IMWRITE_JPEG_QUALITY, 85),
           with_orientation(J.encode(J.content('smooth', 3000, 4000, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 92), 6)]
  model = make_model(1242, 375, len(files), 0)
  for s in (2, 4):
    frames, status = decode_jpeg_device(files, DEV, progressive=True, reduce=s)
    assert status.cpu().tolist() == [0, 0, 0]
    model.forward_device_frames(frames)
    got = fetch_results(model, 0)
    model.forward_device_frames([torch.from_numpy(imdecode(f, s)).to(DEV) for f in files])
    want = fetch_results(model, 0)
    for k in want:
      assert np.array_equal(got[k], want[k]), (s, k)
