"""decode_jpeg_device(any_layout=True) / sqdet_decode_jpeg_options: frames bitwise cv2.imdecode (IMREAD_COLOR
and IMREAD_REDUCED_COLOR_2/4/8) for CMYK, YCCK and RGB-coded files and samplings cv2's encoder never
writes, sequential and progressive, mixed with ordinary files whose frames stay those of the plain
call; a corrupt CMYK file fails alone; a 12 MP CMYK file at 1/4; and frames that give the forward's
records of cv2's frames."""
import cv2
import numpy as np
import pytest
import torch

from squeezedet_b200.jpeg import decode_jpeg_device

from oracle.jpeg_decode import with_orientation

import jpeg_corpus as J
import jpeg_layouts as JL
from gpu_util import fetch_results

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
FLAGS = {1: cv2.IMREAD_COLOR, 2: cv2.IMREAD_REDUCED_COLOR_2, 4: cv2.IMREAD_REDUCED_COLOR_4,
         8: cv2.IMREAD_REDUCED_COLOR_8}


def imdecode(f, s):
  return cv2.imdecode(np.frombuffer(f, np.uint8), FLAGS[s])


def layout_corpus():
  out = JL.corpus(seed=3)
  out += JL.remainders([(4, 2), (1, 1), (1, 1)], [JL.JFIF], seed=100)
  out += JL.remainders([(2, 2), (1, 1), (1, 1), (2, 2)], [JL.adobe(2)], seed=200)
  base = JL.make(37, 58, [(1, 2), (1, 1), (2, 1), (1, 2)], markers=[JL.adobe(0)], seed=7)
  out += [('cmyk exif %d' % o, with_orientation(base, o)) for o in range(1, 9)]
  return out


@pytest.fixture(scope='module')
def mixed():
  items = layout_corpus()
  ordinary = J.corpus(seed=1, big=False)[::2]
  items += [('ordinary ' + n, f) for n, f in ordinary]
  rng = np.random.default_rng(5)
  return [items[i] for i in rng.permutation(len(items))]


def check_batch(named, s):
  frames, status = decode_jpeg_device([f for _, f in named], DEV, progressive=True, reduce=s, any_layout=True)
  st = status.cpu().numpy()
  for (name, f), fr, code in zip(named, frames, st):
    want = imdecode(f, s)
    assert code == 0, '%s 1/%d: status %d' % (name, s, code)
    got = fr.cpu().numpy()
    assert got.shape == want.shape, (name, s)
    assert np.array_equal(got, want), '%s 1/%d: %d pixels differ' % (name, s, int((got != want).any(2).sum()))
  return frames


def batches(items, sizes=(1, 7, 32, 19, 3, 64)):
  i, k = 0, 0
  while i < len(items):
    n = sizes[k % len(sizes)]
    yield items[i:i + n]
    i += n
    k += 1


@pytest.mark.parametrize('s', (1, 2, 4, 8))
def test_mixed_batches(mixed, s):
  for b in batches(mixed):
    check_batch(b, s)


@pytest.mark.parametrize('s', (1, 4))
def test_ordinary_files_are_the_plain_call(mixed, s):
  batch = mixed[:96]
  frames = check_batch(batch, s)
  plain = [(k, f) for k, (n, f) in enumerate(batch) if n.startswith('ordinary ')]
  ref, st = decode_jpeg_device([f for _, f in plain], DEV, reduce=s)
  assert st.cpu().tolist() == [0] * len(plain)
  for (k, _), r in zip(plain, ref):
    assert torch.equal(frames[k], r)


def test_corrupt_cmyk_fails_alone():
  good = [JL.make(64, 96, [(2, 2), (1, 1), (1, 1), (2, 2)], seed=1),
          J.encode(J.content('smooth', 64, 96, 3, np.random.default_rng(2)), cv2.IMWRITE_JPEG_QUALITY, 90),
          JL.make(64, 96, [(1, 1)] * 3, markers=[JL.adobe(0)], seed=3, script=())]
  junk = bytearray(JL.make(64, 96, [(1, 1)] * 4, markers=[JL.adobe(2)], seed=4))
  k = junk.index(b'\xff\xda')
  junk[k + 40:k + 80] = b'\xff\x00' * 20
  for s in (1, 2, 8):
    frames, status = decode_jpeg_device([good[0], bytes(junk), good[1], good[2]], DEV, progressive=True,
                                        reduce=s, any_layout=True)
    st = status.cpu().tolist()
    assert st[1] < 0 and st[0] == st[2] == st[3] == 0, st
    for i, f in ((0, good[0]), (2, good[1]), (3, good[2])):
      assert np.array_equal(frames[i].cpu().numpy(), imdecode(f, s))


def test_camera_size_cmyk_reduced():
  img = J.imdecode(J.camera()[0][1])
  cmyk = np.concatenate([255 - img, np.full(img.shape[:2] + (1,), 30, np.uint8)], axis=2)
  f = with_orientation(JL.pillow(cmyk, 'CMYK', quality=92), 6)
  check_batch([('4000x3000 cmyk exif 6', f)], 4)


def test_forward_on_layout_frames():
  from squeezedet_b200.bench_device_frames import make_model
  rng = np.random.default_rng(17)
  img = J.content('smooth', 750, 2484, 3, rng)
  files = [JL.pillow(np.concatenate([img, img[..., :1]], axis=2), 'CMYK', quality=90),
           JL.pillow(img[..., ::-1].copy(), 'RGB', quality=90, keep_rgb=True),
           JL.make(600, 1000, [(1, 1), (2, 2), (2, 1)], markers=[JL.JFIF], seed=9)]
  model = make_model(1242, 375, len(files), 0)
  for s in (1, 2):
    frames, status = decode_jpeg_device(files, DEV, reduce=s, any_layout=True)
    assert status.cpu().tolist() == [0, 0, 0]
    model.forward_device_frames(frames)
    got = fetch_results(model, 0)
    model.forward_device_frames([torch.from_numpy(imdecode(f, s)).to(DEV) for f in files])
    want = fetch_results(model, 0)
    for k in want:
      assert np.array_equal(got[k], want[k]), (s, k)
