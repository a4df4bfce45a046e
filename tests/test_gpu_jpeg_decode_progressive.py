"""decode_jpeg_device(progressive=True) / sqdet_decode_jpeg_progressive: frames bitwise
cv2.imdecode's for cv2's progressive files, foreign scan scripts and baseline files in mixed
batches, at camera sizes and through encode_jpeg_device(progressive=True); corrupt entropy data in a
first or a refinement scan fails only its own file."""
import cv2
import numpy as np
import pytest
import torch

from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import decode_jpeg_device, encode_jpeg_device, jpeg_bytes

from oracle import jpeg_decode_progressive as P
from oracle.jpeg_decode import CorruptData, parse

import jpeg_corpus as J
from gpu_util import fetch_results
import progressive_writer as W
from progressive_inputs import cap_frame

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
PROG = cv2.IMWRITE_JPEG_PROGRESSIVE


def prog_corpus(seed=0):
  """[(name, file)]: cv2 progressive files over the corpus kinds, sizes, samplings, qualities,
  restart intervals, grayscale and EXIF orientations, and the writer's foreign scripts."""
  rng = np.random.default_rng(seed)
  out = []
  for si, samp in enumerate(J.SAMPLINGS):
    for zi, (h, w) in enumerate(J.SIZES):
      kind = J.KINDS[(si + zi) % len(J.KINDS)]
      q = (1, 5, 25, 50, 75, 90, 95, 100)[(si * 3 + zi) % 8]
      rst = (0, 1, 3, 0, 7)[(si + zi) % 5]
      out.append(('prog %s %dx%d s%06x q%d r%d' % (kind, h, w, samp, q, rst),
                  J.encode(J.content(kind, h, w, 3, rng), PROG, 1, cv2.IMWRITE_JPEG_QUALITY, q,
                           cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp, cv2.IMWRITE_JPEG_RST_INTERVAL, rst)))
  for q in (10, 85):
    out.append(('prog gray q%d' % q, J.encode(J.content('smooth', 45, 70, 1, rng)[..., 0], PROG, 1,
                                              cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, q // 40)))
  base = J.encode(J.content('smooth', 37, 58, 3, rng), PROG, 1)
  for o in range(1, 9):
    out.append(('prog exif %d' % o, J.with_orientation(base, o, o % 2 == 0)))
  for samp in (0x221111, 0x111111, 0x411111):
    f = J.encode(J.content('smooth', 45, 70, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90,
                 cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)
    for name, script in W.COMPLETE.items():
      out.append(('%s s%06x' % (name, samp), W.write(f, script)))
    out.append(('restarts s%06x' % samp, W.write(f, W.SPECTRAL, restarts={1: 2, 3: 0, 4: 5})))
    out.append(('dqt after s%06x' % samp, W.write(f, W.DC_SUBSETS, dqt_after=1)))
    for name, script in W.UNSMOOTHED.items():
      out.append(('%s s%06x' % (name, samp), W.write(f, script)))
  g = J.encode(J.content('noise', 45, 70, 1, rng)[..., 0])
  out.append(('gray deep', W.write(g, W.GRAY_DEEP, restarts={0: 3, 4: 1, 8: 0})))
  out.append(('0x7fff eobrun', J.encode(cap_frame(), PROG, 1)))
  # RSTn markers after a scan's last interval, which libjpeg skips
  f = J.encode(J.content('smooth', 32, 48, 3, rng), PROG, 1)
  out += [('trailing rst %d x%d' % (i, k), W.with_trailing_rst(f, i, k)) for i, k in ((0, 1), (3, 2), (9, 9))]
  f = J.encode(J.content('noise', 45, 70, 3, rng), PROG, 1, cv2.IMWRITE_JPEG_RST_INTERVAL, 2)
  out.append(('trailing rst after intervals', W.with_trailing_rst(f, 2, 3)))
  return out


@pytest.fixture(scope='module')
def mixed():
  items = prog_corpus() + J.corpus(seed=1, big=False)
  rng = np.random.default_rng(5)
  return [items[i] for i in rng.permutation(len(items))]


@pytest.fixture
def sub_bits():
  lib = _lib.load()
  yield lambda bits: _lib.check(lib.sqdet_jpeg_decode_set_subsequence_bits(bits))
  _lib.check(lib.sqdet_jpeg_decode_set_subsequence_bits(0))


def check_batch(named):
  frames, status = decode_jpeg_device([f for _, f in named], DEV, progressive=True)
  st = status.cpu().numpy()
  for (name, f), fr, s in zip(named, frames, st):
    want = J.imdecode(f)
    assert s == 0, '%s: status %d' % (name, s)
    got = fr.cpu().numpy()
    assert got.shape == want.shape, name
    assert np.array_equal(got, want), '%s: %d pixels differ' % (name, int((got != want).any(2).sum()))


def batches(items, sizes=(1, 7, 32, 19, 3, 128)):
  i, k = 0, 0
  while i < len(items):
    n = sizes[k % len(sizes)]
    yield items[i:i + n]
    i += n
    k += 1


def test_mixed_batches(mixed):
  for b in batches(mixed):
    check_batch(b)


def test_batch_of_128(mixed):
  check_batch((mixed * 2)[:128])


def test_baseline_files_as_the_plain_call():
  files = [f for _, f in J.corpus(seed=2, big=False)][:40]
  a, sa = decode_jpeg_device(files, DEV)
  b, sb = decode_jpeg_device(files, DEV, progressive=True)
  assert torch.equal(sa, sb)
  assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize('bits', [32, 64])
def test_small_subsequences(mixed, sub_bits, bits):
  """The subsequence size applies to the sequential files of a mixed batch; the progressive files
  beside them must come out unchanged."""
  sub_bits(bits)
  for b in batches(mixed, sizes=(32, 17)):
    check_batch(b)


def test_camera_sizes():
  rng = np.random.default_rng(7)
  cam = [(name, J.encode(J.imdecode(f), PROG, 1, cv2.IMWRITE_JPEG_QUALITY, 92))
         for name, f in J.camera()[:2]]
  cam += [('1x8191', J.encode(J.content('smooth', 1, 8191, 3, rng), PROG, 1)),
          ('8191x1', J.encode(J.content('smooth', 8191, 1, 3, rng), PROG, 1))]
  for item in cam:
    check_batch([item])


@pytest.mark.parametrize('fmt', ['bgr', 'nv12', 'rgba'])
def test_round_trip(fmt):
  rng = np.random.default_rng(11)
  bgr = J.content('smooth', 120, 170, 3, rng)
  if fmt == 'bgr':
    frame = torch.from_numpy(bgr).to(DEV)
  elif fmt == 'rgba':
    frame = torch.from_numpy(cv2.cvtColor(bgr, cv2.COLOR_BGR2RGBA)).to(DEV)
  else:
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    y, u, v = i420[:120], i420[120:150].reshape(60, 85), i420[150:].reshape(60, 85)
    frame = torch.from_numpy(np.concatenate([y, np.stack([u, v], -1).reshape(60, 170)])).to(DEV)
  for sampling, rst in (('420', 0), ('444', 3), ('422', 1)):
    data, lengths = encode_jpeg_device([frame], fmt, progressive=True, sampling=sampling,
                                       restart_interval=rst)
    files = jpeg_bytes(data, lengths)
    check_batch([('%s %s r%d' % (fmt, sampling, rst), files[0])])


def corrupt(f, scan_index):
  """f with bytes in the middle of its scan_index-th scan's data changed (no 0xFF written)."""
  b = bytearray(f)
  at = [i for i in range(len(b) - 1) if b[i] == 0xFF and b[i + 1] == 0xDA][scan_index]
  n = int.from_bytes(b[at + 2:at + 4], 'big')
  start = at + 2 + n
  end = start
  while not (b[end] == 0xFF and b[end + 1] not in (0x00,) and not 0xD0 <= b[end + 1] <= 0xD7):
    end += 1
  for k in range(start + (end - start) // 3, start + (end - start) // 3 + 6):
    if b[k] != 0xFF and b[k - 1] != 0xFF:
      b[k] = 0xFE
  return bytes(b)


def test_corrupt_scans_fail_only_their_file():
  """Corrupt progressive and sequential files interleaved: each status lands at its file's index,
  whichever stages decode the file."""
  rng = np.random.default_rng(13)
  good = [('good %d' % i, J.encode(J.content('smooth', 64, 96, 3, rng), PROG, 1)) for i in range(3)]
  good.append(('good baseline', J.encode(J.content('smooth', 64, 96, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90)))
  noise = J.encode(J.content('noise', 64, 96, 3, rng), PROG, 1, cv2.IMWRITE_JPEG_QUALITY, 100)
  # a first scan, a refinement and data that runs out inside the last scan (a file cut earlier
  # would miss whole scans, which libjpeg smooths, so it is refused)
  bad = [corrupt(noise, 1), corrupt(noise, 5), noise[:len(noise) - 300], W.with_dri(noise, 1)]
  # baseline files: 0xFF 0x00 runs (all-ones bits, an invalid code) and an RSTn marker removed
  junk = bytearray(J.encode(J.content('smooth', 64, 96, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90))
  scan = parse(bytes(junk)).scan
  junk[scan + 10:scan + 50] = b'\xff\x00' * 20
  rst = J.encode(J.content('smooth', 64, 96, 3, rng), cv2.IMWRITE_JPEG_RST_INTERVAL, 2)
  k = rst.index(b'\xff\xd1', parse(rst).scan)
  bad += [bytes(junk), rst[:k] + rst[k + 2:]]
  for f in bad:                       # corrupt as the oracle sees it too
    with pytest.raises(CorruptData):
      P.decode(f)
  files = [good[0][1], bad[4], bad[0], good[3][1], good[1][1], bad[1], bad[5], bad[2], good[2][1], bad[3]]
  frames, status = decode_jpeg_device(files, DEV, progressive=True)
  st = status.cpu().numpy()
  assert all(st[k] < 0 for k in (1, 2, 5, 6, 7, 9)), st
  for k, (name, f) in zip((0, 4, 8, 3), good):
    assert st[k] == 0, (name, st)
    assert np.array_equal(frames[k].cpu().numpy(), J.imdecode(f)), name


def test_forward_on_decoded_frames():
  from squeezedet_b200.bench_device_frames import make_model
  rng = np.random.default_rng(17)
  files = [J.encode(J.content('smooth', 375, 1242, 3, rng), PROG, 1, cv2.IMWRITE_JPEG_QUALITY, q)
           for q in (95, 60, 85)]
  model = make_model(1242, 375, len(files), 0)
  frames, status = decode_jpeg_device(files, DEV, progressive=True)
  assert status.cpu().tolist() == [0, 0, 0]
  model.forward_device_frames(frames)
  got = fetch_results(model, 0)
  model.forward_device_frames([torch.from_numpy(J.imdecode(f)).to(DEV) for f in files])
  want = fetch_results(model, 0)
  for k in want:
    assert np.array_equal(got[k], want[k]), k
