"""decode_jpeg_device / sqdet_decode_jpeg: the frames are bitwise cv2.imdecode's (and
oracle.jpeg_decode's) over the whole corpus, in mixed batches, through every synchronisation
path of the parallel Huffman decode; corrupt entropy data fails only its own file."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import decode_jpeg_device, encode_jpeg_device, jpeg_bytes

import jpeg_corpus as J
from gpu_util import fetch_results

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def corpus():
  return J.corpus(seed=0)


@pytest.fixture
def sub_bits():
  """Sets the subsequence size of the parallel Huffman decode for one test."""
  lib = _lib.load()
  yield lambda bits: _lib.check(lib.sqdet_jpeg_decode_set_subsequence_bits(bits))
  _lib.check(lib.sqdet_jpeg_decode_set_subsequence_bits(0))


def check_batch(named):
  files = [f for _, f in named]
  frames, status = decode_jpeg_device(files, DEV)
  st = status.cpu().numpy()
  for (name, f), fr, s in zip(named, frames, st):
    want = J.imdecode(f)
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


def test_corpus_mixed_batches(corpus):
  rng = np.random.default_rng(3)
  order = rng.permutation(len(corpus))
  for b in batches([corpus[i] for i in order]):
    check_batch(b)


@pytest.mark.parametrize('bits', [32, 64, 256])
def test_small_subsequences_cross_cta(corpus, sub_bits, bits):
  # a few hundred bits per subsequence puts many tiles of 128 subsequences in a small file, so the
  # synchronisation across CTAs runs on every file
  sub_bits(bits)
  small = [c for c in corpus if '1080' not in c[0]]
  for b in batches(small, sizes=(32, 17)):
    check_batch(b)


def sync_stress_files():
  rng = np.random.default_rng(9)
  out = []
  flat = J.content('flat', 720, 1280, 3, rng)                 # EOB-only blocks after the first
  out.append(('flat 720p', J.encode(flat, cv2.IMWRITE_JPEG_QUALITY, 90)))
  out.append(('flat gray 1080p', J.encode(flat[..., 0].repeat(2, 0)[:1080].repeat(2, 1)[:, :1920],
                                          cv2.IMWRITE_JPEG_QUALITY, 50)))
  chk = J.content('check', 240, 320, 3, rng)                  # the longest codes
  for samp in (0x111111, 0x221111):
    out.append(('check q100 s%x' % samp, J.encode(chk, cv2.IMWRITE_JPEG_QUALITY, 100,
                                                  cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)))
  out.append(('blocks q100', J.encode(J.content('blocks', 200, 264, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 100)))
  noise = J.content('noise', 96, 130, 3, rng)
  for samp in J.SAMPLINGS:
    out.append(('rst1 s%x' % samp, J.encode(noise, cv2.IMWRITE_JPEG_RST_INTERVAL, 1,
                                            cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp)))
  out.append(('rst1 smooth 1080p', J.encode(J.content('smooth', 1080, 1920, 3, rng),
                                             cv2.IMWRITE_JPEG_RST_INTERVAL, 1)))
  for q in (1, 100):
    out.append(('1x1 q%d' % q, J.encode(J.content('noise', 1, 1, 3, rng), cv2.IMWRITE_JPEG_QUALITY, q)))
  out.append(('tiny segment', J.encode(J.content('flat', 8, 8, 1, rng)[..., 0], cv2.IMWRITE_JPEG_QUALITY, 10)))
  return out


def test_handmade_files():
  # SOF1 with 16-bit tables up to dequantized values that overflow 16 bits, colour-space markers
  # libjpeg reads as YCbCr, and data and RSTs it skips
  check_batch(J.handmade())


@pytest.mark.parametrize('bits', [0, 32])
def test_sync_stress(sub_bits, bits):
  sub_bits(bits)
  check_batch(sync_stress_files())


def test_padded_pitch_odd_start(corpus):
  lib = _lib.load()
  named = [c for c in corpus if '1080' not in c[0]][::5][:24]
  files = [f for _, f in named]
  n = len(files)
  want = [J.imdecode(f) for f in files]
  bufs = [C.create_string_buffer(f, len(f)) for f in files]
  ptrs = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
  lens = (C.c_int64 * n)(*[len(f) for f in files])
  sb = lib.sqdet_jpeg_decode_staging_bytes(n, ptrs, lens)
  cb = lib.sqdet_jpeg_decode_scratch_bytes(n, ptrs, lens)
  staging = torch.empty((sb,), dtype=torch.uint8, pin_memory=True)
  scratch = torch.empty((cb,), dtype=torch.uint8, device=DEV)
  status = torch.full((n,), 7, dtype=torch.int32, device=DEV)
  outs, pitches, views = [], [], []
  for i, w in enumerate(want):
    h, wd = w.shape[:2]
    pitch = 3 * wd + 1 + 13 * (i % 4)
    off = 1 + i % 7
    buf = torch.full((off + h * pitch + 16,), 0xA5, dtype=torch.uint8, device=DEV)
    outs.append(buf.data_ptr() + off)
    pitches.append(pitch)
    views.append((buf, off, pitch, h, wd))
  _lib.check(lib.sqdet_decode_jpeg(n, ptrs, lens, (C.c_void_p * n)(*outs), (C.c_int64 * n)(*pitches),
                                   staging.data_ptr(), sb, scratch.data_ptr(), cb, status.data_ptr(), None))
  torch.cuda.synchronize()
  assert status.cpu().tolist() == [0] * n
  for (buf, off, pitch, h, wd), w, (name, _) in zip(views, want, named):
    host = buf.cpu().numpy()
    rows = host[off:off + h * pitch].reshape(h, pitch)
    assert np.array_equal(rows[:, :3 * wd].reshape(h, wd, 3), w), name
    assert (rows[:, 3 * wd:] == 0xA5).all() and (host[:off] == 0xA5).all(), name + ': wrote outside'
    assert (host[off + h * pitch:] == 0xA5).all(), name


@pytest.mark.parametrize('fmt', ['bgr', 'rgb', 'bgra', 'rgba', 'rgb_planar', 'nv12', 'i420'])
def test_round_trip(fmt):
  rng = np.random.default_rng(5)
  h, w = 120, 202
  img = J.content('smooth', h, w, 3, rng)
  if fmt in ('bgr', 'rgb', 'bgra', 'rgba'):
    code = {'bgr': None, 'rgb': cv2.COLOR_BGR2RGB, 'bgra': cv2.COLOR_BGR2BGRA, 'rgba': cv2.COLOR_BGR2RGBA}[fmt]
    frame = torch.from_numpy(img if code is None else cv2.cvtColor(img, code)).to(DEV)
  elif fmt == 'rgb_planar':
    rgb = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
    frame = tuple(torch.from_numpy(np.ascontiguousarray(rgb[..., i])).to(DEV) for i in range(3))
  else:
    yuv = J.content('smooth', h * 3 // 2, w, 1, rng)[..., 0]
    frame = (torch.from_numpy(yuv[:h]).to(DEV), torch.from_numpy(yuv[h:]).to(DEV)) if fmt == 'nv12' \
        else torch.from_numpy(yuv).to(DEV)
  data, lengths = encode_jpeg_device([frame], fmt, quality=90)
  f = jpeg_bytes(data, lengths)[0]
  frames, status = decode_jpeg_device([f], DEV)
  assert status.item() == 0
  assert np.array_equal(frames[0].cpu().numpy(), J.imdecode(f))


@pytest.mark.parametrize('order', ['demo', 'eval'])
def test_forward_on_decoded_frames(order):
  from squeezedet_b200.bench_device_frames import make_model
  rng = np.random.default_rng(11)
  files = [J.encode(J.content('smooth', h, w, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 95)
           for h, w in ((375, 1242), (480, 640), (1080, 1920))]
  model = make_model(1242, 375, len(files), 0)
  frames, status = decode_jpeg_device(files, DEV)
  assert status.cpu().tolist() == [0, 0, 0]
  model.forward_device_frames(frames, order=order)
  got = fetch_results(model, 0)
  uploaded = [torch.from_numpy(J.imdecode(f)).to(DEV) for f in files]
  model.forward_device_frames(uploaded, order=order)
  want = fetch_results(model, 0)
  for k in want:
    assert np.array_equal(got[k], want[k]), k


def test_corrupt_file_fails_alone(corpus):
  rng = np.random.default_rng(13)
  good = [c for c in corpus if '45x70' in c[0]][:6]
  base = J.encode(J.content('smooth', 64, 96, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90)
  rst = J.encode(J.content('smooth', 64, 96, 3, rng), cv2.IMWRITE_JPEG_RST_INTERVAL, 2)
  from oracle.jpeg_decode import parse
  scan = parse(base).scan
  bad = []
  for start in (20, 180):                   # flipped bits that reach an invalid code (a flip the
    flipped = bytearray(base)               # decoder resynchronises past is not detectable)
    for j in range(scan + start, scan + start + 4):
      flipped[j] ^= 0x5A
    bad.append(bytes(flipped))
  bad.append(base[:scan + (len(base) - scan) // 2])   # truncated entropy data
  bad.append(base[:scan + 3] + b'\xff\xd9')
  r = bytearray(rst)                        # an RST marker renumbered
  k = bytes(r).index(b'\xff\xd1', parse(rst).scan)
  r[k + 1] = 0xD5
  bad.append(bytes(r))
  r = bytearray(rst)                        # a bogus RST inserted
  k = scan + 30
  bad.append(bytes(r[:k]) + b'\xff\xd3' + bytes(r[k:]))
  junk = bytearray(base)                    # 0xFF 0x00 runs: invalid codes
  junk[scan + 10:scan + 50] = b'\xff\x00' * 20
  bad.append(bytes(junk))
  for b in bad:
    files = [g for _, g in good[:3]] + [b] + [g for _, g in good[3:]]
    frames, status = decode_jpeg_device(files, DEV)
    st = status.cpu().tolist()
    assert st[3] < 0, st
    for i, f in enumerate(files):
      if i != 3:
        assert st[i] == 0
        assert np.array_equal(frames[i].cpu().numpy(), J.imdecode(f))
