"""encode_jpeg_device at every quality, at camera sizes and at the longest sides a JPEG may have, and
decode_jpeg_device on the longest strips and past cv2's limits: every file is bitwise
cv2.imencode's, every frame cv2.imdecode's.

The camera-size frames have more than 1024 chunks of 256 blocks, so the encoder's per-frame scan
of block sums runs a second round and carries the first round's total into it; 1080p has 192.
The strips have thousands of MCUs in one row, and luma's DC prediction walks back over the dummy
blocks of every MCU of a 1- or 8-high strip."""
import cv2
import numpy as np
import pytest
import torch

from oracle import jpeg_decode as D
from squeezedet_b200.jpeg import decode_jpeg_device, encode_jpeg_device, jpeg_bytes, max_bytes

import jpeg_corpus as J
from gpu_util import Frame, content, raw_encode, want

pytestmark = pytest.mark.gpu

FORMATS = ('bgr', 'rgb', 'bgra', 'rgba', 'rgb_planar', 'nv12', 'i420')
MAX_SIDE = 65500
DEV = torch.device('cuda', 0)


def block_chunks(h, w):
  """The encoder's chunks of 256 blocks (kChunk) for an h x w crop: six blocks per 16 x 16 MCU."""
  return -(-(-(-h // 16) * -(-w // 16) * 6) // 256)


def even(v):
  return v + (v & 1)


def encode_check(frames, crops, quality, fmt):
  """One encode_jpeg_device call -> the crops whose files are not cv2's."""
  got = jpeg_bytes(*encode_jpeg_device([f.dev for f in frames], fmt, crops, quality))
  crops = crops or [(0, 0, f.bgr.shape[1], f.bgr.shape[0]) for f in frames]
  return [(i, c) for i, (f, c, g) in enumerate(zip(frames, crops, got)) if g != want(f, c, quality)]


# ---- every quality ---------------------------------------------------------------------------------
@pytest.mark.parametrize('fmt', FORMATS)
def test_every_quality(fmt, gpu_device):
  """Qualities 1-100: below 50 the tables scale by 5000 / quality, and at low qualities their
  entries clamp to 255.  Six small frames of mixed sizes and contents per call, 4:2:0 frames
  cropped at odd origins."""
  rng = np.random.default_rng(FORMATS.index(fmt))
  yuv = fmt in ('nv12', 'i420')
  frames, crops = [], []
  for (h, w), kind in zip([(1, 1), (17, 23), (16, 16), (61, 97), (9, 40), (33, 8)],
                          ('noise', 'check', 'blocks', 'grad', 'dots', 'noise')):
    fh, fw = (even(h + 1), even(w + 1)) if yuv else (h + 2, w + 1)
    frames.append(Frame(fmt, fh, fw, rng, gpu_device, kind))
    crops.append((fw - w, fh - h, w, h))
  bad = {}
  for q in range(1, 101):
    wrong = encode_check(frames, crops, q, fmt)
    if wrong:
      bad[q] = wrong
  assert not bad, bad


# ---- camera sizes ----------------------------------------------------------------------------------
def test_camera_sizes_reach_a_second_scan_round():
  for h, w in [(3000, 4000), (4000, 3000), (2999, 3999), (3024, 4032)]:
    assert block_chunks(h, w) > 1024, (h, w)
  assert block_chunks(1080, 1920) == 192


@pytest.mark.parametrize('fmt', FORMATS)
def test_camera_sizes(fmt, gpu_device):
  """4000 x 3000 both ways up, gradient and noise, at quality 95 in one call."""
  rng = np.random.default_rng(40 + FORMATS.index(fmt))
  frames = [Frame(fmt, h, w, rng, gpu_device, kind)
            for h, w in [(3000, 4000), (4000, 3000)] for kind in ('grad', 'noise')]
  assert not encode_check(frames, None, 95, fmt)


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_camera_crop_at_odd_origin(fmt, gpu_device):
  f = Frame(fmt, 3000, 4000, np.random.default_rng(5), gpu_device, 'noise')
  assert not encode_check([f], [(1, 1, 3999, 2999)], 95, fmt)


def test_largest_camera_file(gpu_device):
  """4032 x 3024 noise at quality 100, the largest file at camera size (about 24 MB in 4:2:0):
  within max_bytes."""
  f = Frame('bgr', 3024, 4032, np.random.default_rng(6), gpu_device, 'noise')
  g = jpeg_bytes(*encode_jpeg_device([f.dev], 'bgr', None, 100))[0]
  assert g == want(f, (0, 0, 4032, 3024), 100)
  assert 20 << 20 < len(g) <= max_bytes(3024, 4032)


# ---- the longest sides -----------------------------------------------------------------------------
@pytest.mark.parametrize('quality', [95, 30])
def test_longest_sides_bgr(quality, gpu_device):
  rng = np.random.default_rng(quality)
  sizes = [(1, MAX_SIDE), (MAX_SIDE, 1), (16, MAX_SIDE), (MAX_SIDE, 16), (17, MAX_SIDE),
           (1, 8191), (8191, 1)]
  kinds = ('noise', 'grad', 'blocks', 'noise', 'check', 'grad', 'noise')
  frames = [Frame('bgr', h, w, rng, gpu_device, k) for (h, w), k in zip(sizes, kinds)]
  assert not encode_check(frames, None, quality, 'bgr')


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_longest_sides_420(fmt, gpu_device):
  """2-sample strips, and a 4-high strip cropped at (1, 1) to 3 x 65499."""
  rng = np.random.default_rng(7)
  frames = [Frame(fmt, h, w, rng, gpu_device, k)
            for (h, w), k in zip([(2, MAX_SIDE), (MAX_SIDE, 2), (4, MAX_SIDE)], ('noise', 'grad', 'noise'))]
  crops = [(0, 0, MAX_SIDE, 2), (0, 0, 2, MAX_SIDE), (1, 1, MAX_SIDE - 1, 3)]
  assert not encode_check(frames, crops, 95, fmt)


# ---- launch groups and capacity at camera size ----------------------------------------------------
def test_camera_frame_among_small_ones(gpu_device):
  """17 frames in one call, a 12 MP frame at index 5: two launch groups, and in the first the
  small frames' CTAs return early from the big frame's grid."""
  rng = np.random.default_rng(8)
  small = [(1, 1), (1, 17), (17, 1), (2, 3), (8, 8), (15, 31), (16, 16), (17, 23), (61, 97)]
  kinds = ('noise', 'grad', 'check', 'blocks', 'dots', 'flat')
  frames = []
  for i in range(17):
    h, w = (3000, 4000) if i == 5 else small[i % len(small)]
    frames.append(Frame('bgr', h, w, rng, gpu_device, kinds[i % len(kinds)]))
  assert not encode_check(frames, None, 90, 'bgr')


def test_capacity_at_camera_size(gpu_device):
  """A cap between the gradient's and the noise's file: only the noise frame gets -1, and the
  other frames' bytes are exact."""
  rng = np.random.default_rng(9)
  hosts = [content('grad', 3000, 4000, 3, rng), content('noise', 3000, 4000, 3, rng),
           content('blocks', 61, 97, 3, rng)]
  wants = [cv2.imencode('.jpg', h, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() for h in hosts]
  cap = (len(wants[0]) + len(wants[1])) // 2
  assert len(wants[0]) < cap < len(wants[1]) and len(wants[2]) < cap
  data, lengths, _ = raw_encode([torch.from_numpy(h).to(gpu_device) for h in hosts], cap)
  torch.cuda.synchronize(gpu_device)
  lens = lengths.cpu().tolist()
  assert lens[1] == -1, lens
  for i in (0, 2):
    assert lens[i] == len(wants[i])
    assert data[i, :lens[i]].cpu().numpy().tobytes() == wants[i]


# ---- the decoder on the longest strips, and past cv2's limits ---------------------------------------
def test_decode_longest_strips():
  """cv2 files of 65500-long strips in grayscale and every sampling, with and without a restart
  interval, and one with EXIF orientation 6, in one batch."""
  rng = np.random.default_rng(10)
  named = []
  for h, w in [(1, MAX_SIDE), (MAX_SIDE, 1), (16, MAX_SIDE), (MAX_SIDE, 16)]:
    img = J.content('smooth', h, w, 3, rng)
    for rst in (0, 7):
      named.append(('%dx%d gray rst %d' % (h, w, rst),
                    J.encode(img[..., 0], cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_RST_INTERVAL, rst)))
      named += [('%dx%d s%06x rst %d' % (h, w, s, rst),
                 J.encode(img, cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, s,
                          cv2.IMWRITE_JPEG_RST_INTERVAL, rst)) for s in J.SAMPLINGS]
  wide = J.encode(J.content('smooth', 16, MAX_SIDE, 3, rng), cv2.IMWRITE_JPEG_QUALITY, 90)
  named.append(('16x65500 exif 6', D.with_orientation(wide, 6)))
  frames, status = decode_jpeg_device([f for _, f in named], DEV)
  st = status.cpu().tolist()
  for (name, f), fr, s in zip(named, frames, st):
    want_img = J.imdecode(f)
    got = fr.cpu().numpy()
    assert s == 0 and got.shape == want_img.shape and np.array_equal(got, want_img), name


def test_device_round_trip_of_the_longest_strip(gpu_device):
  f = Frame('bgr', 1, MAX_SIDE, np.random.default_rng(11), gpu_device, 'grad')
  g = jpeg_bytes(*encode_jpeg_device([f.dev], 'bgr', None, 95))[0]
  assert g == want(f, (0, 0, MAX_SIDE, 1), 95)
  frames, status = decode_jpeg_device([g], DEV)
  assert status.cpu().tolist() == [0]
  assert np.array_equal(frames[0].cpu().numpy(), J.imdecode(g))


def with_size(f, h, w):
  b = bytearray(f)
  k = bytes(b).index(b'\xff\xc0')
  b[k + 5:k + 9] = h.to_bytes(2, 'big') + w.to_bytes(2, 'big')
  return bytes(b)


def test_decode_refuses_past_cv2s_limits():
  """A 65501-wide file and a file of more than 2^30 pixels: ValueError naming the file, before
  anything is allocated (a header of a few hundred bytes must not size gigabytes)."""
  ok = J.encode(J.content('smooth', 16, 16, 3, np.random.default_rng(12)))
  decode_jpeg_device([ok], DEV)                       # staging and allocator warm
  torch.cuda.synchronize(DEV)
  for h, w in [(16, MAX_SIDE + 1), (32768, 32769), (65535, 65535)]:
    bad = with_size(ok, h, w)
    before = torch.cuda.memory_allocated(DEV)
    with pytest.raises(ValueError, match='file 1.*larger than cv2 decodes'):
      decode_jpeg_device([ok, bad], DEV)
    assert torch.cuda.memory_allocated(DEV) == before, (h, w)
