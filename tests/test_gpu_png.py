"""encode_png_device / sqdet_encode_png: the files are byte for byte cv2.imencode('.png')'s (and
oracle.png's) of the crops converted to BGR, in every pixel format."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

import oracle.png
from squeezedet_b200 import _lib
from squeezedet_b200.png import MAX_SIDE, encode_png_device, max_bytes, png_bytes

import png_traps
from gpu_util import Frame

pytestmark = pytest.mark.gpu

FORMATS = ('bgr', 'rgb', 'bgra', 'rgba', 'rgb_planar', 'nv12', 'i420')
SIZES = [(1, 1), (1, 17), (17, 1), (2, 3), (8, 8), (15, 31), (16, 16), (17, 23), (61, 97),
         (375, 1242), (370, 1224), (376, 1241)]


def even(v):
  return v + (v & 1)


def want(frame, crop):
  x, y, w, h = crop
  return cv2.imencode('.png', np.ascontiguousarray(frame.bgr[y:y + h, x:x + w]))[1].tobytes()


@pytest.mark.parametrize('fmt', FORMATS)
def test_size_table_bitwise(fmt, gpu_device):
  """The size table as one call of mixed sizes and contents; 4:2:0 frames are the next even size
  and cropped to the size at an odd origin where there is room."""
  rng = np.random.default_rng(FORMATS.index(fmt))
  kinds = ('noise', 'grad', 'flat', 'check', 'blocks', 'dots')
  frames, crops = [], []
  for i, (h, w) in enumerate(SIZES):
    yuv = fmt in ('nv12', 'i420')
    fh, fw = (even(h + 1), even(w + 1)) if yuv else (h, w)
    frames.append(Frame(fmt, fh, fw, rng, gpu_device, kinds[i % len(kinds)]))
    crops.append((fw - w, fh - h, w, h))
  got = png_bytes(*encode_png_device([f.dev for f in frames], fmt, crops))
  for f, crop, g in zip(frames, crops, got):
    assert g == want(f, crop), (fmt, crop)
  x, y, cw, ch = crops[9]
  assert got[9] == oracle.png.encode(frames[9].bgr[y:y + ch, x:x + cw])


@pytest.mark.parametrize('fmt', FORMATS)
def test_pitched_planes_and_odd_crops(fmt, gpu_device):
  rng = np.random.default_rng(3)
  frames = [Frame(fmt, 64, 90, rng, gpu_device, 'noise', pad=13, off=1),
            Frame(fmt, 50, 36, rng, gpu_device, 'grad', pad=7, off=3)]
  if fmt == 'i420':                       # a stacked I420 frame is tight
    frames = [Frame(fmt, 64, 90, rng, gpu_device), Frame(fmt, 50, 36, rng, gpu_device)]
  crops = [(5, 3, 77, 41), (1, 7, 33, 43)]
  got = png_bytes(*encode_png_device([f.dev for f in frames], fmt, crops))
  for f, c, g in zip(frames, crops, got):
    assert g == want(f, c)


@pytest.mark.parametrize('fmt', ['bgr', 'nv12'])
def test_128_frames_one_call(fmt, gpu_device):
  """128 frames of mixed sizes, contents and crops in one call: eight launch groups."""
  rng = np.random.default_rng(11)
  kinds = ('noise', 'grad', 'flat', 'check', 'blocks', 'dots')
  frames, crops = [], []
  for i in range(128):
    h, w = int(rng.integers(1, 120)), int(rng.integers(1, 200))
    h, w = even(h), even(w)
    frames.append(Frame(fmt, h, w, rng, gpu_device, kinds[i % len(kinds)]))
    x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
    crops.append((x, y, w - x, h - y))
  got = png_bytes(*encode_png_device([f.dev for f in frames], fmt, crops))
  for f, c, g in zip(frames, crops, got):
    assert g == want(f, c), c


@pytest.mark.parametrize('fmt', FORMATS)
def test_1080p_bitwise(fmt, gpu_device):
  rng = np.random.default_rng(7)
  frames = [Frame(fmt, 1080, 1920, rng, gpu_device, kind) for kind in ('noise', 'grad', 'dots')]
  got = png_bytes(*encode_png_device([f.dev for f in frames], fmt))
  for f, g in zip(frames, got):
    assert g == want(f, (0, 0, 1920, 1080))


def test_traps_bitwise(gpu_device):
  """Every corner case of the oracle tests (stored blocks, empty final blocks, runs across rows
  and past 258, forced codes, the 15-bit repair, a zlib stream of 2 x 8192 bytes) in one call."""
  items = list(png_traps.traps().items())
  imgs = [img for _, (img, _) in items]
  got = png_bytes(*encode_png_device([torch.from_numpy(i).to(gpu_device) for i in imgs], 'bgr'))
  for (name, _), img, g in zip(items, imgs, got):
    assert g == cv2.imencode('.png', img)[1].tobytes(), name


def test_window_headers(gpu_device):
  """One-row images at every size where the zlib header's window field changes."""
  rng = np.random.default_rng(5)
  imgs = [rng.integers(0, 256, (1, w, 3), dtype=np.uint8) for w in png_traps.header_widths()]
  for first in range(0, len(imgs), 128):
    part = imgs[first:first + 128]
    got = png_bytes(*encode_png_device([torch.from_numpy(i).to(gpu_device) for i in part], 'bgr'))
    for img, g in zip(part, got):
      assert g == cv2.imencode('.png', img)[1].tobytes(), img.shape


@pytest.mark.parametrize('shape', [(1, MAX_SIDE), (MAX_SIDE, 1), (2, MAX_SIDE)])
def test_largest_sides(shape, gpu_device):
  rng = np.random.default_rng(9)
  img = rng.integers(0, 256, shape + (3,), dtype=np.uint8)
  img[:, : shape[1] // 2] = 40                       # half flat: runs and literals
  got = png_bytes(*encode_png_device([torch.from_numpy(img).to(gpu_device)], 'bgr'))
  assert got[0] == cv2.imencode('.png', img)[1].tobytes()


def test_capacity_overflow_leaves_others(gpu_device):
  """A frame whose file exceeds cap gets length -1; the other frames are bitwise right."""
  rng = np.random.default_rng(12)
  small = np.full((40, 40, 3), 3, np.uint8)
  big = rng.integers(0, 256, (40, 40, 3), dtype=np.uint8)
  lib = _lib.load()
  imgs = [torch.from_numpy(i).to(gpu_device) for i in (small, big, small)]
  n = 3
  planes = (C.c_void_p * (3 * n))(*sum([[t.data_ptr(), None, None] for t in imgs], []))
  hs, ws = (C.c_int32 * n)(*[40] * n), (C.c_int32 * n)(*[40] * n)
  sb = lib.sqdet_png_scratch_bytes(n, hs, ws, None)
  want_small = cv2.imencode('.png', small)[1].tobytes()
  cap = len(want_small) + 10
  assert cap < len(cv2.imencode('.png', big)[1].tobytes()) <= max_bytes(40, 40)
  data = torch.zeros((n, cap), dtype=torch.uint8, device=gpu_device)
  lengths = torch.zeros((n,), dtype=torch.int64, device=gpu_device)
  scratch = torch.empty((sb,), dtype=torch.uint8, device=gpu_device)
  _lib.check(lib.sqdet_encode_png(n, 0, planes, None, hs, ws, None, data.data_ptr(), cap,
                                  lengths.data_ptr(), scratch.data_ptr(), sb, None))
  torch.cuda.synchronize(gpu_device)
  lens = lengths.cpu().tolist()
  assert lens[1] == -1
  for i in (0, 2):
    assert data[i, :lens[i]].cpu().numpy().tobytes() == want_small
