"""encode_jpeg_device / sqdet_encode_jpeg: the files are byte for byte cv2.imencode's (and
oracle.jpeg's) of the crops converted to BGR, in every pixel format."""
import ctypes as C
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

import oracle.jpeg
from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import encode_jpeg_device, jpeg_bytes, max_bytes

from gpu_util import Frame, content, raw_encode, want

pytestmark = pytest.mark.gpu

FORMATS = ('bgr', 'rgb', 'bgra', 'rgba', 'rgb_planar', 'nv12', 'i420')
SIZES = [(1, 1), (1, 17), (17, 1), (2, 3), (8, 8), (15, 31), (16, 16), (17, 23), (61, 97),
         (375, 1242), (370, 1224), (376, 1241)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def even(v):
  return v + (v & 1)


@pytest.mark.parametrize('quality', [50, 95, 100])
@pytest.mark.parametrize('fmt', FORMATS)
def test_size_table_bitwise(fmt, quality, gpu_device):
  """The size table as one call of mixed sizes and contents; 4:2:0 frames are the next even size
  and cropped to the size at an odd origin where there is room."""
  rng = np.random.default_rng(quality)
  kinds = ('noise', 'grad', 'flat', 'check', 'blocks', 'dots')
  frames, crops = [], []
  for i, (h, w) in enumerate(SIZES):
    yuv = fmt in ('nv12', 'i420')
    fh, fw = (even(h + 1), even(w + 1)) if yuv else (h, w)
    frames.append(Frame(fmt, fh, fw, rng, gpu_device, kinds[i % len(kinds)]))
    crops.append((fw - w, fh - h, w, h))
  data, lengths = encode_jpeg_device([f.dev for f in frames], fmt, crops, quality)
  got = jpeg_bytes(data, lengths)
  for f, crop, g in zip(frames, crops, got):
    w = want(f, crop, quality)
    assert g == w, (fmt, quality, crop)
  x, y, cw, ch = crops[9]
  assert got[9] == oracle.jpeg.encode(np.ascontiguousarray(frames[9].bgr[y:y + ch, x:x + cw]), quality)


@pytest.mark.parametrize('quality', [50, 95, 100])
@pytest.mark.parametrize('fmt', FORMATS)
def test_1080p_bitwise(fmt, quality, gpu_device):
  rng = np.random.default_rng(7)
  frames = [Frame(fmt, 1080, 1920, rng, gpu_device, kind) for kind in ('noise', 'grad')]
  got = jpeg_bytes(*encode_jpeg_device([f.dev for f in frames], fmt, None, quality))
  for f, g in zip(frames, got):
    assert g == want(f, (0, 0, 1920, 1080), quality)


@pytest.mark.parametrize('fmt', FORMATS)
def test_pitched_planes_and_odd_crops(fmt, gpu_device):
  rng = np.random.default_rng(3)
  frames = [Frame(fmt, 64, 90, rng, gpu_device, 'noise', pad=13, off=1),
            Frame(fmt, 50, 36, rng, gpu_device, 'grad', pad=7, off=3)]
  if fmt == 'i420':                       # a stacked I420 frame is tight
    frames = [Frame(fmt, 64, 90, rng, gpu_device), Frame(fmt, 50, 36, rng, gpu_device)]
  crops = [(5, 3, 77, 41), (1, 7, 33, 43)]
  got = jpeg_bytes(*encode_jpeg_device([f.dev for f in frames], fmt, crops, 95))
  for f, c, g in zip(frames, crops, got):
    assert g == want(f, c, 95)


@pytest.mark.parametrize('fmt', FORMATS)
def test_128_frames_one_call(fmt, gpu_device):
  """128 frames of mixed sizes, contents and crops in one call: eight launch groups."""
  rng = np.random.default_rng(11 + FORMATS.index(fmt))
  frames, crops = [], []
  for i in range(128):
    h, w = 2 * int(rng.integers(1, 60)), 2 * int(rng.integers(1, 90))
    frames.append(Frame(fmt, h, w, rng, gpu_device, ('noise', 'grad', 'check', 'blocks')[i % 4]))
    x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
    crops.append((x, y, int(rng.integers(1, w - x + 1)), int(rng.integers(1, h - y + 1))))
  got = jpeg_bytes(*encode_jpeg_device([f.dev for f in frames], fmt, crops, 90))
  for f, c, g in zip(frames, crops, got):
    assert g == want(f, c, 90)


def test_raw_stream_that_is_not_current(gpu_device):
  """A raw cudaStream_t of a stream that is not torch's current one: the outputs and the scratch
  are allocated in that stream's order, so allocations made on the current stream while the
  encode runs cannot take the scratch.  A spin ahead of the encode keeps it in flight while the
  current stream allocates and writes many buffers."""
  rng = np.random.default_rng(8)
  frames = [Frame('bgr', 720, 1280, rng, gpu_device, kind) for kind in ('noise', 'grad', 'blocks')]
  side = torch.cuda.Stream(gpu_device)
  torch.cuda.synchronize(gpu_device)
  side_raw = side.cuda_stream
  assert torch.cuda.current_stream(gpu_device).cuda_stream != side_raw
  with torch.cuda.stream(side):
    torch.cuda._sleep(20_000_000)
  data, lengths = encode_jpeg_device([f.dev for f in frames], 'bgr', None, 95, stream=side_raw)
  junk = [torch.full((1 << 22,), 255, dtype=torch.uint8, device=gpu_device) for _ in range(64)]
  got = jpeg_bytes(data, lengths, stream=side_raw)
  del junk
  for f, g in zip(frames, got):
    assert g == want(f, (0, 0, 1280, 720), 95)


def test_cap_overflow_is_one_frame(gpu_device):
  rng = np.random.default_rng(5)
  hosts = [content('flat', 40, 40, 3, rng), content('noise', 40, 40, 3, rng),
           content('grad', 40, 40, 3, rng)]
  wants = [cv2.imencode('.jpg', h, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() for h in hosts]
  cap = max(len(wants[0]), len(wants[2]))
  assert len(wants[1]) > cap
  frames = [torch.from_numpy(h).to(gpu_device) for h in hosts]
  data, lengths, _ = raw_encode(frames, cap)
  torch.cuda.synchronize(gpu_device)
  lens = lengths.cpu().tolist()
  assert lens[1] == -1
  for i in (0, 2):
    assert lens[i] == len(wants[i])
    assert data[i, :lens[i]].cpu().numpy().tobytes() == wants[i]
  with pytest.raises(ValueError):
    jpeg_bytes(data, lengths)


def test_max_bytes_bounds_the_worst_content(gpu_device):
  """The checkerboard at quality 100 is among the largest files; it stays within max_bytes."""
  rng = np.random.default_rng(1)
  for h, w in [(1, 1), (16, 16), (17, 23)]:
    for kind in ('check', 'noise'):
      f = Frame('bgr', h, w, rng, gpu_device, kind)
      g = jpeg_bytes(*encode_jpeg_device([f.dev], 'bgr', None, 100))[0]
      assert g == want(f, (0, 0, w, h), 100)
      assert len(g) <= max_bytes(h, w)


def test_no_host_synchronisation(gpu_device):
  """The call returns while a kernel ahead of it on the same stream is still running."""
  rng = np.random.default_rng(2)
  frame = torch.from_numpy(content('noise', 1080, 1920, 3, rng)).to(gpu_device)
  stream = torch.cuda.Stream(gpu_device)
  data, lengths, scratch = raw_encode([frame], max_bytes(1080, 1920))   # warm up, allocate
  torch.cuda.synchronize(gpu_device)
  lib = _lib.load()
  planes = (C.c_void_p * 3)(frame.data_ptr(), None, None)
  hs, ws = (C.c_int32 * 1)(1080), (C.c_int32 * 1)(1920)
  with torch.cuda.stream(stream):
    torch.cuda._sleep(20_000_000)
    _lib.check(lib.sqdet_encode_jpeg(1, 0, planes, None, hs, ws, None, 95, data.data_ptr(),
                                     data.shape[1], lengths.data_ptr(), scratch.data_ptr(),
                                     scratch.numel(), stream.cuda_stream))
    assert not stream.query()
  stream.synchronize()
  n = int(lengths[0])
  assert data[0, :n].cpu().numpy().tobytes() == cv2.imencode(
      '.jpg', frame.cpu().numpy(), [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes()


def test_demo_video_tiles_writes_cv2_files(tmp_path, gpu_device):
  """demo.py --mode video --tiles writes the files cv2.imwrite writes for the drawn frames."""
  rng = np.random.default_rng(4)
  video = str(tmp_path / 'in.avi')
  vw = cv2.VideoWriter(video, cv2.VideoWriter_fourcc(*'MJPG'), 10, (1280, 720))
  for _ in range(3):
    vw.write(cv2.GaussianBlur(rng.integers(0, 256, (720, 1280, 3), dtype=np.uint8), (9, 9), 3))
  vw.release()
  out_dev, out_host = tmp_path / 'dev', tmp_path / 'host'
  env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
  for out, extra in ((out_dev, []), (out_host, ['--host_encode'])):
    subprocess.check_call([sys.executable, '-m', 'squeezedet_b200.demo', '--mode', 'video',
                           '--tiles', '--input_path', video, '--out_dir', str(out),
                           '--gpu', str(gpu_device), '--checkpoint', 'synthetic'] + extra, cwd=ROOT, env=env)
  names = sorted(os.listdir(out_host))
  assert names and names == sorted(os.listdir(out_dev))
  for name in names:
    assert (out_dev / name).read_bytes() == (out_host / name).read_bytes(), name
