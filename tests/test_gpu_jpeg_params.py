"""encode_jpeg_device with cv2's other JPEG parameters (sqdet_encode_jpeg_params): sampling factors,
optimized tables, restart intervals and separate luma and chroma quality give cv2.imencode's bytes,
in every pixel format, and every file decodes on the device to cv2.imdecode's pixels."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

from oracle import jpeg_params
from squeezedet_b200 import _lib
from squeezedet_b200.jpeg import decode_jpeg_device, encode_jpeg_device, jpeg_bytes, max_bytes

from gpu_util import Frame, raw_encode

pytestmark = pytest.mark.gpu

FORMATS = ('bgr', 'rgb', 'bgra', 'rgba', 'rgb_planar', 'nv12', 'i420')
SAMPLINGS = tuple(jpeg_params.SAMPLING_FACTORS)
KINDS = ('noise', 'grad', 'flat', 'check', 'blocks', 'dots')
SETTINGS = [dict(), dict(optimize=True), dict(restart_interval=1), dict(restart_interval=3, optimize=True),
            dict(luma_quality=90, chroma_quality=40), dict(luma_quality=70), dict(chroma_quality=20),
            dict(quality=100, optimize=True, restart_interval=7), dict(quality=1, restart_interval=65535),
            dict(quality=50, restart_interval=2)]


def even(v):
  return v + (v & 1)


def want(frame, crop, **kw):
  x, y, w, h = crop
  ok, buf = cv2.imencode('.jpg', np.ascontiguousarray(frame.bgr[y:y + h, x:x + w]),
                         jpeg_params.cv2_params(**kw))
  assert ok
  return buf.tobytes()


def check_decodes(files, device):
  frames, status = decode_jpeg_device(files, device)
  assert (status.cpu() == 0).all()
  for f, got in zip(files, frames):
    assert np.array_equal(got.cpu().numpy(), cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR))


def edge_sizes(sampling):
  hs, vs = jpeg_params.SAMPLING_FACTORS[sampling]
  mw, mh = 8 * hs, 8 * vs
  return [(1 + i % mh, 1 + i % mw) for i in range(0, max(mw, mh), 3)] + \
      [(mh + 1 + i % mh, mw + 1 + i % mw) for i in range(max(mw, mh))] + [(61, 97)]


@pytest.mark.parametrize('sampling', SAMPLINGS)
@pytest.mark.parametrize('fmt', FORMATS)
def test_grid_bitwise(fmt, sampling, gpu_device):
  """Every MCU-edge remainder of the sampling, crops at odd origins, each call of one setting."""
  rng = np.random.default_rng(FORMATS.index(fmt) * 10 + SAMPLINGS.index(sampling))
  sizes = edge_sizes(sampling)
  yuv = fmt in ('nv12', 'i420')
  frames, crops = [], []
  for i, (h, w) in enumerate(sizes):
    fh, fw = (even(h + 1), even(w + 1)) if yuv else (h + 1, w + 2)
    frames.append(Frame(fmt, fh, fw, rng, gpu_device, KINDS[i % len(KINDS)]))
    crops.append((fw - w, fh - h, w, h))
  for kw in SETTINGS:
    kw = dict(kw, sampling=sampling)
    data, lengths = encode_jpeg_device([f.dev for f in frames], fmt, crops, **kw)
    got = jpeg_bytes(data, lengths)
    for f, c, g in zip(frames, crops, got):
      assert g == want(f, c, **kw), (fmt, c, kw)
    if fmt == 'bgr':
      check_decodes(got, gpu_device)


@pytest.mark.parametrize('sampling', SAMPLINGS)
@pytest.mark.parametrize('fmt', ['bgr', 'nv12'])
def test_camera_sizes(fmt, sampling, gpu_device):
  rng = np.random.default_rng(5)
  sizes = [(1080, 1920), (375, 1242), (370, 1224), (376, 1241)]
  if fmt == 'nv12':
    sizes = [(even(h), even(w)) for h, w in sizes]
  frames = [Frame(fmt, h, w, rng, gpu_device, kind) for (h, w), kind in zip(sizes, ('noise', 'grad', 'dots', 'noise'))]
  for kw in (dict(optimize=True), dict(restart_interval=5), dict(luma_quality=85, chroma_quality=60),
             dict(optimize=True, restart_interval=120, quality=75)):
    kw = dict(kw, sampling=sampling)
    got = jpeg_bytes(*encode_jpeg_device([f.dev for f in frames], fmt, None, **kw))
    for f, g, (h, w) in zip(frames, got, sizes):
      assert g == want(f, (0, 0, w, h), **kw), (h, w, kw)
    check_decodes(got, gpu_device)


def test_worst_case_fits(gpu_device):
  """Noise at quality 100, 4:4:4, optimized tables and an interval of one MCU fits max_bytes."""
  rng = np.random.default_rng(9)
  kw = dict(quality=100, sampling='444', optimize=True, restart_interval=1)
  f = Frame('bgr', 97, 131, rng, gpu_device, 'noise')
  data, lengths = encode_jpeg_device([f.dev], 'bgr', None, **kw)
  assert data.shape[1] == max_bytes(97, 131, **kw)
  assert 0 < int(lengths[0]) <= data.shape[1]
  assert jpeg_bytes(data, lengths)[0] == want(f, (0, 0, 131, 97), **kw)


def test_default_params_are_sqdet_encode_jpeg(gpu_device):
  rng = np.random.default_rng(10)
  frames = [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).to(f'cuda:{gpu_device}')
            for h, w in ((61, 97), (480, 640))]
  for q in (1, 75, 95, 100):
    cap = max(max_bytes(t.shape[0], t.shape[1]) for t in frames)
    data, lengths, _ = raw_encode(frames, cap, q)
    torch.cuda.synchronize()
    old = [data[i, :int(lengths[i])].cpu().numpy().tobytes() for i in range(len(frames))]
    assert jpeg_bytes(*encode_jpeg_device(frames, 'bgr', None, q)) == old
    assert jpeg_bytes(*encode_jpeg_device(frames, 'bgr', None, q, sampling='420', optimize=False,
                                          restart_interval=0)) == old


def test_many_frames_groups(gpu_device):
  """40 frames (three launch groups) of mixed sizes with optimized tables and restart markers: each
  frame's tables and intervals are its own."""
  rng = np.random.default_rng(12)
  frames = [Frame('bgr', int(rng.integers(1, 200)), int(rng.integers(1, 300)), rng, gpu_device, KINDS[i % 6])
            for i in range(40)]
  for kw in (dict(optimize=True, restart_interval=2, sampling='422'), dict(optimize=True, sampling='411')):
    got = jpeg_bytes(*encode_jpeg_device([f.dev for f in frames], 'bgr', None, **kw))
    for f, g in zip(frames, got):
      h, w = f.bgr.shape[:2]
      assert g == want(f, (0, 0, w, h), **kw)
