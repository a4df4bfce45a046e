"""encode_jpeg_device(progressive=True) (sqdet_encode_jpeg_progressive) gives cv2.imencode's bytes with
IMWRITE_JPEG_PROGRESSIVE, in every pixel format and sampling, at camera sizes, on the two inputs
that reach the rarer EOBRUN flushes and over several launch groups."""
import cv2
import numpy as np
import pytest
import torch

from oracle import jpeg_params
from squeezedet_b200.jpeg import (decode_jpeg_device, encode_jpeg_device, jpeg_bytes, jpeg_info,
                                  max_bytes)

from gpu_util import Frame
from progressive_inputs import CORRECTION_QUALITY, cap_frame, correction_frame

pytestmark = pytest.mark.gpu

FORMATS = ('bgr', 'rgb', 'bgra', 'rgba', 'rgb_planar', 'nv12', 'i420')
SAMPLINGS = tuple(jpeg_params.SAMPLING_FACTORS)
KINDS = ('noise', 'grad', 'flat', 'check', 'blocks', 'dots')
SETTINGS = [dict(), dict(restart_interval=1), dict(restart_interval=3, quality=50),
            dict(restart_interval=7, quality=100), dict(restart_interval=65535, quality=1),
            dict(luma_quality=90, chroma_quality=40), dict(luma_quality=70, chroma_quality=70),
            dict(optimize=True, restart_interval=2)]


def cv2_list(**kw):
  return jpeg_params.cv2_params(**kw) + [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]


def want(bgr, **kw):
  ok, buf = cv2.imencode('.jpg', np.ascontiguousarray(bgr), cv2_list(**kw))
  assert ok
  return buf.tobytes()


def even(v):
  return v + (v & 1)


def edge_sizes(sampling):
  hs, vs = jpeg_params.SAMPLING_FACTORS[sampling]
  mw, mh = 8 * hs, 8 * vs
  return [(1 + i % mh, 1 + i % mw) for i in range(0, max(mw, mh), 3)] + \
      [(mh + 1 + i % mh, mw + 1 + i % mw) for i in range(max(mw, mh))] + [(61, 97)]


def check_files(got, bgrs, device, **kw):
  """Each file is cv2's, parses as progressive, and decodes (cv2) to the pixels the device decoder
  gives for the device's baseline file of the same frame."""
  for g, bgr in zip(got, bgrs):
    assert g == want(bgr, **kw), kw
    info = jpeg_info(g)
    assert not info['supported'] and info['reason'] == 2, info
  base = jpeg_bytes(*encode_jpeg_device([torch.from_numpy(np.ascontiguousarray(b)).to(device) for b in bgrs],
                                        'bgr', None, **kw))
  frames, status = decode_jpeg_device(base, device)
  assert (status.cpu() == 0).all()
  for g, f in zip(got, frames):
    assert np.array_equal(cv2.imdecode(np.frombuffer(g, np.uint8), cv2.IMREAD_COLOR), f.cpu().numpy())


@pytest.mark.parametrize('sampling', SAMPLINGS)
@pytest.mark.parametrize('fmt', FORMATS)
def test_grid_bitwise(fmt, sampling, gpu_device):
  """Every MCU-edge remainder of the sampling, crops at odd origins, each call of one setting."""
  rng = np.random.default_rng(FORMATS.index(fmt) * 10 + SAMPLINGS.index(sampling))
  yuv = fmt in ('nv12', 'i420')
  frames, crops = [], []
  for i, (h, w) in enumerate(edge_sizes(sampling)):
    fh, fw = (even(h + 1), even(w + 1)) if yuv else (h + 1, w + 2)
    frames.append(Frame(fmt, fh, fw, rng, gpu_device, KINDS[i % len(KINDS)]))
    crops.append((fw - w, fh - h, w, h))
  bgrs = [f.bgr[y:y + h, x:x + w] for f, (x, y, w, h) in zip(frames, crops)]
  for kw in SETTINGS:
    kw = dict(kw, sampling=sampling)
    got = jpeg_bytes(*encode_jpeg_device([f.dev for f in frames], fmt, crops, progressive=True, **kw))
    for g, b, c in zip(got, bgrs, crops):
      assert g == want(b, **kw), (fmt, c, kw)
    if fmt == 'bgr':
      check_files(got, bgrs, f'cuda:{gpu_device}', **kw)


@pytest.mark.parametrize('sampling', SAMPLINGS)
@pytest.mark.parametrize('fmt', ['bgr', 'nv12'])
def test_camera_sizes(fmt, sampling, gpu_device):
  rng = np.random.default_rng(5)
  sizes = [(1080, 1920), (375, 1242), (370, 1224), (376, 1241)]
  if fmt == 'nv12':
    sizes = [(even(h), even(w)) for h, w in sizes]
  frames = [Frame(fmt, h, w, rng, gpu_device, kind) for (h, w), kind in zip(sizes, ('noise', 'grad', 'dots', 'noise'))]
  for kw in (dict(), dict(restart_interval=5, quality=75), dict(luma_quality=85, chroma_quality=60)):
    kw = dict(kw, sampling=sampling)
    got = jpeg_bytes(*encode_jpeg_device([f.dev for f in frames], fmt, None, progressive=True, **kw))
    check_files(got, [f.bgr for f in frames], f'cuda:{gpu_device}', **kw)


def test_eobrun_cap(gpu_device):
  """A flat frame of 33 024 luma blocks: each luma AC scan's EOBRUN reaches 0x7FFF."""
  img = cap_frame()
  for kw in (dict(), dict(restart_interval=40000), dict(sampling='444')):
    got = jpeg_bytes(*encode_jpeg_device([torch.from_numpy(img).to(f'cuda:{gpu_device}')], 'bgr', None,
                                         progressive=True, **kw))
    assert got[0] == want(img, **kw), kw


def test_correction_bit_overflow(gpu_device):
  """Refinement scans that buffer more than 937 correction bits before any symbol."""
  img, _ = correction_frame(256, 192)
  for kw in (dict(), dict(restart_interval=100)):
    kw = dict(kw, quality=CORRECTION_QUALITY, sampling='444')
    got = jpeg_bytes(*encode_jpeg_device([torch.from_numpy(img).to(f'cuda:{gpu_device}')], 'bgr', None,
                                         progressive=True, **kw))
    assert got[0] == want(img, **kw), kw


def test_worst_case_fits(gpu_device):
  """Noise at quality 100, 4:4:4 and an interval of one MCU fits max_bytes(..., progressive=True)."""
  rng = np.random.default_rng(9)
  kw = dict(quality=100, sampling='444', restart_interval=1)
  f = Frame('bgr', 97, 131, rng, gpu_device, 'noise')
  data, lengths = encode_jpeg_device([f.dev], 'bgr', None, progressive=True, **kw)
  assert data.shape[1] == max_bytes(97, 131, progressive=True, **kw)
  assert 0 < int(lengths[0]) <= data.shape[1]
  assert jpeg_bytes(data, lengths)[0] == want(f.bgr, **kw)


def test_many_frames_groups(gpu_device):
  """40 frames (three launch groups) of mixed sizes: each frame's tables and intervals are its own."""
  rng = np.random.default_rng(12)
  frames = [Frame('bgr', int(rng.integers(1, 200)), int(rng.integers(1, 300)), rng, gpu_device, KINDS[i % 6])
            for i in range(40)]
  for kw in (dict(restart_interval=2, sampling='422'), dict(sampling='411')):
    got = jpeg_bytes(*encode_jpeg_device([f.dev for f in frames], 'bgr', None, progressive=True, **kw))
    for f, g in zip(frames, got):
      assert g == want(f.bgr, **kw)
