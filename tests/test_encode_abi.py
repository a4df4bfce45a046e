"""sqdet_encode_jpeg and sqdet_encode_png make the same checks, in the same order, before any device
work: each refusal here is asked of both encoders, so without a GPU too, except the last test,
which needs device memory."""
import ctypes as C

import numpy as np
import pytest

from squeezedet_b200 import _lib

FMT_BGR, FMT_NV12 = 0, 5
FAKE = 1 << 40            # never dereferenced: the argument checks come first
CODECS = ('jpeg', 'png')


def arrays(n=1, h=16, w=16, crops=None):
  hs, ws = (C.c_int32 * n)(*[h] * n), (C.c_int32 * n)(*[w] * n)
  cr = None if crops is None else (C.c_int32 * (4 * n))(*crops)
  return hs, ws, cr


def host_planes(n=1):
  buf = (C.c_uint8 * 4096)()
  p = (C.c_void_p * (3 * n))(*[C.addressof(buf)] * (3 * n))
  p._keep = buf
  return p


def call(codec, n, fmt, planes, heights, widths, crops, out, cap, lengths, scratch, scratch_bytes):
  """sqdet_encode_<codec> (JPEG at quality 95) with these arguments."""
  lib = _lib.load()
  if codec == 'jpeg':
    return lib.sqdet_encode_jpeg(n, fmt, planes, None, heights, widths, crops, 95, out, cap, lengths,
                                 scratch, scratch_bytes, None)
  return lib.sqdet_encode_png(n, fmt, planes, None, heights, widths, crops, out, cap, lengths, scratch,
                              scratch_bytes, None)


def encode(codec, n=1, fmt=FMT_BGR, planes='host', h=16, w=16, crops=None, out=FAKE, cap=1 << 20,
           lengths=FAKE, scratch=FAKE, scratch_bytes=1 << 40):
  hs, ws, cr = arrays(max(n, 1), h, w, crops)
  pl = host_planes(max(n, 1)) if planes == 'host' else planes
  return call(codec, n, fmt, pl, hs, ws, cr, out, cap, lengths, scratch, scratch_bytes)


def refused(rc, *words):
  assert rc == -1
  msg = _lib.load().sqdet_last_error()
  assert all(w.encode() in msg for w in words), msg


@pytest.mark.parametrize('codec', CODECS)
def test_null_arguments(codec):
  hs, ws, _ = arrays()
  pl = host_planes()
  for args in [(None, hs, ws), (pl, None, ws), (pl, hs, None)]:
    refused(call(codec, 1, FMT_BGR, *args, None, FAKE, 100, FAKE, FAKE, 1 << 30), 'null')
  refused(encode(codec, out=None), 'null')
  refused(encode(codec, lengths=None), 'null')
  refused(encode(codec, scratch=None), 'null')


@pytest.mark.parametrize('codec', CODECS)
def test_counts_format_cap(codec):
  refused(encode(codec, n=0), 'n must be in [1, 128]')
  refused(encode(codec, n=129), 'n must be in [1, 128]')
  refused(encode(codec, fmt=7), 'unknown format')
  refused(encode(codec, fmt=-1), 'unknown format')
  refused(encode(codec, cap=0), 'cap')


@pytest.mark.parametrize('codec', CODECS)
def test_frame_refusals(codec):
  refused(encode(codec, h=0), 'frame 0 is empty')
  refused(encode(codec, crops=[0, 0, 0, 4]), 'empty crop')
  refused(encode(codec, crops=[10, 0, 8, 4]), 'crop outside the frame')
  refused(encode(codec, crops=[10, 0, 10, 4]), 'crop outside the frame')
  refused(encode(codec, fmt=FMT_NV12, h=15, w=16), 'even')
  null_plane = (C.c_void_p * 3)(None, None, None)
  refused(encode(codec, planes=null_plane, fmt=FMT_BGR), 'null pointer')


@pytest.mark.parametrize('codec', CODECS)
def test_misaligned_scratch_or_lengths(codec):
  """The scratches hold 16-byte vector, int64, 16-bit and 32-bit atomic regions and lengths_dev
  int64s: a misaligned pointer is refused rather than faulting a kernel."""
  for off in (1, 8, 16, 128):
    refused(encode(codec, scratch=FAKE + off), 'scratch_dev must be 256-byte aligned')
  for off in (1, 4):
    refused(encode(codec, lengths=FAKE + off), 'lengths_dev must be 8-byte aligned')
  refused(encode(codec, out=FAKE + 1), 'frame 0')        # out_dev may start at any byte


@pytest.mark.parametrize('codec', CODECS)
def test_scratch_too_small(codec):
  hs, ws, _ = arrays()
  need = getattr(_lib.load(), 'sqdet_%s_scratch_bytes' % codec)(1, hs, ws, None)
  for sb in (100, need - 1):
    refused(encode(codec, scratch_bytes=sb), 'scratch_bytes is below sqdet_%s_scratch_bytes' % codec)


@pytest.mark.parametrize('codec', CODECS)
def test_memory_not_on_a_device(codec):
  """Host memory for the frames, the output or the scratch is refused, naming it."""
  refused(encode(codec), 'frame 0', 'not inside one device allocation')


@pytest.mark.gpu
@pytest.mark.parametrize('codec', CODECS)
def test_outputs_outside_a_device_allocation(codec, gpu_device):
  """With device frames, an output, lengths or scratch in host memory, an output or scratch running
  past the end of its cudaMalloc allocation, or a misaligned scratch or lengths, is refused before
  any device work."""
  import cv2
  import torch

  from squeezedet_b200._lib import DeviceBuffer
  from gpu_util import content
  lib = _lib.load()
  frame = torch.from_numpy(content('noise', 32, 48, 3, np.random.default_rng(0))).to(gpu_device)
  planes = (C.c_void_p * 3)(frame.data_ptr(), None, None)
  hs, ws = (C.c_int32 * 1)(32), (C.c_int32 * 1)(48)
  sb = getattr(lib, 'sqdet_%s_scratch_bytes' % codec)(1, hs, ws, None)
  cap = getattr(lib, 'sqdet_%s_max_bytes' % codec)(32, 48)
  up = lambda v: -(-v // 512) * 512
  out = DeviceBuffer(up(cap), gpu_device)
  out_short = DeviceBuffer(up(cap) - 512, gpu_device)                   # shorter than cap
  lengths = DeviceBuffer(512, gpu_device)
  scratch = DeviceBuffer(up(sb), gpu_device)
  host_buf = np.zeros(up(max(cap, sb)) + 256, np.uint8)
  host = host_buf[-host_buf.ctypes.data % 256:]                         # 256-byte aligned
  lib.sqdet_memcpy_h2d(lengths.ptr, np.full(1, 7, np.int64).ctypes.data, 8, None)
  lib.sqdet_memcpy_h2d(out.ptr, host.ctypes.data, up(cap), None)

  def encode_dev(o, ln, sc, sbytes):
    return call(codec, 1, FMT_BGR, planes, hs, ws, None, o, cap, ln, sc, sbytes)

  cases = {
      'out in host memory': (host.ctypes.data, lengths.ptr, scratch.ptr, sb),
      'out past its allocation': (out_short.ptr, lengths.ptr, scratch.ptr, sb),
      'lengths in host memory': (out.ptr, host.ctypes.data, scratch.ptr, sb),
      'scratch in host memory': (out.ptr, lengths.ptr, host.ctypes.data, sb),
      'scratch past its allocation': (out.ptr, lengths.ptr, scratch.ptr, up(sb) + 512),
  }
  accepted = []
  for what, args in cases.items():
    rc = encode_dev(*args)
    if rc != -1 or b'not inside one device allocation' not in lib.sqdet_last_error():
      accepted.append((what, rc, lib.sqdet_last_error()))
  assert not accepted, accepted
  rc = encode_dev(out.ptr, lengths.ptr, scratch.ptr + 16, sb - 512)
  assert rc == -1 and b'256-byte aligned' in lib.sqdet_last_error()
  rc = encode_dev(out.ptr, lengths.ptr + 4, scratch.ptr, sb)
  assert rc == -1 and b'8-byte aligned' in lib.sqdet_last_error()
  # nothing ran: the output and the length are as they were, and then a good call works
  assert lengths.to_numpy(np.int64, (1,))[0] == 7 and not out.to_numpy(np.uint8, (up(cap),)).any()
  _lib.check(encode_dev(out.ptr, lengths.ptr, scratch.ptr, sb))
  n = int(lengths.to_numpy(np.int64, (1,))[0])
  params = [cv2.IMWRITE_JPEG_QUALITY, 95] if codec == 'jpeg' else []
  assert out.to_numpy(np.uint8, (up(cap),))[:n].tobytes() == cv2.imencode(
      '.' + codec, frame.cpu().numpy(), params)[1].tobytes()
