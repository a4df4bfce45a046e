"""JPEG files of uint8 frames in device memory (sqdet_encode_jpeg), byte for byte what cv2.imwrite /
cv2.imencode('.jpg', ...) writes for the same BGR image, with no frame copied to the host.

  data, lengths = encode_jpeg_device(frames, 'nv12', quality=95)
  files = jpeg_bytes(data, lengths)        # one bytes object per frame

Frames are torch CUDA tensors in any pixel format of ModelSkeleton.forward_device_frames_fmt and are
laid out as it takes them; crop i is written as cv2.imencode writes
cv2.cvtColor(frame_i, code)[y:y+h, x:x+w], with the format's code (oracle/pixfmt.py).  No engine is
needed."""
from __future__ import annotations

import ctypes as C

from . import _lib
from .nn_skeleton import PIXEL_FORMATS, ModelSkeleton


class _Frames:
  """ModelSkeleton's frame packing and checks, for frames on cuda:`gpu_id` without an engine."""
  _pack_frames = ModelSkeleton._pack_frames
  _frame_planes = ModelSkeleton._frame_planes

  def __init__(self, gpu_id):
    self.gpu_id = gpu_id


def _first_tensor(f):
  return f[0] if isinstance(f, (tuple, list)) else f


def max_bytes(h, w):
  """The largest JPEG file of an h x w image (sqdet_jpeg_max_bytes)."""
  if not (1 <= int(h) <= 65535 and 1 <= int(w) <= 65535):
    raise ValueError('a JPEG is 1 to 65535 pixels wide and high, got %dx%d' % (w, h))
  return int(_lib.load().sqdet_jpeg_max_bytes(int(h), int(w)))


def _torch_stream(stream, device):
  """`stream` (a torch.cuda.Stream, a raw cudaStream_t, or None for torch's current stream on
  `device`) as a torch stream, so that allocations can be ordered on it."""
  import torch
  if stream is None:
    return torch.cuda.current_stream(device)
  if isinstance(stream, torch.cuda.Stream):
    return stream
  raw = int(stream)
  return torch.cuda.default_stream(device) if raw == 0 else torch.cuda.ExternalStream(raw, device=device)


def encode_jpeg_device(frames, fmt, crops=None, quality=95, stream=None):
  """-> (data [n, cap] uint8, lengths [n] int64), both on the frames' device: frame i's file is
  data[i, :lengths[i]], and lengths[i] is -1 if it did not fit cap = the largest file of the
  largest crop.  Asynchronous on `stream` (a torch.cuda.Stream, a raw cudaStream_t, or None for
  torch's current stream): run it on the stream that wrote the frames, and read the results on it
  (jpeg_bytes with the same `stream`) or after synchronising it.  The outputs and the scratch are
  allocated on that stream.

  Every size is a worst case, so that nothing waits for the device: cap is what the crop would
  take if every block had its longest codes and every byte were 0xFF (sqdet_jpeg_max_bytes, about
  20 MB for 1920 x 1080, whose quality-95 files of natural pictures are under 1 MB), and the
  scratch is about 17 MB per 1080p frame of each group of 16.  128 1080p frames take about 2.6 GB
  of output; encode fewer frames per call where that matters."""
  import torch
  frames = list(frames)
  if not 1 <= len(frames) <= 128:
    raise ValueError('need 1 to 128 frames, got %d' % len(frames))
  if fmt not in PIXEL_FORMATS:
    raise ValueError('fmt must be one of %s, got %r' % (', '.join(PIXEL_FORMATS), fmt))
  if not 1 <= int(quality) <= 100:
    raise ValueError('quality must be in [1, 100], got %r' % (quality,))
  device = getattr(_first_tensor(frames[0]), 'device', None)
  if getattr(device, 'type', None) != 'cuda':
    raise ValueError('frame 0: need a CUDA tensor, got %s' % (device,))
  n = len(frames)
  planes, pitches, hs, ws, rects = _Frames(device.index)._pack_frames(frames, fmt, crops)
  lib = _lib.load()
  cap = max(max_bytes(rects[4 * i + 3], rects[4 * i + 2]) for i in range(n))
  scratch_bytes = lib.sqdet_jpeg_scratch_bytes(n, hs, ws, rects)
  if scratch_bytes < 0:
    raise _lib.SqdetError(-1, lib.sqdet_last_error().decode('utf-8', 'replace'))
  s = _torch_stream(stream, device)
  # allocated on s: the caching allocator hands the scratch to a later allocation only in s's
  # order, after the encode has finished with it
  with torch.cuda.device(device), torch.cuda.stream(s):
    data = torch.empty((n, cap), dtype=torch.uint8, device=device)
    lengths = torch.empty((n,), dtype=torch.int64, device=device)
    scratch = torch.empty((scratch_bytes,), dtype=torch.uint8, device=device)
    _lib.check(lib.sqdet_encode_jpeg(n, PIXEL_FORMATS.index(fmt), planes, pitches, hs, ws, rects,
                                     int(quality), data.data_ptr(), cap, lengths.data_ptr(),
                                     scratch.data_ptr(), scratch_bytes, s.cuda_stream))
  return data, lengths


def jpeg_bytes(data, lengths, stream=None):
  """The files of encode_jpeg_device's (data, lengths) as bytes objects, copying back only each
  file's own bytes, in order after the work on `stream` (as encode_jpeg_device takes it: pass the
  encode's stream).  ValueError for a frame whose file did not fit."""
  import torch
  with torch.cuda.device(data.device), torch.cuda.stream(_torch_stream(stream, data.device)):
    lens = lengths.cpu().tolist()
    out = []
    for i, n in enumerate(lens):
      if n < 0:
        raise ValueError('frame %d: the file did not fit the output capacity' % i)
      out.append(data[i, :n].cpu().numpy().tobytes())
  return out
