"""Frames in device memory as the library's frame calls take them (sqdet_forward_frames,
sqdet_forward_tiles, sqdet_draw_dets, sqdet_encode_jpeg, sqdet_encode_png): the pixel formats, the
C arrays of a batch of uint8 CUDA tensors, the checks those calls share, and what the encoders
share: the call itself, its stream and the copy-back of the files."""
from __future__ import annotations

import ctypes as C

from . import _lib

# The pixel formats, in SQDET_FMT_* order
PIXEL_FORMATS = ('bgr', 'rgb', 'bgra', 'rgba', 'rgb_planar', 'nv12', 'i420')
# The pre-processing orders (SQDET_PRE_*): 'demo' resizes then subtracts the means, 'eval'
# subtracts then resizes
ORDERS = {'demo': 0, 'eval': 1}


def order_code(order):
  """The SQDET_PRE_* code of 'demo' or 'eval', or ValueError."""
  if order not in ORDERS:
    raise ValueError("order must be 'demo' or 'eval', got %r" % (order,))
  return ORDERS[order]


def frame_count(frames, most):
  """len(frames), or ValueError unless it is 1 to `most`."""
  n = len(frames)
  if not 1 <= n <= most:
    raise ValueError('need 1 to %d frames, got %d' % (most, n))
  return n


def pack_frames(frames, fmt, crops, gpu_id):
  """The C arrays (planes [3n], pitches [3n], heights [n], widths [n], crops [4n]) of the n frames
  on cuda:`gpu_id` in pixel format `fmt` and their crops (None, or per frame None for the whole
  frame or (x, y, w, h) inside it), or ValueError naming what does not fit."""
  if fmt not in PIXEL_FORMATS:
    raise ValueError('fmt must be one of %s, got %r' % (', '.join(PIXEL_FORMATS), fmt))
  n = len(frames)
  crops = [None] * n if crops is None else list(crops)
  if len(crops) != n:
    raise ValueError('need one crop (or None) per frame, got %d for %d frames' % (len(crops), n))
  planes, pitches, hs, ws, rects = [], [], [], [], []
  for i, f in enumerate(frames):
    h, w, ps = _frame_planes(i, f, fmt, gpu_id)
    rect = (0, 0, w, h) if crops[i] is None else tuple(int(v) for v in crops[i])
    x, y, cw, ch = rect if len(rect) == 4 else (0, 0, 0, 0)
    if len(rect) != 4 or cw < 1 or ch < 1 or x < 0 or y < 0 or x + cw > w or y + ch > h:
      raise ValueError('frame %d: crop %r is not a non-empty (x, y, w, h) inside %dx%d'
                       % (i, crops[i], w, h))
    ps = ps + [(None, 0)] * (3 - len(ps))
    planes.extend(p for p, _ in ps)
    pitches.extend(q for _, q in ps)
    hs.append(h)
    ws.append(w)
    rects.extend(rect)
  return ((C.c_void_p * (3 * n))(*planes), (C.c_int64 * (3 * n))(*pitches),
          (C.c_int32 * n)(*hs), (C.c_int32 * n)(*ws), (C.c_int32 * (4 * n))(*rects))


def first_tensor(f):
  """Frame f's tensor, or its first plane's when f is a tuple of planes."""
  return f[0] if isinstance(f, (tuple, list)) else f


def torch_stream(stream, device):
  """`stream` (a torch.cuda.Stream, a raw cudaStream_t, or None for torch's current stream on
  `device`) as a torch stream, so that allocations can be ordered on it."""
  import torch
  if stream is None:
    return torch.cuda.current_stream(device)
  if isinstance(stream, torch.cuda.Stream):
    return stream
  raw = int(stream)
  return torch.cuda.default_stream(device) if raw == 0 else torch.cuda.ExternalStream(raw, device=device)


def encode_frames(frames, fmt, crops, stream, max_bytes, scratch_call, encode_call, settle=tuple):
  """The files of an encoder (encode_jpeg_device, encode_png_device): the checks in this order
  (1 to 128 frames, fmt, the codec's settings, frame 0 on a CUDA device, pack_frames), then cap =
  max_bytes(h, w) of the largest crop, the scratch the C call `scratch_call` (n, heights, widths,
  crops, *extra) gives and the C call `encode_call` (n, format, planes, pitches, heights, widths,
  crops, *extra, data, cap, lengths, scratch, scratch_bytes, stream), where extra = settle() checks
  the codec's settings and holds its further arguments to both calls."""
  import torch
  frames = list(frames)
  n = frame_count(frames, 128)
  if fmt not in PIXEL_FORMATS:
    raise ValueError('fmt must be one of %s, got %r' % (', '.join(PIXEL_FORMATS), fmt))
  extra = settle()
  device = getattr(first_tensor(frames[0]), 'device', None)
  if getattr(device, 'type', None) != 'cuda':
    raise ValueError('frame 0: need a CUDA tensor, got %s' % (device,))
  planes, pitches, hs, ws, rects = pack_frames(frames, fmt, crops, device.index)
  lib = _lib.load()
  cap = max(max_bytes(rects[4 * i + 3], rects[4 * i + 2]) for i in range(n))
  nbytes = getattr(lib, scratch_call)(n, hs, ws, rects, *extra)
  if nbytes < 0:
    raise _lib.SqdetError(-1, lib.sqdet_last_error().decode('utf-8', 'replace'))
  s = torch_stream(stream, device)
  # allocated on s: the caching allocator hands the scratch to a later allocation only in s's
  # order, after the encode has finished with it
  with torch.cuda.device(device), torch.cuda.stream(s):
    data = torch.empty((n, cap), dtype=torch.uint8, device=device)
    lengths = torch.empty((n,), dtype=torch.int64, device=device)
    scratch = torch.empty((nbytes,), dtype=torch.uint8, device=device)
    _lib.check(getattr(lib, encode_call)(n, PIXEL_FORMATS.index(fmt), planes, pitches, hs, ws,
                                         rects, *extra, data.data_ptr(), cap, lengths.data_ptr(),
                                         scratch.data_ptr(), nbytes, s.cuda_stream))
  return data, lengths


def file_bytes(data, lengths, stream=None):
  """The files of an encoder's (data, lengths) as bytes objects, copying back only each file's own
  bytes, in order after the work on `stream` (as the encoder takes it: pass the encode's stream).
  ValueError for a frame whose file did not fit."""
  import torch
  with torch.cuda.device(data.device), torch.cuda.stream(torch_stream(stream, data.device)):
    lens = lengths.cpu().tolist()
    out = []
    for i, n in enumerate(lens):
      if n < 0:
        raise ValueError('frame %d: the file did not fit the output capacity' % i)
      out.append(data[i, :n].cpu().numpy().tobytes())
  return out


def _frame_planes(i, f, fmt, gpu_id):
  """(h, w, [(pointer, row pitch) per plane]) of frame i in `fmt`, or ValueError naming it."""
  def on_device(name, t):
    dtype, device = getattr(t, 'dtype', None), getattr(t, 'device', None)
    if str(dtype) != 'torch.uint8':
      raise ValueError('frame %d: need a uint8 %s tensor, got %s' % (i, name, dtype))
    if getattr(device, 'type', None) != 'cuda' or device.index != gpu_id:
      raise ValueError('frame %d: need a %s tensor on cuda:%d, got %s'
                       % (i, name, gpu_id, device))

  def plane(name, t, rows=None, cols=None):
    on_device(name, t)
    shape, stride = tuple(t.shape), tuple(t.stride())
    if (len(shape) != 2 or min(shape) < 1 or (rows is not None and shape[0] != rows)
        or (cols is not None and shape[1] != cols)):
      raise ValueError('frame %d: %s plane of shape %r does not fit' % (i, name, shape))
    pitch = stride[0] if shape[0] > 1 else shape[1]       # a single row's stride is never used
    if stride[1] != 1 or pitch < shape[1]:
      raise ValueError('frame %d: need %s strides (row, 1) with row >= w, got %r'
                       % (i, name, stride))
    return t.data_ptr(), pitch

  def even(h, w):
    if h < 2 or w < 2 or h % 2 or w % 2:
      raise ValueError('frame %d: need an even height and width of at least 2, got %dx%d'
                       % (i, w, h))

  def parts(k, what):
    if not isinstance(f, (tuple, list)):
      return None
    if len(f) != k:
      raise ValueError('frame %d: need a tensor or a %s tuple' % (i, what))
    return f

  shape = tuple(getattr(f, 'shape', ()))
  if fmt in ('bgr', 'rgb', 'bgra', 'rgba'):
    c = 4 if fmt in ('bgra', 'rgba') else 3
    on_device('frame', f)
    if len(shape) != 3 or shape[2] != c or shape[0] < 1 or shape[1] < 1:
      raise ValueError('frame %d: need shape [h, w, %d], got %r' % (i, c, shape))
    stride = tuple(f.stride())
    pitch = stride[0] if shape[0] > 1 else c * shape[1]   # a single row's stride is never used
    if stride[2] != 1 or stride[1] != c or pitch < c * shape[1]:
      raise ValueError('frame %d: need strides (row, %d, 1) with row >= %d * w, got %r'
                       % (i, c, c, stride))
    return shape[0], shape[1], [(f.data_ptr(), pitch)]
  if fmt == 'rgb_planar':
    rgb = parts(3, '(r, g, b)')
    if rgb is None:
      if len(shape) != 3 or shape[0] != 3:
        raise ValueError('frame %d: need shape [3, h, w], got %r' % (i, shape))
      rgb = (f[0], f[1], f[2])
    h, w = (tuple(getattr(rgb[0], 'shape', ())) + (0, 0))[:2]
    return h, w, [plane(name, t, h, w) for name, t in zip(('R', 'G', 'B'), rgb)]
  if fmt == 'nv12':
    yc = parts(2, '(luma, chroma)')
    if yc is None:
      if len(shape) != 2 or shape[0] % 3:
        raise ValueError('frame %d: need shape [3H/2, W], got %r' % (i, shape))
      h = 2 * shape[0] // 3
      yc = (f[:h], f[h:])
    h, w = (tuple(getattr(yc[0], 'shape', ())) + (0, 0))[:2]
    even(h, w)
    return h, w, [plane('luma', yc[0], h, w), plane('chroma', yc[1], h // 2, w)]
  yuv = parts(3, '(y, u, v)')
  if yuv is not None:
    h, w = (tuple(getattr(yuv[0], 'shape', ())) + (0, 0))[:2]
    even(h, w)
    return h, w, [plane('Y', yuv[0], h, w), plane('U', yuv[1], h // 2, w // 2),
                  plane('V', yuv[2], h // 2, w // 2)]
  on_device('frame', f)
  if len(shape) != 2 or shape[0] % 3:
    raise ValueError('frame %d: need shape [3h/2, w], got %r' % (i, shape))
  h, w = 2 * shape[0] // 3, shape[1]
  even(h, w)
  if tuple(f.stride()) != (w, 1):
    raise ValueError('frame %d: a stacked I420 frame must be tight, strides (%d, 1), got %r'
                     % (i, w, tuple(f.stride())))
  y = f.data_ptr()
  return h, w, [(y, w), (y + h * w, w // 2), (y + h * w + h * w // 4, w // 2)]
