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
from .frames import encode_frames, file_bytes, torch_stream

# cv2's IMWRITE_JPEG_SAMPLING_FACTOR value of each sampling encode_jpeg_device takes
SAMPLINGS = {'411': 0x411111, '420': 0x221111, '422': 0x211111, '440': 0x121111, '444': 0x111111}


def jpeg_params(quality=95, sampling='420', optimize=False, restart_interval=0, luma_quality=None,
                chroma_quality=None):
  """The sqdet_jpeg_params of these settings, checked as the C ABI checks them: qualities in
  [1, 100] (luma_quality and chroma_quality None when unset), sampling one of SAMPLINGS,
  restart_interval in [0, 65535] MCUs.  cv2.imencode clamps values out of range instead."""
  for name, q in (('quality', quality), ('luma_quality', luma_quality),
                  ('chroma_quality', chroma_quality)):
    if (q is not None or name == 'quality') and not 1 <= int(q) <= 100:
      raise ValueError('%s must be in [1, 100], got %r' % (name, q))
  if sampling not in SAMPLINGS:
    raise ValueError('sampling must be one of %s, got %r' % (', '.join(SAMPLINGS), sampling))
  if not 0 <= int(restart_interval) <= 65535:
    raise ValueError('restart_interval must be in [0, 65535], got %r' % (restart_interval,))
  return _lib.JpegParams(int(quality), -1 if luma_quality is None else int(luma_quality),
                         -1 if chroma_quality is None else int(chroma_quality), SAMPLINGS[sampling],
                         int(bool(optimize)), int(restart_interval))


def max_bytes(h, w, progressive=False, **params):
  """The largest JPEG file of an h x w image (sqdet_jpeg_max_bytes_params, or with progressive
  sqdet_jpeg_max_bytes_progressive) with the keyword settings of encode_jpeg_device.  Sides are at
  most 65500, libjpeg's JPEG_MAX_DIMENSION, as for cv2.imencode."""
  p = jpeg_params(**params)
  if not (1 <= int(h) <= 65500 and 1 <= int(w) <= 65500):
    raise ValueError('a JPEG is 1 to 65500 pixels wide and high, got %dx%d' % (w, h))
  fn = 'sqdet_jpeg_max_bytes_progressive' if progressive else 'sqdet_jpeg_max_bytes_params'
  return int(getattr(_lib.load(), fn)(int(h), int(w), C.byref(p)))


def encode_jpeg_device(frames, fmt, crops=None, quality=95, stream=None, *, sampling='420',
                       optimize=False, restart_interval=0, luma_quality=None, chroma_quality=None,
                       progressive=False):
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
  of output; encode fewer frames per call where that matters.

  The keywords are cv2's other JPEG parameters, and the file is what cv2.imencode writes with them:
  sampling ('411', '420', '422', '440' or '444': IMWRITE_JPEG_SAMPLING_FACTOR), optimize
  (IMWRITE_JPEG_OPTIMIZE: each frame's own optimal Huffman tables), restart_interval
  (IMWRITE_JPEG_RST_INTERVAL, in MCUs, 0 for none), luma_quality and chroma_quality
  (IMWRITE_JPEG_LUMA_QUALITY / _CHROMA_QUALITY: luma_quality replaces quality, chroma_quality
  counts only with it, and two different ones give 4:4:4 whatever `sampling` says).  4:4:4
  doubles the worst-case sizes of 4:2:0.  Values cv2 would clamp raise ValueError.

  progressive=True writes what cv2.imencode writes with IMWRITE_JPEG_PROGRESSIVE as well
  (sqdet_encode_jpeg_progressive): the same coefficients in jpeg_simple_progression's ten scans,
  each with its own optimal tables, so optimize has no effect; a restart interval counts blocks in
  the eight single-component scans.  Its worst-case cap is about 2.1 times the baseline one at
  4:2:0.  decode_jpeg_device(..., progressive=True) reads these files back."""
  settings = dict(quality=quality, sampling=sampling, optimize=optimize,
                  restart_interval=restart_interval, luma_quality=luma_quality,
                  chroma_quality=chroma_quality)
  kind = 'progressive' if progressive else 'params'
  return encode_frames(frames, fmt, crops, stream,
                       lambda h, w: max_bytes(h, w, progressive=progressive, **settings),
                       'sqdet_jpeg_scratch_bytes_' + kind,
                       'sqdet_encode_jpeg_' + kind, lambda: (C.byref(jpeg_params(**settings)),))


# the files of encode_jpeg_device's (data, lengths)
jpeg_bytes = file_bytes


# ---- decoding ------------------------------------------------------------------------------------
JPEG_TOO_LARGE = 10       # SQDET_JPEG_TOO_LARGE: past cv2's limits, so cv2.imdecode refuses it too
JPEG_BAD_PROGRESSION = 11  # SQDET_JPEG_BAD_PROGRESSION: cv2.imdecode returns None
JPEG_CODED_TOO_LARGE = 15  # SQDET_JPEG_CODED_TOO_LARGE: cv2.imdecode decodes it at this scale
JPEG_COMPONENTS = 6       # SQDET_JPEG_COMPONENTS: with any_layout, cv2.imdecode returns None too
JPEG_BAD_SAMPLING = 16    # SQDET_JPEG_BAD_SAMPLING: cv2.imdecode returns None
# the scales decode_jpeg_device takes: cv2's IMREAD_COLOR and IMREAD_REDUCED_COLOR_2, _4 and _8
REDUCTIONS = (1, 2, 4, 8)


def _decode_call(progressive, reduce, any_layout=False):
  """(suffix of the C functions, their sqdet_jpeg_decode_params / _options or None): the plain or
  _progressive functions at full size, the _params ones at a reduced scale, the _options ones
  with any_layout."""
  if reduce not in REDUCTIONS:
    raise ValueError('reduce must be one of %s, got %r' % (', '.join(map(str, REDUCTIONS)), reduce))
  if any_layout:
    return '_options', _lib.JpegDecodeOptions(int(bool(progressive)), reduce, 1)
  if reduce == 1:
    return ('_progressive' if progressive else ''), None
  return '_params', _lib.JpegDecodeParams(int(bool(progressive)), reduce)


def jpeg_info(file_bytes, progressive=False, reduce=1, any_layout=False):
  """sqdet_jpeg_parse of one file -> dict: height and width of the decoded frame (after the EXIF
  orientation, and at scale 1 / reduce), coded_height, coded_width, components, h_samp, v_samp
  (luma sampling), orientation, restart_interval, supported (bool), reason (a SQDET_JPEG_* code)
  and reason_text (the library's words for it).  With progressive, sqdet_jpeg_parse_progressive:
  whether decode_jpeg_device(..., progressive=True) decodes it; with reduce 2, 4 or 8,
  sqdet_jpeg_parse_params: whether decode_jpeg_device(..., reduce=reduce) does; with any_layout,
  sqdet_jpeg_parse_options: whether decode_jpeg_device(..., any_layout=True) does.  Host only."""
  kind, params = _decode_call(progressive, reduce, any_layout)
  b = bytes(file_bytes)
  info = _lib.JpegInfo()
  buf = C.create_string_buffer(b, len(b))
  lib = _lib.load()
  parse = getattr(lib, 'sqdet_jpeg_parse' + kind)
  rc = parse(buf, len(b), *((C.byref(params),) if params else ()), C.byref(info))
  if rc not in (_lib.OK, -3):
    _lib.check(rc)
  out = {k: int(getattr(info, k)) for k, _ in _lib.JpegInfo._fields_ if k != 'reserved'}
  out['supported'] = bool(out['supported'])
  out['reason_text'] = 'ok' if rc == _lib.OK else \
      lib.sqdet_last_error().decode('utf-8', 'replace').split('not supported: ', 1)[-1]
  return out


class _Staging:
  """Two pinned host staging buffers used in turn, each with the event recorded after the call
  that last read it.  A call waits (on the host) only for the call before the previous one, so it
  packs its files while the previous call's decode runs."""

  def __init__(self):
    self.bufs = [None, None]
    self.events = [None, None]
    self.turn = 0

  def get(self, nbytes):
    """-> (slot, buffer of at least nbytes), free to write."""
    import torch
    k = self.turn
    self.turn ^= 1
    if self.events[k] is not None:
      self.events[k].synchronize()
    if self.bufs[k] is None or self.bufs[k].numel() < nbytes:
      self.bufs[k] = torch.empty((max(nbytes, 1 << 20),), dtype=torch.uint8, pin_memory=True)
    return k, self.bufs[k]


_staging = {}


def decode_jpeg_device(files, device, stream=None, *, progressive=False, reduce=1, any_layout=False):
  """JPEG files (bytes-like, on the host) -> (frames, status): frames[i] is a uint8 [H, W, 3] BGR
  CUDA tensor on `device` with exactly the pixels of cv2.imdecode(files[i], cv2.IMREAD_COLOR), and
  status an int32 [n] CUDA tensor, 0 where the file decoded and negative where its entropy-coded
  data is corrupt (that frame's pixels are then unspecified; the others are unaffected).

  Decoded are baseline and extended sequential Huffman files with 8-bit samples, 1 or 3
  components and 4:4:4, 4:2:2, 4:4:0, 4:2:0 or 4:1:1 sampling, with or without restart markers;
  the EXIF orientation is applied.  ValueError, naming the file's index, for any other file
  (progressive, arithmetic, 12-bit, CMYK, ...): route those to cv2.imdecode.  A file whose coded
  side is above 65500 (libjpeg's JPEG_MAX_DIMENSION) or with more than 2^30 coded pixels (cv2's
  default CV_IO_MAX_IMAGE_PIXELS) raises ValueError too, before anything is allocated; cv2.imdecode
  decodes none of those either.  1 to 128 files.

  Asynchronous on `stream` (a torch.cuda.Stream, a raw cudaStream_t, or None for torch's current
  stream): the frames, status and scratch are allocated on it, so read them on it or after
  synchronising it.  The files go to the device through two pinned staging buffers this module
  owns per device and uses in turn; a call waits (on the host) only until the call before the
  previous one has finished on its stream.

  progressive=True (sqdet_decode_jpeg_progressive) decodes progressive (SOF2) files too, in the
  same batch, again to exactly cv2.imdecode's pixels; the other files give the frames of the plain
  call.  Besides the plain call's refusals it raises ValueError for a scan script libjpeg rejects
  (cv2.imdecode returns None) or warns on or lets overwrite a coefficient, for a scan whose
  components are out of the frame's order, for a file libjpeg would block-smooth (an incomplete
  one: complete files, such as every file cv2 or encode_jpeg_device writes, are not smoothed) and
  for more than 256 scans; route those to cv2.imdecode.  A progressive scan without restart
  markers is decoded by one GPU lane, so these files decode much slower than sequential ones.

  reduce=2, 4 or 8 (sqdet_decode_jpeg_params) decodes each file at that fraction of its size, to
  exactly the pixels of cv2.imdecode(files[i], cv2.IMREAD_REDUCED_COLOR_<reduce>): a frame of
  ceil(H / reduce) x ceil(W / reduce) before the orientation, from libjpeg's scaled IDCTs, so a
  12 MP camera file takes a 2.3 MB frame at 1/4 instead of 36 MB.  The size limit then applies to
  the reduced frame, as in cv2; a file of more than 2^30 coded pixels whose reduced frame fits
  still raises ValueError, and cv2.imdecode decodes it.  Any other reduce raises ValueError.

  any_layout=True (sqdet_decode_jpeg_options) decodes, besides those, the colour spaces and
  samplings of every other Huffman-coded 8-bit file cv2.imdecode reads, again to exactly its
  pixels, and combines with progressive and reduce: CMYK and YCCK files (4 components, as
  Photoshop and Pillow write them), RGB-coded files (Adobe transform 0, or ids 'R', 'G', 'B'
  without JFIF) and any sampling with integral ratios and at most 10 blocks per interleaved MCU.
  Files libjpeg rejects (other sampling, 2 or more than 4 components) raise ValueError saying that
  cv2.imdecode does not decode them either."""
  import torch
  kind, params = _decode_call(progressive, reduce, any_layout)
  files = [bytes(f) for f in files]
  n = len(files)
  if not 1 <= n <= 128:
    raise ValueError('need 1 to 128 files, got %d' % n)
  device = torch.device(device)
  if device.type != 'cuda':
    raise ValueError('device must be a CUDA device, got %s' % (device,))
  if device.index is None:
    device = torch.device('cuda', torch.cuda.current_device())
  infos = []
  for i, f in enumerate(files):
    if len(f) < 4:
      raise ValueError('file %d: not a JPEG file (%d bytes)' % (i, len(f)))
    info = jpeg_info(f, progressive, reduce, any_layout)
    if not info['supported']:
      refused = (JPEG_TOO_LARGE, JPEG_BAD_PROGRESSION) + \
          ((JPEG_COMPONENTS, JPEG_BAD_SAMPLING) if any_layout else ())
      raise ValueError('file %d: not supported (%s); %s' % (
          i, info['reason_text'], 'nor does cv2.imdecode decode it'
          if info['reason'] in refused else 'decode it with cv2.imdecode'))
    infos.append(info)
  lib = _lib.load()
  bufs = [C.create_string_buffer(f, len(f)) for f in files]
  ptrs = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
  lens = (C.c_int64 * n)(*[len(f) for f in files])
  pargs = (C.byref(params),) if params else ()
  staging_bytes = getattr(lib, 'sqdet_jpeg_decode_staging_bytes' + kind)(n, ptrs, lens, *pargs)
  scratch_bytes = getattr(lib, 'sqdet_jpeg_decode_scratch_bytes' + kind)(n, ptrs, lens, *pargs)
  if staging_bytes < 0 or scratch_bytes < 0:
    raise _lib.SqdetError(-1, lib.sqdet_last_error().decode('utf-8', 'replace'))
  s = torch_stream(stream, device)
  staging = _staging.setdefault(device.index, _Staging())
  slot, buf = staging.get(staging_bytes)
  with torch.cuda.device(device), torch.cuda.stream(s):
    frames = [torch.empty((info['height'], info['width'], 3), dtype=torch.uint8, device=device)
              for info in infos]
    status = torch.empty((n,), dtype=torch.int32, device=device)
    scratch = torch.empty((scratch_bytes,), dtype=torch.uint8, device=device)
    outs = (C.c_void_p * n)(*[t.data_ptr() for t in frames])
    pitches = (C.c_int64 * n)(*[3 * t.shape[1] for t in frames])
    _lib.check(getattr(lib, 'sqdet_decode_jpeg' + kind)(
        n, ptrs, lens, *pargs, outs, pitches, buf.data_ptr(), buf.numel(), scratch.data_ptr(),
        scratch_bytes, status.data_ptr(), s.cuda_stream))
    staging.events[slot] = torch.cuda.Event()
    staging.events[slot].record(s)
  return frames, status
