"""PNG files of uint8 frames in device memory (sqdet_encode_png), byte for byte what cv2.imwrite /
cv2.imencode('.png', ...) writes for the same BGR image, with no frame copied to the host.

  data, lengths = encode_png_device(frames, 'nv12')
  files = png_bytes(data, lengths)         # one bytes object per frame

Frames are taken as encode_jpeg_device takes them; crop i is written as cv2.imencode writes
cv2.cvtColor(frame_i, code)[y:y+h, x:x+w].  Only cv2's default PNG parameters are reproduced:
route IMWRITE_PNG_COMPRESSION, _STRATEGY or filter choices, alpha, grayscale and 16-bit output to
cv2.  No engine is needed."""
from __future__ import annotations

from . import _lib
from .frames import encode_frames, file_bytes

MAX_SIDE = 1000000        # libpng's PNG_USER_WIDTH_MAX / PNG_USER_HEIGHT_MAX

# the files of encode_png_device's (data, lengths): the same per-file copy-back as JPEG's
png_bytes = file_bytes


def max_bytes(h, w):
  """The largest PNG file of an h x w image (sqdet_png_max_bytes).  Sides are at most 1000000,
  libpng's user limits, as for cv2.imencode."""
  if not (1 <= int(h) <= MAX_SIDE and 1 <= int(w) <= MAX_SIDE):
    raise ValueError('a PNG is 1 to %d pixels wide and high, got %dx%d' % (MAX_SIDE, w, h))
  return int(_lib.load().sqdet_png_max_bytes(int(h), int(w)))


def encode_png_device(frames, fmt, crops=None, stream=None):
  """-> (data [n, cap] uint8, lengths [n] int64), both on the frames' device: frame i's file is
  data[i, :lengths[i]], and lengths[i] is -1 if it did not fit cap = the largest file of the
  largest crop.  Asynchronous on `stream` (a torch.cuda.Stream, a raw cudaStream_t, or None for
  torch's current stream): run it on the stream that wrote the frames, and read the results on it
  (png_bytes with the same `stream`) or after synchronising it.  The outputs and the scratch are
  allocated on that stream.

  Every size is a worst case, so that nothing waits for the device: cap is what the crop would
  take if every filtered byte cost 9 bits (sqdet_png_max_bytes, about 7 MB for 1920 x 1080), and
  the scratch is about 26 MB per 1080p frame of each group of 16.  Sides above 1000000 raise
  ValueError before anything is allocated; cv2.imencode refuses them too."""
  return encode_frames(frames, fmt, crops, stream, max_bytes, 'sqdet_png_scratch_bytes',
                       'sqdet_encode_png')
