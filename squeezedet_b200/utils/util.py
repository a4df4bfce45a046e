"""Host-side utility functions of the reference's ``src/utils/util.py`` that callers
of the hot path use around it (box format conversion, Timer, BGR->RGB).  The
numerically hot ones — ``batch_iou`` / ``nms`` / ``safe_exp`` — run on the GPU
inside ``libsqdet_b200`` (csrc/postproc.cu); they are deliberately NOT re-implemented
on the CPU here (no CPU fallback).  ``nms`` below routes through the GPU filter
kernel so reference-style callers keep working."""
from __future__ import annotations

import time

import numpy as np


def bbox_transform(bbox):
  """[cx, cy, w, h] -> [xmin, ymin, xmax, ymax]; works on scalars or arrays
  (reference util.py:167-179; used by eval.py:91 on the kept boxes)."""
  cx, cy, w, h = bbox
  return [cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2]


def bbox_transform_inv(bbox):
  """[xmin, ymin, xmax, ymax] -> [cx, cy, w, h] with the reference's +1 on width
  and height (util.py:181-196)."""
  xmin, ymin, xmax, ymax = bbox
  width = xmax - xmin + 1.0
  height = ymax - ymin + 1.0
  return [xmin + 0.5 * width, ymin + 0.5 * height, width, height]


def bgr_to_rgb(ims):
  """Convert a list of images from BGR to RGB (util.py:160-165)."""
  return [im[:, :, ::-1] for im in ims]


class Timer(object):
  """tic/toc wall-clock timer with running average (util.py:198-217)."""

  def __init__(self):
    self.total_time = 0.0
    self.calls = 0
    self.start_time = 0.0
    self.duration = 0.0
    self.average_time = 0.0

  def tic(self):
    self.start_time = time.time()

  def toc(self, average=True):
    self.duration = time.time() - self.start_time
    self.total_time += self.duration
    self.calls += 1
    self.average_time = self.total_time / self.calls
    return self.average_time if average else self.duration


def tile_grid(frame_w, frame_h, tile_w, tile_h, min_overlap):
  """Overlapping tiles that cover a frame_w x frame_h frame at native scale, as (x, y, w, h) in
  row-major order, for ModelSkeleton.forward_device_tiles.  Per axis: the fewest tiles whose
  neighbours overlap by at least `min_overlap` pixels, evenly spaced, the first at 0 and the last
  flush with the far edge.  A frame smaller than a tile on an axis gets one tile of the frame's
  size there (the forward then resizes it up).  1920x1080 with 1242x375 tiles and
  min_overlap = 128 gives 2 x 4 tiles."""
  def axis(frame, tile):
    if frame <= tile:
      return [(0, frame)]
    if not 0 <= min_overlap < tile:
      raise ValueError('min_overlap must be in [0, %d), got %r' % (tile, min_overlap))
    span, step = frame - tile, tile - min_overlap
    c = 1 + -(-span // step)
    return [(i * span // (c - 1), tile) for i in range(c)]

  if min(frame_w, frame_h, tile_w, tile_h) < 1:
    raise ValueError('frame and tile sizes must be positive')
  return [(x, y, w, h) for y, h in axis(int(frame_h), int(tile_h))
          for x, w in axis(int(frame_w), int(tile_w))]


def nms(boxes, probs, threshold, device=0):
  """Reference util.nms semantics (util.py:56-76) on the GPU: returns the keep
  mask (list of bool) for centre-format `boxes` ranked by `probs`."""
  import ctypes as C
  from .. import _lib
  boxes = np.ascontiguousarray(np.asarray(boxes, np.float32)).reshape(-1, 4)
  probs = np.ascontiguousarray(np.asarray(probs, np.float32)).reshape(-1)
  n = len(probs)
  if n == 0:
    return []
  if n > 1024:
    raise _lib.SqdetError(-3, 'nms: more than 1024 boxes in one call')
  lib = _lib.load()
  cls = np.zeros(n, np.int64)
  pool = _lib.scratch_pool(device)       # pooled scratch: no cudaMalloc/cudaFree per call
  p_boxes, p_probs, p_cls, p_dets, p_cnt = pool.carve(boxes.nbytes, probs.nbytes, cls.nbytes,
                                                      n * _lib.DET_DTYPE.itemsize, 4)
  pool.upload(p_boxes, boxes)
  pool.upload(p_probs, probs)
  pool.upload(p_cls, cls)
  # top_n = 0 selects the threshold branch; -inf threshold keeps every box as a
  # candidate in original order, so only the NMS rule decides.
  _lib.check(lib.sqdet_topk_nms(p_boxes, p_probs, p_cls, 1, n, 1, 0, C.c_float(-np.inf),
                                C.c_float(threshold), p_dets, p_cnt, n, None))
  dets = pool.download(p_dets, _lib.DET_DTYPE, (n,))
  cnt = int(pool.download(p_cnt, np.int32, (1,))[0])
  keep = [False] * n
  for a in dets['anchor'][:cnt]:
    keep[int(a)] = True
  return keep
