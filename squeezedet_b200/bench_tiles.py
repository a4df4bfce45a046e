#!/usr/bin/env python
"""What detecting over whole 1080p frames as tiles costs, two ways.

  python -m squeezedet_b200.bench_tiles --rounds 5 --steps 10 --warmup 3

A SqueezeDet engine at 1242x375 runs `frames` 1080p frames (synthesised on the device from a seed)
as a utils.util.tile_grid of 8 tiles each (2 x 4, 128 px overlap), so b = 8 * frames.  Two frame
formats: NV12 (a hardware decoder's output) and packed BGR.  Two forms of a step, each ending with
every frame's merged detections on the host:
  (a) forward_device_frames_fmt over the tiles as crops with rescale=True, then det_boxes,
      det_probs and det_class of the tiles copied back and each frame's union (boxes shifted by
      the tile origin) filtered on the host by oracle.tiles.merge_tiles, the numpy
      filter_prediction: what a user writes without the merge;
  (b) forward_device_tiles, then the merged records and counts copied back.
The forms alternate within each round; a round times `steps` steps of one form with a host clock
(each step ends in a device synchronisation).  Every step's merged results of (b) are checked
bitwise against (a)'s.

The merge kernels alone (tile_top_n_kernel + merge_tiles_kernel) are timed in a separate pass under
torch.profiler: the device duration of each, median over the launches it records.

Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import time

import numpy as np

from .bench_device_frames import make_model
from .bench_device_u8 import gpu_info

FORMS = ('a_forward_frames_then_host_merge', 'b_forward_tiles')
MERGE_KERNELS = ('tile_top_n_kernel', 'merge_tiles_kernel')
FRAME_W, FRAME_H, OVERLAP = 1920, 1080, 128


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--frames', type=int, default=2)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def measure_workload(args, name, model, fmt, frames, grid, torch):
  from oracle import tiles as oracle_tiles
  from . import _lib
  lib, mc = model._lib, model.mc
  n = len(frames)
  tiles = [(f,) + g for f in range(n) for g in grid]
  t = len(tiles)
  A = model.det_probs.shape[1]
  stream = torch.cuda.Stream(device=frames[0].device)
  sptr = stream.cuda_stream
  res = model.results_device()
  boxes = np.empty((t, A, 4), np.float32)
  probs = np.empty((t, A), np.float32)
  cls = np.empty((t, A), np.int64)

  def form_a():
    model.forward_device_frames_fmt([frames[tl[0]] for tl in tiles], fmt,
                                    crops=[tl[1:] for tl in tiles], rescale=True, stream=sptr)
    _lib.check(lib.sqdet_stream_sync(args.gpu, sptr))
    for arr, key in ((boxes, 'det_boxes'), (probs, 'det_probs'), (cls, 'det_class')):
      _lib.check(lib.sqdet_memcpy_d2h(arr.ctypes.data, res[key], arr.nbytes, None))
    _lib.check(lib.sqdet_stream_sync(args.gpu, None))
    out = oracle_tiles.merge_tiles(boxes, probs, cls, tiles, n, mc.CLASSES, mc.TOP_N_DETECTION,
                                   mc.PROB_THRESH, mc.NMS_THRESH)
    return [(np.asarray(fb, np.float32).reshape(-1, 4).tobytes(),
             np.asarray(fp, np.float32).tobytes(), list(fc), list(src))
            for fb, fp, fc, src in out]

  def form_b():
    model.forward_device_tiles(frames, fmt, tiles, stream=sptr)
    dets, counts = model.tile_results(n, stream=sptr)
    out = []
    for f in range(n):
      d = dets[f][:int(counts[f])]
      out.append((np.stack([d['cx'], d['cy'], d['w'], d['h']], -1).tobytes(), d['prob'].tobytes(),
                  d['cls'].tolist(), d['anchor'].tolist()))
    return out

  steps = {FORMS[0]: form_a, FORMS[1]: form_b}
  want = form_a()
  assert any(len(w[3]) for w in want), '%s: no detections to compare' % name
  for form in FORMS:
    for _ in range(args.warmup):
      steps[form]()
  sec = {form: [] for form in FORMS}
  for r in range(args.rounds):
    for form in (FORMS if r % 2 == 0 else FORMS[::-1]):
      t0 = time.perf_counter()
      outs = [steps[form]() for _ in range(args.steps)]
      sec[form].append((time.perf_counter() - t0) / args.steps)
      for got in outs:
        assert got == want, '%s: the merged results of %s differ' % (name, form)

  # the merge kernels alone, in a pass of their own under the profiler
  from torch.autograd import DeviceType
  from torch.profiler import ProfilerActivity, profile
  launches = 20
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(launches):
      model.forward_device_tiles(frames, fmt, tiles, stream=sptr)
    stream.synchronize()
  kern = {}
  for k in MERGE_KERNELS:
    durs = [ev.time_range.elapsed_us() for ev in prof.events()
            if ev.device_type == DeviceType.CUDA and k in ev.name]
    # the profiler may drop an activity record at the edge of its window; the median needs most
    assert len(durs) >= (launches + 1) // 2, 'found %d %s in %d calls' % (len(durs), k, launches)
    kern[k] = {'us_median': float(np.median(durs)), 'launches_timed': len(durs)}

  row = {'workload': name, 'engine': '%dx%d b=%d' % (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT,
                                                     mc.BATCH_SIZE),
         'frames': n, 'tiles': t, 'frame': '%dx%d %s' % (FRAME_W, FRAME_H, fmt),
         'detections_per_frame': [len(w[3]) for w in want]}
  for form in FORMS:
    med = float(np.median(sec[form]))
    row[form] = {'ms_per_step_min': 1e3 * min(sec[form]), 'ms_per_step_median': 1e3 * med,
                 'ms_per_step_max': 1e3 * max(sec[form]), 'frames_per_s_median': n / med,
                 'tiles_per_s_median': t / med}
  row['merge_kernels'] = kern
  return row


def measure(args):
  import torch
  from . import _lib
  from .utils.util import tile_grid
  if _lib.device_count() < 1:
    raise SystemExit('bench_tiles: no CUDA device visible; the engine has no CPU fallback')
  dev = torch.device('cuda', args.gpu)
  gen = torch.Generator(device=dev)
  gen.manual_seed(7)
  grid = tile_grid(FRAME_W, FRAME_H, 1242, 375, OVERLAP)
  assert len(grid) == 8, grid
  n = args.frames
  model = make_model(1242, 375, n * len(grid), args.gpu)

  def frames(*shape):
    return [torch.randint(0, 256, shape, dtype=torch.uint8, device=dev, generator=gen)
            for _ in range(n)]

  rows = [measure_workload(args, 'nv12_1080p', model, 'nv12', frames(FRAME_H * 3 // 2, FRAME_W),
                           grid, torch),
          measure_workload(args, 'bgr_1080p', model, 'bgr', frames(FRAME_H, FRAME_W, 3), grid,
                           torch)]
  return {'workload': 'squeezeDet 1242x375, 1080p frames in device memory (random bytes) as a '
                      'tile_grid of 8 tiles (128 px overlap), random (calibrated) weights, '
                      'order=demo',
          'gpu': gpu_info(args.gpu),
          'timer': 'host clock around `steps` steps of one form, each ending with the merged '
                   'results on the host; merge kernels: torch.profiler device duration, median '
                   'over the launches it records',
          'rounds': args.rounds, 'steps': args.steps, 'forms': list(FORMS), 'rows': rows}


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
