#!/usr/bin/env python
"""What drawing the detections onto 1080p frames in device memory costs, two ways.

  python -m squeezedet_b200.bench_draw --rounds 5 --steps 10 --warmup 3

A SqueezeDet engine at 1242x375 runs `frames` 1080p frames (synthesised on the device from a seed)
as a utils.util.tile_grid of 8 tiles each (2 x 4, 128 px overlap), so b = 8 * frames, as
bench_tiles does.  Two frame formats: packed BGR and NV12.  A step starts from fresh copies of the
frames on the device and ends with the annotated frames on the device:
  (a) forward_device_tiles, then the merged records and every frame copied to the host, drawn there
      (BGR: demo.draw_detections, i.e. cv2 through utils.viz.draw_box; NV12, which cv2 cannot draw
      on: oracle.draw's numpy rule) and copied back: what a user writes without the kernel;
  (b) forward_device_tiles, then draw_detections_device on the same stream.
The forms alternate within each round; a round times `steps` steps of one form with a host clock
(each step ends in a device synchronisation).  Every step's annotated frames of (b) are checked
bitwise against (a)'s.

The draw kernel alone (draw_dets_kernel) is timed in a separate pass under torch.profiler: its device
duration, median over the launches it records.

Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import time

import numpy as np

from .bench_device_frames import make_model
from .bench_device_u8 import gpu_info

FORMS = ('a_host_draw', 'b_draw_detections_device')
FRAME_W, FRAME_H, OVERLAP = 1920, 1080, 128


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--frames', type=int, default=2)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def host_draw(mc, model, fmt, im, dets, count):
  """Form (a)'s drawing of one frame on the host, in place."""
  from oracle import draw
  from .demo import draw_detections
  from .utils.viz import CLASS_COLORS
  if fmt == 'bgr':
    draw_detections(mc, im, *model.records_to_lists(dets, count))
    return
  colours = np.array([CLASS_COLORS.get(n, (0, 255, 0)) for n in mc.CLASS_NAMES], np.uint8)
  H = FRAME_H
  draw.draw_yuv420(im[:H], im[H:, 0::2], im[H:, 1::2], (0, 0, FRAME_W, H), dets, count,
                   list(mc.CLASS_NAMES), colours, mc.PLOT_PROB_THRESH, 0.3)


def measure_workload(args, name, model, fmt, clean, grid, torch):
  mc = model.mc
  n = len(clean)
  tiles = [(f,) + g for f in range(n) for g in grid]
  stream = torch.cuda.Stream(device=clean[0].device)
  sptr = stream.cuda_stream
  work = [torch.empty_like(c) for c in clean]

  def fresh():
    with torch.cuda.stream(stream):
      for w, c in zip(work, clean):
        w.copy_(c)

  def form_a():
    fresh()
    model.forward_device_tiles(work, fmt, tiles, stream=sptr)
    dets, counts = model.tile_results(n, stream=sptr)
    with torch.cuda.stream(stream):
      for f in range(n):
        im = work[f].cpu().numpy()
        host_draw(mc, model, fmt, im, dets[f], int(counts[f]))
        work[f].copy_(torch.from_numpy(im))
    stream.synchronize()
    return [w.clone() for w in work], int(counts.sum())

  def form_b():
    fresh()
    model.forward_device_tiles(work, fmt, tiles, stream=sptr)
    model.draw_detections_device(work, fmt, which='tiles', stream=sptr)
    stream.synchronize()
    return [w.clone() for w in work], None

  steps = {FORMS[0]: form_a, FORMS[1]: form_b}
  want, kept = form_a()
  assert kept > 0, '%s: no detections to draw' % name
  assert any(not torch.equal(w, c) for w, c in zip(want, clean)), '%s: nothing drawn' % name
  for form in FORMS:
    for _ in range(args.warmup):
      steps[form]()
  sec = {form: [] for form in FORMS}
  for r in range(args.rounds):
    for form in (FORMS if r % 2 == 0 else FORMS[::-1]):
      t0 = time.perf_counter()
      outs = [steps[form]()[0] for _ in range(args.steps)]
      sec[form].append((time.perf_counter() - t0) / args.steps)
      for got in outs:
        assert all(torch.equal(g, w) for g, w in zip(got, want)), \
            '%s: the frames of %s differ' % (name, form)

  # the draw kernel alone, in a pass of its own under the profiler
  from torch.autograd import DeviceType
  from torch.profiler import ProfilerActivity, profile
  fresh()
  model.forward_device_tiles(work, fmt, tiles, stream=sptr)
  launches = 20
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(launches):
      model.draw_detections_device(work, fmt, which='tiles', stream=sptr)
    stream.synchronize()
  durs = [ev.time_range.elapsed_us() for ev in prof.events()
          if ev.device_type == DeviceType.CUDA and 'draw_dets_kernel' in ev.name]
  # the profiler may drop an activity record at the edge of its window; the median needs most
  assert len(durs) >= (launches + 1) // 2, 'found %d draw launches in %d calls' % (len(durs), launches)

  row = {'workload': name, 'engine': '%dx%d b=%d' % (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT,
                                                     mc.BATCH_SIZE),
         'frames': n, 'tiles': len(tiles), 'frame': '%dx%d %s' % (FRAME_W, FRAME_H, fmt),
         'records_drawn_per_step': kept}
  for form in FORMS:
    med = float(np.median(sec[form]))
    row[form] = {'ms_per_step_min': 1e3 * min(sec[form]), 'ms_per_step_median': 1e3 * med,
                 'ms_per_step_max': 1e3 * max(sec[form]), 'frames_per_s_median': n / med}
  row['draw_kernel'] = {'us_median': float(np.median(durs)), 'launches_timed': len(durs)}
  return row


def measure(args):
  import torch
  from . import _lib
  from .utils.util import tile_grid
  if _lib.device_count() < 1:
    raise SystemExit('bench_draw: no CUDA device visible; the engine has no CPU fallback')
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

  rows = [measure_workload(args, 'bgr_1080p', model, 'bgr', frames(FRAME_H, FRAME_W, 3), grid,
                           torch),
          measure_workload(args, 'nv12_1080p', model, 'nv12', frames(FRAME_H * 3 // 2, FRAME_W),
                           grid, torch)]
  return {'workload': 'squeezeDet 1242x375, 1080p frames in device memory (random bytes) as a '
                      'tile_grid of 8 tiles (128 px overlap), random (calibrated) weights, '
                      'order=demo, PLOT_PROB_THRESH %g' % model.mc.PLOT_PROB_THRESH,
          'gpu': gpu_info(args.gpu),
          'timer': 'host clock around `steps` steps of one form, each ending with the annotated '
                   'frames on the device; draw kernel: torch.profiler device duration, median '
                   'over the launches it records',
          'rounds': args.rounds, 'steps': args.steps, 'forms': list(FORMS), 'rows': rows}


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
