#!/usr/bin/env python
"""What writing annotated 1080p frames as JPEG files costs, two ways.

  python -m squeezedet_b200.bench_jpeg --rounds 5 --steps 10 --warmup 3

A SqueezeDet engine at 1242x375 runs `frames` 1080p frames (smooth synthetic pictures made on the
device from a seed: upsampled noise plus a little grain) as a utils.util.tile_grid of 8 tiles each,
and draw_detections_device draws the merged records on them, as bench_draw does.  Two frame
formats: packed BGR and NV12.  Each step then ends one of two ways:
  (a) every frame copied to the host, cv2.cvtColor'd to BGR (NV12), and cv2.imencode('.jpg'):
      what demo.py did before the encoder;
  (b) encode_jpeg_device on the same stream, then jpeg_bytes copies back only each file's bytes.
The forms alternate within each round.  A step's time is split at a device synchronisation after
the draw: `ending` is the encode and copy alone, `step` the whole step (a fresh copy of the frames,
forward, draw, ending).  Every step's files of (b) are checked bitwise against (a)'s.

The encode kernels alone are timed in a separate pass under torch.profiler: the device durations of
the encode_jpeg_device calls' kernels and memsets, summed, per frame.

Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import time

import numpy as np

from .bench_device_frames import make_model
from .bench_device_u8 import gpu_info

FRAME_W, FRAME_H, OVERLAP = 1920, 1080, 128
QUALITY = 95
SAMPLING_FACTORS = {'411': 0x411111, '420': 0x221111, '422': 0x211111, '440': 0x121111, '444': 0x111111}
KERNELS = ('transform_kernel', 'hist_kernel', 'table_kernel', 'interval_kernel', 'block_bits_kernel', 'scan_kernel', 'pack_kernel',
           'count_ff_kernel', 'stuff_kernel', 'prog_units_kernel', 'prog_eobrun_kernel', 'prog_table_kernel',
           'prog_bits_kernel', 'prog_interval_kernel', 'prog_pack_kernel')


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--frames', type=int, default=2)
  ap.add_argument('--gpu', type=int, default=0)
  # cv2's other JPEG parameters, passed alike to both forms; the defaults are cv2's
  ap.add_argument('--sampling', default='420', choices=('411', '420', '422', '440', '444'))
  ap.add_argument('--optimize', action='store_true')
  ap.add_argument('--restart', type=int, default=0, help='restart interval in MCUs (0: none)')
  ap.add_argument('--progressive', action='store_true', help='IMWRITE_JPEG_PROGRESSIVE')
  return ap.parse_args(argv)


def jpeg_settings(args):
  """encode_jpeg_device's keywords of the command line."""
  return dict(quality=QUALITY, sampling=args.sampling, optimize=args.optimize,
              restart_interval=args.restart, progressive=args.progressive)


@dataclasses.dataclass
class Encoder:
  """What the benchmarks of the file encoders (this one, bench_png) differ in."""
  name: str                 # 'jpeg': form (b) is encode_<name>_device, the benchmark bench_<name>
  ext: str                  # cv2.imencode's extension
  cv2_params: list          # cv2.imencode's parameters, the same settings as encode's
  encode: object            # (frames, fmt, stream) -> (data, lengths) on the device
  files: object             # (data, lengths, stream) -> the files as bytes objects
  kernels: tuple            # the encode's kernels, as the profiler names them
  launches: int             # the encode's launches and memsets per 16 frames
  what: str                 # the files, as the workload names them
  row: dict                 # the encoder's settings, as each row gives them
  by_kernel: bool = False   # also give each kernel's device time

  @property
  def forms(self):
    return ('a_host_imencode', 'b_encode_%s_device' % self.name)


def jpeg_encoder(args):
  import cv2
  from .jpeg import encode_jpeg_device, jpeg_bytes
  settings = jpeg_settings(args)
  cv2_params = [cv2.IMWRITE_JPEG_QUALITY, QUALITY,
                cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING_FACTORS[args.sampling]]
  if args.optimize:
    cv2_params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
  if args.restart:
    cv2_params += [cv2.IMWRITE_JPEG_RST_INTERVAL, args.restart]
  if args.progressive:
    cv2_params += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
  # per 16 frames: a memset and seven launches, two more with optimize and two with restart
  # markers; progressive files take a memset and fourteen launches whatever the other settings
  launches = 15 if args.progressive else 8 + 2 * args.optimize + 2 * bool(args.restart)
  return Encoder('jpeg', '.jpg', cv2_params,
                 lambda frames, fmt, stream: encode_jpeg_device(frames, fmt, stream=stream, **settings),
                 jpeg_bytes, KERNELS, launches,
                 'JPEG quality %d%s files' % (QUALITY, ' progressive' if args.progressive else ''),
                 {'quality': QUALITY, 'sampling': args.sampling, 'optimize': args.optimize,
                  'restart': args.restart, 'progressive': args.progressive})


def measure_workload(enc, args, name, model, fmt, clean, grid, torch):
  import cv2
  forms = enc.forms
  mc = model.mc
  n = len(clean)
  tiles = [(f,) + g for f in range(n) for g in grid]
  stream = torch.cuda.Stream(device=clean[0].device)
  sptr = stream.cuda_stream
  work = [torch.empty_like(c) for c in clean]

  def drawn():
    with torch.cuda.stream(stream):
      for w, c in zip(work, clean):
        w.copy_(c)
    model.forward_device_tiles(work, fmt, tiles, stream=sptr)
    model.draw_detections_device(work, fmt, which='tiles', stream=sptr)
    stream.synchronize()

  def end_a():
    files = []
    with torch.cuda.stream(stream):
      for w in work:
        im = w.cpu().numpy()
        if fmt == 'nv12':
          im = cv2.cvtColor(im, cv2.COLOR_YUV2BGR_NV12)
        files.append(cv2.imencode(enc.ext, im, enc.cv2_params)[1].tobytes())
    return files

  def end_b():
    with torch.cuda.stream(stream):
      data, lengths = enc.encode(work, fmt, stream)
      return enc.files(data, lengths, stream=stream)

  ends = {forms[0]: end_a, forms[1]: end_b}
  drawn()
  want = end_a()
  assert end_b() == want, '%s: the files differ' % name
  for form in forms:
    for _ in range(args.warmup):
      drawn()
      ends[form]()
  step = {form: [] for form in forms}
  ending = {form: [] for form in forms}
  for r in range(args.rounds):
    for form in (forms if r % 2 == 0 else forms[::-1]):
      for _ in range(args.steps):
        t0 = time.perf_counter()
        drawn()
        t1 = time.perf_counter()
        got = ends[form]()
        t2 = time.perf_counter()
        step[form].append(t2 - t0)
        ending[form].append(t2 - t1)
        assert got == want, '%s: the files of %s differ' % (name, form)

  # the encode kernels alone, in a pass of their own under the profiler
  from torch.autograd import DeviceType
  from torch.profiler import ProfilerActivity, profile
  drawn()
  calls = 20
  outs = []
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(calls):
      outs.append(enc.encode(work, fmt, stream))
    stream.synchronize()
  names = enc.kernels + ('emset',)
  evs = [ev for ev in prof.events() if ev.device_type == DeviceType.CUDA and
         any(k in ev.name for k in names)]
  launches = calls * -(-n // 16) * enc.launches
  assert len(evs) >= launches * 9 // 10, 'found %d of %d encode launches' % (len(evs), launches)
  us = sum(ev.time_range.elapsed_us() for ev in evs) / calls

  row = {'workload': name, 'engine': '%dx%d b=%d' % (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT,
                                                     mc.BATCH_SIZE),
         'frames': n, 'frame': '%dx%d %s' % (FRAME_W, FRAME_H, fmt), **enc.row,
         'file_bytes_mean': float(np.mean([len(f) for f in want]))}
  for form in forms:
    row[form] = {'ms_per_frame_ending_median': 1e3 * float(np.median(ending[form])) / n,
                 'ms_per_frame_ending_min': 1e3 * min(ending[form]) / n,
                 'ms_per_frame_step_median': 1e3 * float(np.median(step[form])) / n}
  row['encode_kernels'] = {'us_per_frame_mean': us / n, 'calls_timed': calls}
  if enc.by_kernel:
    row['encode_kernels']['us_per_frame_by_kernel'] = {
        k: sum(ev.time_range.elapsed_us() for ev in evs if k in ev.name) / calls / n for k in names}
  return row


def measure(args, enc):
  import torch
  import torch.nn.functional as F
  from . import _lib
  from .utils.util import tile_grid
  if _lib.device_count() < 1:
    raise SystemExit('bench_%s: no CUDA device visible; the engine has no CPU fallback' % enc.name)
  dev = torch.device('cuda', args.gpu)
  gen = torch.Generator(device=dev)
  gen.manual_seed(7)
  grid = tile_grid(FRAME_W, FRAME_H, 1242, 375, OVERLAP)
  assert len(grid) == 8, grid
  n = args.frames
  model = make_model(1242, 375, n * len(grid), args.gpu)

  def picture(h, w, c):
    """A smooth uint8 [h, w, c] picture: bilinear upsampled noise plus grain."""
    low = torch.rand((1, c, h // 24, w // 24), device=dev, generator=gen) * 255
    up = F.interpolate(low, size=(h, w), mode='bilinear', align_corners=False)[0]
    grain = torch.randn((c, h, w), device=dev, generator=gen) * 4
    return (up + grain).clamp(0, 255).to(torch.uint8).permute(1, 2, 0).contiguous()

  rows = [measure_workload(enc, args, 'bgr_1080p', model, 'bgr',
                           [picture(FRAME_H, FRAME_W, 3) for _ in range(n)], grid, torch),
          measure_workload(enc, args, 'nv12_1080p', model, 'nv12',
                           [picture(FRAME_H * 3 // 2, FRAME_W, 1)[..., 0] for _ in range(n)],
                           grid, torch)]
  return {'workload': 'squeezeDet 1242x375, 1080p frames in device memory (smooth synthetic '
                      'pictures) as a tile_grid of 8 tiles (128 px overlap), detections drawn, '
                      'then %s on the host' % enc.what,
          'gpu': gpu_info(args.gpu),
          'timer': 'host clock per step, split at a device synchronisation after the draw; '
                   'encode kernels: torch.profiler device durations of the calls, summed, per frame',
          'rounds': args.rounds, 'steps': args.steps,
          'forms': list(enc.forms), 'rows': rows}


def main(argv=None):
  args = parse_args(argv)
  print(json.dumps(measure(args, jpeg_encoder(args))))


if __name__ == '__main__':
  main()
