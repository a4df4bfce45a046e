#!/usr/bin/env python
"""What running NV12 frames from a hardware video decoder, already in device memory, costs, two
ways.

  python -m squeezedet_b200.bench_device_nv12 --rounds 5 --steps 20 --warmup 5

The frames are 1920x1080 NV12 (luma plane stacked on the interleaved U,V plane, [1620, 1920]
uint8, the layout decoders hand over), synthesised on the device from a seed.  Three workloads,
each a SqueezeDet engine at b = 20 and one stream:
  crop_1080p       1242x375 engine; video_demo's crop frame[500:-205, 239:-439], 1242x375, so the
                   resize is a copy and only the conversion is real work;
  crop_1080p_1248  SqueezeDet's own 1248x384 config on the same crop (a real resize);
  full_1080p       1242x375 engine on the whole frames.
Two forms of a step:
  (a) what a user writes today: cv2's NV12 -> BGR integer conversion as torch int32 ops on the
      device, into a preallocated uint8 BGR batch [n, 1080, 1920, 3], then forward_device_frames
      on crop views of it;
  (b) forward_device_frames_nv12 on the NV12 frames: one launch converts, crops, resizes and
      subtracts the means; no BGR frame is written.
The forms alternate within each round; a round times `steps` steps of one form between two CUDA
events.  The records and counts of (b) are checked bitwise against (a)'s.

The conversion kernel alone is timed in a separate pass under torch.profiler (CUDA activity: the
kernel's device duration, the median over the launches it records).  Its algorithmic bytes,
n*H*W*12 written plus 1.5 bytes per crop pixel read, over that time give a rate to set against the
H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth.

Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.
"""
from __future__ import annotations

import argparse
import json

import numpy as np

from .bench_device_frames import HBM_BYTES_PER_S, make_model
from .bench_device_u8 import gpu_info

FORMS = ('a_torch_convert_then_forward_frames', 'b_forward_frames_nv12')
KERNEL = 'resize_meansub_u8_batch_kernel'   # form (b)'s only launch of that name
FRAME_H, FRAME_W = 1080, 1920
VIDEO_DEMO_CROP = (239, 500, 1242, 375)     # (x, y, w, h): frame[500:-205, 239:-439]


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--batch', type=int, default=20)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def torch_nv12_to_bgr(nv12, out, torch):
  """cv2.cvtColor(COLOR_YUV2BGR_NV12) of a batch [n, 3H/2, W] into uint8 out [n, H, W, 3], as
  torch int32 ops (oracle.nv12.nv12_to_bgr's arithmetic)."""
  n, rows, w = nv12.shape
  h = 2 * rows // 3
  y = nv12[:, :h].to(torch.int32)
  uv = nv12[:, h:].to(torch.int32).view(n, h // 2, w // 2, 2)
  uv = uv.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2) - 128
  u, v = uv[..., 0], uv[..., 1]
  yy = (y - 16).clamp_(min=0) * 1220542 + (1 << 19)
  out[..., 0] = ((yy + 2116026 * u) >> 20).clamp_(0, 255)
  out[..., 1] = ((yy - 852492 * v - 409993 * u) >> 20).clamp_(0, 255)
  out[..., 2] = ((yy + 1673527 * v) >> 20).clamp_(0, 255)


def measure_workload(args, name, model, nv12, crop, torch):
  """nv12: [n, 3H/2, W] uint8 CUDA tensor; crop: (x, y, w, h) or None (whole frames)."""
  from . import _lib
  lib = model._lib
  mc = model.mc
  H, W = mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH
  n = nv12.shape[0]
  dev = nv12.device
  stream = torch.cuda.Stream(device=dev)
  sptr = stream.cuda_stream
  bgr = torch.empty((n, FRAME_H, FRAME_W, 3), dtype=torch.uint8, device=dev)
  x, y, cw, ch = crop or (0, 0, FRAME_W, FRAME_H)
  views = [bgr[i, y:y + ch, x:x + cw] for i in range(n)]
  frames = [nv12[i] for i in range(n)]
  crops = [crop] * n

  def form_a():
    with torch.cuda.stream(stream):
      torch_nv12_to_bgr(nv12, bgr, torch)
    model.forward_device_frames(views, order='demo', stream=sptr)

  def form_b():
    model.forward_device_frames_nv12(frames, crops=crops, order='demo', stream=sptr)

  res = model.results_device()

  def records():
    dets = np.empty((n, res['max_dets']), _lib.DET_DTYPE)
    counts = np.empty((n,), np.int32)
    stream.synchronize()
    _lib.check(lib.sqdet_memcpy_d2h(dets.ctypes.data, res['dets'], dets.nbytes, None))
    _lib.check(lib.sqdet_memcpy_d2h(counts.ctypes.data, res['counts'], counts.nbytes, None))
    _lib.check(lib.sqdet_stream_sync(args.gpu, None))
    return dets.tobytes() + counts.tobytes()

  steps = {FORMS[0]: form_a, FORMS[1]: form_b}
  want = None
  for form in FORMS:
    for _ in range(args.warmup):
      steps[form]()
    got = records()
    if want is None:
      want = got
    assert got == want, '%s: the records of %s differ from those of (a)' % (name, form)
  ms = {form: [] for form in FORMS}
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for r in range(args.rounds):
    for form in (FORMS if r % 2 == 0 else FORMS[::-1]):
      e0.record(stream)
      for _ in range(args.steps):
        steps[form]()
      e1.record(stream)
      stream.synchronize()
      ms[form].append(e0.elapsed_time(e1) / args.steps)

  # the conversion kernel alone, in a pass of its own under the profiler
  from torch.autograd import DeviceType
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.steps):
      form_b()
    stream.synchronize()
  durs = [ev.time_range.elapsed_us() for ev in prof.events()
          if ev.device_type == DeviceType.CUDA and KERNEL in ev.name]
  # the profiler may drop an activity record at the edge of its window; the median needs most
  assert len(durs) >= (args.steps + 1) // 2, 'found %d %s in %d steps' % (len(durs), KERNEL,
                                                                        args.steps)
  kernel_us = float(np.median(durs))
  kernel_bytes = n * H * W * 12 + int(n * cw * ch * 1.5)

  row = {'workload': name, 'engine': '%dx%d b=%d' % (W, H, mc.BATCH_SIZE), 'n': n,
         'frame': '%dx%d NV12' % (FRAME_W, FRAME_H), 'crop_xywh': [x, y, cw, ch]}
  for form in FORMS:
    med = float(np.median(ms[form]))
    row[form] = {'ms_per_step_min': min(ms[form]), 'ms_per_step_median': med,
                 'ms_per_step_max': max(ms[form]), 'images_per_s_median': n / (med * 1e-3)}
  row['nv12_kernel'] = {
      'us_median': kernel_us, 'launches_timed': len(durs), 'bytes': kernel_bytes,
      'tb_per_s': kernel_bytes / (kernel_us * 1e-6) / 1e12,
      'share_of_3.35_tb_per_s': kernel_bytes / (kernel_us * 1e-6) / HBM_BYTES_PER_S}
  return row


def measure(args):
  import torch
  from . import _lib
  if _lib.device_count() < 1:
    raise SystemExit('bench_device_nv12: no CUDA device visible; the engine has no CPU fallback')
  dev = torch.device('cuda', args.gpu)
  gen = torch.Generator(device=dev)
  gen.manual_seed(7)
  nv12 = torch.randint(0, 256, (args.batch, FRAME_H * 3 // 2, FRAME_W), dtype=torch.uint8,
                       device=dev, generator=gen)
  rows = []
  model = make_model(1242, 375, args.batch, args.gpu)
  rows.append(measure_workload(args, 'crop_1080p', model, nv12, VIDEO_DEMO_CROP, torch))
  rows.append(measure_workload(args, 'full_1080p', model, nv12, None, torch))
  model = None
  model = make_model(1248, 384, args.batch, args.gpu)
  rows.append(measure_workload(args, 'crop_1080p_1248', model, nv12, VIDEO_DEMO_CROP, torch))
  model = None
  return {'workload': 'squeezeDet, 1920x1080 NV12 frames in device memory (random bytes), random '
                      '(calibrated) weights, order=demo, no rescale',
          'gpu': gpu_info(args.gpu),
          'timer': 'CUDA events around `steps` steps of one form; NV12 kernel: torch.profiler '
                   'device duration, median over the launches it records',
          'bound': 'NV12 kernel: algorithmic bytes over time against 3.35 TB/s (HBM3, H100 SXM '
                   'data sheet)',
          'rounds': args.rounds, 'steps': args.steps, 'forms': list(FORMS), 'rows': rows}


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
