#!/usr/bin/env python
"""What running RGB, RGBA and I420 frames already in device memory costs, two ways.

  python -m squeezedet_b200.bench_device_formats --rounds 5 --steps 20 --warmup 5

The frames are synthesised on the device from a seed.  Four workloads, each a SqueezeDet engine
at b = 20 (1242x375) and one stream:
  chw_kitti    [20, 3, 375, 1242] planar RGB (torch's image layout, what
               torchvision.io.decode_jpeg(device='cuda') returns), whole frames: the resize is a
               copy, so only the conversion is real work;
  chw_1080p    [20, 3, 1080, 1920] planar RGB, whole frames (a real resize);
  rgba_crop    [20, 1080, 1920, 4] RGBA (a capture surface), video_demo's crop
               frame[500:-205, 239:-439];
  i420_crop    [20, 1620, 1920] I420 (Y's rows, then U's and V's bytes), the same crop.
Two forms of a step:
  (a) the fastest conversion a user writes today in torch, then forward_device_frames on BGR
      views: batched flip + permute().contiguous() for CHW; the crop, then flip of the first three
      channels, for RGBA; cv2's I420 -> BGR integer conversion as torch int32 ops into a
      preallocated BGR batch for I420;
  (b) forward_device_frames_fmt on the frames as they are: one launch converts, crops, resizes and
      subtracts the means; no BGR frame is written.
The forms alternate within each round; a round times `steps` steps of one form between two CUDA
events.  The records and counts of (b) are checked bitwise against (a)'s.

The conversion kernel alone is timed in a separate pass under torch.profiler (CUDA activity: the
kernel's device duration, the median over the launches it records).  Its algorithmic bytes,
n*H*W*12 written plus every crop byte read (3 per pixel for planar RGB, 4 for RGBA, 1.5 for I420;
an upper bound for a downscale, which skips source rows), over that time give a rate to set
against the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth.

Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.
"""
from __future__ import annotations

import argparse
import json

import numpy as np

from .bench_device_frames import HBM_BYTES_PER_S, make_model
from .bench_device_u8 import gpu_info

FORMS = ('a_torch_convert_then_forward_frames', 'b_forward_frames_fmt')
KERNEL = 'resize_meansub_u8_batch_kernel'   # form (b)'s only launch of that name
IN_BYTES_PER_PX = {'rgb_planar': 3, 'rgba': 4, 'i420': 1.5}
VIDEO_DEMO_CROP = (239, 500, 1242, 375)     # (x, y, w, h): frame[500:-205, 239:-439]


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--batch', type=int, default=20)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def torch_i420_to_bgr(i420, out, torch):
  """cv2.cvtColor(COLOR_YUV2BGR_I420) of a batch [n, 3H/2, W] into uint8 out [n, H, W, 3], as
  torch int32 ops (oracle.pixfmt.to_bgr's arithmetic)."""
  n, rows, w = i420.shape
  h = 2 * rows // 3
  flat = i420.view(n, -1)
  y = i420[:, :h].to(torch.int32)
  q = (h // 2) * (w // 2)
  u = flat[:, h * w:h * w + q].view(n, h // 2, w // 2).to(torch.int32)
  v = flat[:, h * w + q:].view(n, h // 2, w // 2).to(torch.int32)
  u = u.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2) - 128
  v = v.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2) - 128
  yy = (y - 16).clamp_(min=0) * 1220542 + (1 << 19)
  out[..., 0] = ((yy + 2116026 * u) >> 20).clamp_(0, 255)
  out[..., 1] = ((yy - 852492 * v - 409993 * u) >> 20).clamp_(0, 255)
  out[..., 2] = ((yy + 1673527 * v) >> 20).clamp_(0, 255)


def measure_workload(args, name, model, fmt, batch, crop, torch):
  """batch: the n frames in `fmt` as one uint8 CUDA tensor; crop: (x, y, w, h) or None."""
  from . import _lib
  lib = model._lib
  mc = model.mc
  H, W = mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH
  n = batch.shape[0]
  dev = batch.device
  stream = torch.cuda.Stream(device=dev)
  sptr = stream.cuda_stream
  if fmt == 'rgb_planar':
    fh, fw = batch.shape[2], batch.shape[3]
  elif fmt == 'rgba':
    fh, fw = batch.shape[1], batch.shape[2]
  else:
    fh, fw = 2 * batch.shape[1] // 3, batch.shape[2]
  x, y, cw, ch = crop or (0, 0, fw, fh)
  frames = list(batch)
  crops = [crop] * n
  bgr_i420 = (torch.empty((n, fh, fw, 3), dtype=torch.uint8, device=dev)
              if fmt == 'i420' else None)

  def form_a():
    with torch.cuda.stream(stream):
      if fmt == 'rgb_planar':
        bgr = batch.flip(1).permute(0, 2, 3, 1).contiguous()
      elif fmt == 'rgba':
        bgr = batch[:, y:y + ch, x:x + cw, :3].flip(3)
      else:
        torch_i420_to_bgr(batch, bgr_i420, torch)
        bgr = bgr_i420
    views = [bgr[i] if fmt == 'rgba' else bgr[i, y:y + ch, x:x + cw] for i in range(n)]
    model.forward_device_frames(views, order='demo', stream=sptr)
    return bgr

  def form_b():
    model.forward_device_frames_fmt(frames, fmt, crops=crops, order='demo', stream=sptr)

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
  kernel_bytes = n * H * W * 12 + int(n * cw * ch * IN_BYTES_PER_PX[fmt])

  row = {'workload': name, 'engine': '%dx%d b=%d' % (W, H, mc.BATCH_SIZE), 'n': n,
         'frame': '%dx%d %s' % (fw, fh, fmt), 'crop_xywh': [x, y, cw, ch]}
  for form in FORMS:
    med = float(np.median(ms[form]))
    row[form] = {'ms_per_step_min': min(ms[form]), 'ms_per_step_median': med,
                 'ms_per_step_max': max(ms[form]), 'images_per_s_median': n / (med * 1e-3)}
  row['conversion_kernel'] = {
      'us_median': kernel_us, 'launches_timed': len(durs), 'bytes': kernel_bytes,
      'tb_per_s': kernel_bytes / (kernel_us * 1e-6) / 1e12,
      'share_of_3.35_tb_per_s': kernel_bytes / (kernel_us * 1e-6) / HBM_BYTES_PER_S}
  return row


def measure(args):
  import torch
  from . import _lib
  if _lib.device_count() < 1:
    raise SystemExit('bench_device_formats: no CUDA device visible; the engine has no CPU fallback')
  dev = torch.device('cuda', args.gpu)
  gen = torch.Generator(device=dev)
  gen.manual_seed(7)
  n = args.batch

  def frames(*shape):
    return torch.randint(0, 256, (n,) + shape, dtype=torch.uint8, device=dev, generator=gen)

  model = make_model(1242, 375, n, args.gpu)
  rows = [measure_workload(args, 'chw_kitti', model, 'rgb_planar', frames(3, 375, 1242), None,
                           torch),
          measure_workload(args, 'chw_1080p', model, 'rgb_planar', frames(3, 1080, 1920), None,
                           torch),
          measure_workload(args, 'rgba_crop', model, 'rgba', frames(1080, 1920, 4),
                           VIDEO_DEMO_CROP, torch),
          measure_workload(args, 'i420_crop', model, 'i420', frames(1620, 1920),
                           VIDEO_DEMO_CROP, torch)]
  return {'workload': 'squeezeDet 1242x375, frames in device memory (random bytes), random '
                      '(calibrated) weights, order=demo, no rescale',
          'gpu': gpu_info(args.gpu),
          'timer': 'CUDA events around `steps` steps of one form; conversion kernel: '
                   'torch.profiler device duration, median over the launches it records',
          'bound': 'conversion kernel: algorithmic bytes over time against 3.35 TB/s (HBM3, '
                   'H100 SXM data sheet)',
          'rounds': args.rounds, 'steps': args.steps, 'forms': list(FORMS), 'rows': rows}


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
