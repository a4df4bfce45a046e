#!/usr/bin/env python
"""What running variable-size uint8 BGR frames that already sit in device memory costs, two ways.

  python -m squeezedet_b200.bench_device_frames --rounds 5 --steps 20 --warmup 5

Three workloads, each with one SqueezeDet engine and one stream:
  kitti_mixed     b = 20 at 1242x375; the frames cycle through four KITTI image_2 sizes
                  (1242x375, 1224x370, 1238x374, 1241x376), tightly packed;
  crop_1080p      the same engine; 1920x1080 frames passed as video_demo's crop
                  frame[500:-205, 239:-439], a 375x1242 strided view (a copy, no resampling);
  crop_1080p_1248 SqueezeDet's own 1248x384 config on the same crop views (a real resize).
Two forms of a step:
  (a) today's way: sqdet_preprocess_u8 per frame into an fp32 buffer, then sqdet_forward_n.  It
      needs tightly packed frames, so on the crop workloads each crop is first copied into a tight
      buffer (one torch copy per frame);
  (b) sqdet_forward_frames_u8 on the frames as they are: one resize launch, then the forward.
The forms alternate within each round; a round times `steps` steps of one form between two CUDA
events.  The records and counts of (b) are checked bitwise against (a)'s.

The resize kernel alone is timed in a separate pass under torch.profiler (CUDA activity: the
kernel's device duration, the median over the launches it records), and its algorithmic bytes,
n*H*W*12 written plus the frames' bytes read once, over that time give a rate to set against the
H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth: bytes over time is the bound of this kernel.

Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.
"""
from __future__ import annotations

import argparse
import json

import numpy as np

from .bench_device_u8 import gpu_info

FORMS = ('a_preprocess_then_forward_n', 'b_forward_frames_u8')
KITTI_SIZES = [(375, 1242), (370, 1224), (374, 1238), (376, 1241)]   # (h, w)
HBM_BYTES_PER_S = 3.35e12
KERNEL = 'resize_meansub_u8_batch_kernel'


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--batch', type=int, default=20)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def make_model(width, height, batch, gpu):
  from . import config as cfg, nets
  from .utils import synth
  mc = cfg.kitti_squeezeDet_config()
  mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = width, height, batch
  mc.ANCHOR_BOX = cfg.set_anchors(mc)
  mc.ANCHORS = len(mc.ANCHOR_BOX)
  model = nets.SqueezeDet(mc, gpu)
  model.load_weights(synth.synthetic_weights(synth.model_param_specs(model), seed=0))
  return model


def measure_workload(args, name, model, frames, torch):
  """frames: n uint8 CUDA tensors [h, w, 3] (tight or strided views)."""
  from . import _lib
  lib = model._lib
  mc = model.mc
  H, W, n = mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, len(frames)
  dev = frames[0].device
  stream = torch.cuda.Stream(device=dev)
  sptr = stream.cuda_stream
  means = np.ascontiguousarray(np.asarray(mc.BGR_MEANS, np.float64).reshape(3))
  x_f32 = torch.empty((n, H, W, 3), dtype=torch.float32, device=dev)
  tight = [f if f.is_contiguous() else torch.empty(f.shape, dtype=f.dtype, device=dev)
           for f in frames]
  img_floats = H * W * 3

  def form_a():
    with torch.cuda.stream(stream):
      for f, t in zip(frames, tight):
        if t is not f:
          t.copy_(f)
    for i, t in enumerate(tight):
      _lib.check(lib.sqdet_preprocess_u8(t.data_ptr(), t.shape[0], t.shape[1],
                                         x_f32.data_ptr() + 4 * i * img_floats, H, W,
                                         means.ctypes.data, 0, sptr))
    model.forward_device(x_f32.data_ptr(), sptr, n)

  def form_b():
    model.forward_device_frames(frames, order='demo', stream=sptr)

  res = model.results_device()

  def records():
    dets = np.empty((n, res['max_dets']), _lib.DET_DTYPE)
    counts = np.empty((n,), np.int32)
    stream.synchronize()
    _lib.check(lib.sqdet_memcpy_d2h(dets.ctypes.data, res['dets'], dets.nbytes, None))
    _lib.check(lib.sqdet_memcpy_d2h(counts.ctypes.data, res['counts'], counts.nbytes, None))
    _lib.check(lib.sqdet_stream_sync(args.gpu, None))
    return dets.tobytes() + counts.tobytes()

  steps = {'a_preprocess_then_forward_n': form_a, 'b_forward_frames_u8': form_b}
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

  # the resize kernel alone, in a pass of its own under the profiler
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
  src_bytes = sum(int(f.shape[0]) * int(f.shape[1]) * 3 for f in frames)
  kernel_bytes = n * H * W * 12 + src_bytes

  row = {'workload': name, 'engine': '%dx%d b=%d' % (W, H, mc.BATCH_SIZE), 'n': n,
         'frame_sizes': sorted({'%dx%d' % (int(f.shape[1]), int(f.shape[0])) for f in frames}),
         'strided_views': any(not f.is_contiguous() for f in frames)}
  for form in FORMS:
    med = float(np.median(ms[form]))
    row[form] = {'ms_per_step_min': min(ms[form]), 'ms_per_step_median': med,
                 'ms_per_step_max': max(ms[form]), 'images_per_s_median': n / (med * 1e-3)}
  row['resize_kernel'] = {
      'us_median': kernel_us, 'launches_timed': len(durs), 'bytes': kernel_bytes,
      'tb_per_s': kernel_bytes / (kernel_us * 1e-6) / 1e12,
      'share_of_3.35_tb_per_s': kernel_bytes / (kernel_us * 1e-6) / HBM_BYTES_PER_S}
  return row


def measure(args):
  import torch
  from . import _lib
  if _lib.device_count() < 1:
    raise SystemExit('bench_device_frames: no CUDA device visible; the engine has no CPU fallback')
  dev = torch.device('cuda', args.gpu)
  rng = np.random.default_rng(7)
  B = args.batch
  kitti = [torch.from_numpy(rng.integers(0, 256, KITTI_SIZES[i % 4] + (3,), dtype=np.uint8)).to(dev)
           for i in range(B)]
  full = [torch.from_numpy(rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8)).to(dev)
          for _ in range(B)]
  crops = [f[500:-205, 239:-439] for f in full]
  rows = []
  model = make_model(1242, 375, B, args.gpu)
  rows.append(measure_workload(args, 'kitti_mixed', model, kitti, torch))
  rows.append(measure_workload(args, 'crop_1080p', model, crops, torch))
  model = None
  model = make_model(1248, 384, B, args.gpu)
  rows.append(measure_workload(args, 'crop_1080p_1248', model, crops, torch))
  model = None
  return {'workload': 'squeezeDet, uint8 BGR frames in device memory (random bytes), random '
                      '(calibrated) weights, order=demo, no rescale',
          'gpu': gpu_info(args.gpu),
          'timer': 'CUDA events around `steps` steps of one form; resize kernel: torch.profiler '
                   'device duration, median over the launches it records',
          'bound': 'resize kernel: algorithmic bytes over time against 3.35 TB/s (HBM3, H100 SXM '
                   'data sheet)',
          'rounds': args.rounds, 'steps': args.steps, 'forms': list(FORMS), 'rows': rows}


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
