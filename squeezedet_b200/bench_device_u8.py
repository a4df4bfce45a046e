#!/usr/bin/env python
"""What feeding uint8 BGR batches that already sit in device memory costs, three ways.

  python -m squeezedet_b200.bench_device_u8 --rounds 5 --steps 20 --warmup 5

For SqueezeDet b = 20, SqueezeDet+ b = 20, ResNet50+ConvDet b = 8 and VGG16+ConvDet b = 8 at
1242x375, one engine each, three forms of a step on one stream:
  (a) sqdet_forward_n on fp32 images converted beforehand (the bench.py `value` path);
  (b) sqdet_forward_u8 on the uint8 batch (the first layer reads the bytes, or, for VGG16, one
      launch converts them into the engine's input tensor);
  (c) sqdet_preprocess_u8 per image into an fp32 buffer, then sqdet_forward_n.
The forms alternate within each round; a round times `steps` forwards of one form between two
CUDA events.  (b)'s and (c)'s records and counts are checked bitwise against (a)'s.  Prints one
JSON line with the card's name and power limit, read in the same run; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import subprocess

import numpy as np

WORKLOADS = [('squeezeDet', 20), ('squeezeDet+', 20), ('resnet50', 8), ('vgg16', 8)]
NETS = {'squeezeDet': ('SqueezeDet', 'kitti_squeezeDet_config'),
        'squeezeDet+': ('SqueezeDetPlus', 'kitti_squeezeDetPlus_config'),
        'resnet50': ('ResNet50ConvDet', 'kitti_res50_config'),
        'vgg16': ('VGG16ConvDet', 'kitti_vgg16_config')}
FORMS = ('a_forward_n_f32', 'b_forward_u8', 'c_preprocess_then_forward_n')


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--width', type=int, default=1242)
  ap.add_argument('--height', type=int, default=375)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def gpu_info(index):
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader', '-i', str(index)],
                       capture_output=True, text=True, check=True).stdout.strip()
  name, power, clock = [s.strip() for s in out.split(',')]
  return {'name': name, 'power_limit': power, 'max_sm_clock': clock}


def measure_net(args, net, batch, torch):
  from . import _lib, config as cfg, nets
  from .utils import synth
  lib = _lib.load()
  H, W = args.height, args.width
  mc = getattr(cfg, NETS[net][1])()
  mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = W, H, batch
  mc.ANCHOR_BOX = cfg.set_anchors(mc)
  mc.ANCHORS = len(mc.ANCHOR_BOX)
  model = getattr(nets, NETS[net][0])(mc, args.gpu)
  model.load_weights(synth.synthetic_weights(synth.model_param_specs(model), seed=0))
  dev = torch.device('cuda', args.gpu)
  stream = torch.cuda.Stream(device=dev)
  sptr = stream.cuda_stream
  u8_host = np.random.default_rng(7).integers(0, 256, (batch, H, W, 3), dtype=np.uint8)
  means = np.ascontiguousarray(np.asarray(mc.BGR_MEANS, np.float64).reshape(3))
  f32_host = (u8_host.astype(np.float64) - means).astype(np.float32)
  x_u8 = torch.from_numpy(u8_host).to(dev)
  x_f32 = torch.from_numpy(f32_host).to(dev)
  x_tmp = torch.empty_like(x_f32)
  img_bytes, img_floats = H * W * 3, H * W * 3

  def form_a():
    model.forward_device(x_f32.data_ptr(), sptr)

  def form_b():
    model.forward_device_u8(x_u8.data_ptr(), sptr)

  def form_c():
    for i in range(batch):
      _lib.check(lib.sqdet_preprocess_u8(x_u8.data_ptr() + i * img_bytes, H, W,
                                         x_tmp.data_ptr() + 4 * i * img_floats, H, W,
                                         means.ctypes.data, 0, sptr))
    model.forward_device(x_tmp.data_ptr(), sptr)

  res = model.results_device()

  def records():
    dets = np.empty((batch, res['max_dets']), _lib.DET_DTYPE)
    counts = np.empty((batch,), np.int32)
    stream.synchronize()
    _lib.check(lib.sqdet_memcpy_d2h(dets.ctypes.data, res['dets'], dets.nbytes, None))
    _lib.check(lib.sqdet_memcpy_d2h(counts.ctypes.data, res['counts'], counts.nbytes, None))
    _lib.check(lib.sqdet_stream_sync(args.gpu, None))
    return dets.tobytes() + counts.tobytes()

  steps = {'a_forward_n_f32': form_a, 'b_forward_u8': form_b,
           'c_preprocess_then_forward_n': form_c}
  want = None
  for name in FORMS:
    for _ in range(args.warmup):
      steps[name]()
    got = records()
    if want is None:
      want = got
    assert got == want, '%s: the records of %s differ from those of sqdet_forward_n' % (net, name)
  ms = {name: [] for name in FORMS}
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for r in range(args.rounds):
    order = FORMS if r % 2 == 0 else FORMS[::-1]
    for name in order:
      e0.record(stream)
      for _ in range(args.steps):
        steps[name]()
      e1.record(stream)
      stream.synchronize()
      ms[name].append(e0.elapsed_time(e1) / args.steps)
  row = {'net': net, 'batch': batch, 'fused_first_layer': net != 'vgg16'}
  for name in FORMS:
    row[name] = {'ms_per_step_min': min(ms[name]), 'ms_per_step_median': float(np.median(ms[name])),
                 'ms_per_step_max': max(ms[name]),
                 'images_per_s_median': batch / (float(np.median(ms[name])) * 1e-3)}
  model = None
  return row


def measure(args):
  import torch
  from . import _lib
  if _lib.device_count() < 1:
    raise SystemExit('bench_device_u8: no CUDA device visible; the engine has no CPU fallback')
  rows = [measure_net(args, net, batch, torch) for net, batch in WORKLOADS]
  return {'workload': 'uint8 %dx%d BGR batches in device memory (random bytes), random '
                      '(calibrated) weights' % (args.width, args.height),
          'gpu': gpu_info(args.gpu), 'timer': 'CUDA events around `steps` forwards of one form',
          'rounds': args.rounds, 'steps': args.steps, 'forms': list(FORMS), 'rows': rows}


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
