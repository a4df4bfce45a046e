#!/usr/bin/env python
"""Images/s of the eval.py frames path, and what a short last group costs.

  python -m squeezedet_b200.bench_frames --steps 30 --warmup 5

uint8 1242x375 BGR frames in pinned host memory go through
sqdet_submit_frames_n(order=eval, rescale=1), two submits in flight; the timer is the host wall
clock around K submits and the final wait.  Rows: an engine of batch 1, one of batch 20 at n = 20,
and the batch-20 engine at n = 1 and n = 7, which run the kernels planned for 20 images on
smaller grids.  Prints one JSON line; writes nothing.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import time

import numpy as np


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--width', type=int, default=1242)
  ap.add_argument('--height', type=int, default=375)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def measure(args):
  from . import _lib, config as cfg, nets
  from .utils import synth
  if _lib.device_count() < 1:
    raise SystemExit('bench_frames: no CUDA device visible; the engine has no CPU fallback')
  H, W, nmax = args.height, args.width, 20
  frames = _lib.PinnedArray((nmax, H, W, 3), np.uint8)
  frames.array[...] = np.random.default_rng(7).integers(0, 256, frames.array.shape, dtype=np.uint8)
  ptrs = (C.c_void_p * nmax)(*[frames.ptr + i * H * W * 3 for i in range(nmax)])
  hs = (C.c_int32 * nmax)(*([H] * nmax))
  ws = (C.c_int32 * nmax)(*([W] * nmax))
  lib = _lib.load()
  rows = []
  for batch, ns in ((1, (1,)), (20, (20, 1, 7))):
    mc = cfg.kitti_squeezeDet_config()
    mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = W, H, batch
    mc.ANCHOR_BOX = cfg.set_anchors(mc)
    mc.ANCHORS = len(mc.ANCHOR_BOX)
    model = nets.SqueezeDet(mc, args.gpu)
    model.load_weights(synth.synthetic_weights(synth.model_param_specs(model), seed=0))
    # pinned result slots, one per submit in flight, so the copies back stay asynchronous
    dets = [_lib.PinnedArray((batch, model.max_dets), _lib.DET_DTYPE) for _ in range(2)]
    counts = [_lib.PinnedArray((batch,), np.int32) for _ in range(2)]

    def run(n, k):
      for i in range(k):
        _lib.check(lib.sqdet_submit_frames_n(model._engine, n, ptrs, hs, ws, 1, 1,
                                             dets[i & 1].ptr, counts[i & 1].ptr))
        if i >= 1:
          _lib.check(lib.sqdet_wait(model._engine))
      _lib.check(lib.sqdet_wait(model._engine))

    for n in ns:
      run(n, max(args.warmup, 3))
      t0 = time.perf_counter()
      run(n, args.steps)
      ms = 1e3 * (time.perf_counter() - t0) / args.steps
      rows.append({'engine_batch': batch, 'n': n, 'ms_per_step': ms, 'value': n / (ms * 1e-3)})
    for buf in dets + counts:
      buf.free()
    model = None
  frames.free()
  return {'workload': 'squeezeDet, uint8 %dx%d BGR frames in pinned host memory, '
                      'sqdet_submit_frames_n(order=eval, rescale=1), 2 in flight' % (W, H),
          'unit': 'images/sec', 'timer': 'host wall clock around K submits + final wait',
          'steps': args.steps, 'rows': rows}


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
