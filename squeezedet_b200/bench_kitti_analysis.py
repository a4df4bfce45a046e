#!/usr/bin/env python
"""What the detection error analysis of a val-sized KITTI set costs, on the GPU and as the
reference computes it.

  python -m squeezedet_b200.bench_kitti_analysis --steps 20 --warmup 3

The seeded synthetic set of bench_kitti_eval (3769 images, 64 filtered records each), with label
corners the reference's analysis accepts.  kitti.analyze_device on records already in device
memory is timed with CUDA events per call after warm-up: the three kernels, their memsets and the
copies back of the counts and the error lines.  The host formatting of the block and of
det_error_file.txt (kitti.analysis_text, kitti.error_file_text) is timed separately with a host
clock.  oracle/kitti_analysis.analyze, which reads the label and detection files back and loops in
Python as the reference's analyze_detections does, is timed with a host clock on the files
eval.py's writer makes from the same records, and both error files are compared byte for byte.
Everything is written under a temporary directory.

Prints one JSON line with the card's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

from .bench_device_u8 import gpu_info
from .bench_kitti_eval import synthetic_set


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--images', type=int, default=3769)
  ap.add_argument('--dets', type=int, default=64)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--oracle_runs', type=int, default=2)
  ap.add_argument('--seed', type=int, default=2024)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def _stats(xs):
  return {'median': float(np.median(xs)), 'min': float(np.min(xs)), 'max': float(np.max(xs))}


def measure(args):
  import torch
  from . import kitti
  from .eval import detections_to_all_boxes
  from .utils.viz import write_kitti_detections
  sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
  from oracle import kitti_analysis
  names = ('car', 'pedestrian', 'cyclist')
  dev = torch.device('cuda', args.gpu)
  labels, records = synthetic_set(args.seed, args.images, args.dets, analyzable=True)
  dets = np.stack(records)
  counts = np.full((args.images,), args.dets, np.int32)
  res = {'gpu': gpu_info(args.gpu), 'images': args.images, 'records_per_image': args.dets}
  with tempfile.TemporaryDirectory() as tmp:
    ids = ['%06d' % i for i in range(args.images)]
    lab_dir = os.path.join(tmp, 'training', 'label_2')
    os.makedirs(lab_dir)
    for i, text in zip(ids, labels):
      with open(os.path.join(lab_dir, i + '.txt'), 'w') as f:
        f.write(text)
    lab = kitti.read_labels(lab_dir, ids)
    res['objects'] = len(lab.objs)
    d = torch.from_numpy(dets.view(np.uint8).reshape(args.images, -1)).to(dev)
    c = torch.from_numpy(counts).to(dev)
    for _ in range(args.warmup):
      stats, lines = kitti.analyze_device(d, c, names, lab)
    times = []
    for _ in range(args.steps):
      t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      t0.record()
      stats, lines = kitti.analyze_device(d, c, names, lab)
      t1.record()
      t1.synchronize()
      times.append(t0.elapsed_time(t1))
    res['device_ms'] = _stats(times)
    ft = []
    for _ in range(max(1, args.steps // 4)):
      t = time.perf_counter()
      kitti.analysis_text(stats)
      text = kitti.error_file_text(ids, names, lines)
      ft.append((time.perf_counter() - t) * 1e3)
    res['format_ms'] = _stats(ft)
    res['error_lines'] = len(lines)
    res['stats'] = stats
    all_boxes = [[None] * args.images for _ in names]
    for i, r in enumerate(records):
      per = detections_to_all_boxes(r, len(r), None, len(names))
      for k in range(len(names)):
        all_boxes[k][i] = per[k]
    result = write_kitti_detections(os.path.join(tmp, 'result', 'data'), ids, names, all_boxes)
    ot = []
    for _ in range(args.oracle_runs):
      t = time.perf_counter()
      want, _ = kitti_analysis.analyze(lab_dir, os.path.join(result, 'data'), ids, names)
      ot.append(time.perf_counter() - t)
    res['oracle_s'] = _stats(ot)
    res['bytes_identical'] = bool(want == text and len(want) > 0)
  return res


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
