#!/usr/bin/env python
"""What scoring a val-sized KITTI set costs, on the GPU and with the KITTI devkit's binary.

  python -m squeezedet_b200.bench_kitti_eval --steps 20 --warmup 3

A seeded synthetic set of 3769 images (KITTI's val split size), 2 to 13 labels each with KITTI's
class mix, and 64 filtered records per image, many of them near a label.  The GPU scorer
(kitti.evaluate_device on records already in device memory, labels packed by read_labels) is timed
with CUDA events per call after warm-up: the five kernels, their memsets and the few-KB copy back.
Where oracle/_ref/evaluate_object exists (built by oracle/build_kitti_eval.sh), it is timed with a
host clock on the detection files eval.py's writer makes from the same records, and both sets of
stats files are compared byte for byte.  Everything is written under a temporary directory.

Prints one JSON line with the card's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import tempfile
import time

import numpy as np

from ._lib import DET_DTYPE
from .bench_device_u8 import gpu_info


def label_line(typ, x1, y1, x2, y2, trunc=0.0, occ=0, alpha=-1.57):
  """One KITTI label line: type, truncation, occlusion, alpha, the box, and 7 unscored fields."""
  return '%s %.2f %d %.2f %.2f %.2f %.2f %.2f 1.50 1.60 3.90 1.00 1.70 10.00 -1.50\n' % (
      typ, trunc, occ, alpha, x1, y1, x2, y2)


TYPES = ('Car', 'Pedestrian', 'Cyclist', 'Van', 'Person_sitting', 'Truck', 'Tram', 'Misc',
         'DontCare')
TYPE_P = (0.45, 0.08, 0.03, 0.05, 0.01, 0.02, 0.01, 0.02, 0.33)


def synthetic_set(seed, n, dets=64, max_labels=13, min_labels=2, analyzable=False):
  """(labels, records): label file texts and DET_DTYPE record arrays of a seeded KITTI-like set: n images of min..max labels with KITTI's class mix, 1242x375, and
  `dets` records per image: some jittered around each car / pedestrian / cyclist label (at the
  label's class or another), the rest anywhere.  With `analyzable`, car / pedestrian / cyclist
  labels start at x1 >= 0, as the reference's detection analysis asserts (the same draws, so the
  set is otherwise unchanged)."""
  rng = np.random.default_rng(seed)
  labels, records = [], []
  for _ in range(n):
    k = int(rng.integers(min_labels, max_labels + 1))
    lines, boxes = [], []
    for _ in range(k):
      t = TYPES[int(rng.choice(len(TYPES), p=TYPE_P))]
      w = float(rng.uniform(15, 300))
      h = float(rng.uniform(15, 200)) if rng.random() < 0.8 else float(rng.choice([25, 40]))
      x1, y1 = float(rng.uniform(-20, 1200)), float(rng.uniform(0, 340))
      if analyzable and t in ('Car', 'Pedestrian', 'Cyclist'):
        x1 = abs(x1)
      if t == 'DontCare':
        lines.append(label_line(t, x1, y1, x1 + w, y1 + h, trunc=-1, occ=-1, alpha=-10))
        continue
      trunc = float(rng.choice([0.0, 0.15, 0.3, 0.5, rng.uniform(0, 1)]))
      lines.append(label_line(t, x1, y1, x1 + w, y1 + h, trunc=trunc, occ=int(rng.integers(0, 4)),
                         alpha=float(rng.uniform(-np.pi, np.pi))))
      boxes.append((t, round(x1, 2), round(y1, 2), round(x1 + w, 2), round(y1 + h, 2)))
    r = np.zeros((dets,), DET_DTYPE)
    for j in range(dets):
      if boxes and rng.random() < 0.6:
        t, x1, y1, x2, y2 = boxes[int(rng.integers(len(boxes)))]
        cls = {'Car': 0, 'Van': 0, 'Pedestrian': 1, 'Person_sitting': 1}.get(t, 2)
        if rng.random() < 0.15:
          cls = int(rng.integers(3))
        s = rng.normal(0, 0.08, 4) * np.array([x2 - x1, y2 - y1] * 2)
        x1, y1, x2, y2 = x1 + s[0], y1 + s[1], x2 + s[2], y2 + s[3]
      else:
        cls = int(rng.integers(3))
        x1, y1 = rng.uniform(-20, 1200), rng.uniform(0, 340)
        x2, y2 = x1 + rng.uniform(5, 300), y1 + rng.uniform(5, 200)
      r[j]['cls'] = cls
      r[j]['prob'] = np.float32(rng.random() if rng.random() < 0.9 else rng.integers(0, 1001) / 1000)
      r[j]['cx'], r[j]['cy'] = np.float32((x1 + x2) / 2), np.float32((y1 + y2) / 2)
      r[j]['w'], r[j]['h'] = np.float32(x2 - x1), np.float32(y2 - y1)
    labels.append(''.join(lines))
    records.append(r)
  return labels, records


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--images', type=int, default=3769)
  ap.add_argument('--dets', type=int, default=64)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--binary_runs', type=int, default=3)
  ap.add_argument('--seed', type=int, default=2024)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def _files(result_dir):
  out = {}
  for root, _, names in os.walk(result_dir):
    for name in names:
      if name.startswith('stats_') or os.path.basename(root) == 'plot' and name.endswith('.txt'):
        with open(os.path.join(root, name), 'rb') as f:
          out[os.path.relpath(os.path.join(root, name), result_dir)] = f.read()
  return out


def measure(args):
  import torch
  from . import kitti
  from .eval import EVAL_TOOL, detections_to_all_boxes
  from .utils.viz import write_kitti_detections
  names = ('car', 'pedestrian', 'cyclist')
  dev = torch.device('cuda', args.gpu)
  labels, records = synthetic_set(args.seed, args.images, args.dets)
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
      scores = kitti.evaluate_device(d, c, names, lab)
    times = []
    for _ in range(args.steps):
      t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      t0.record()
      scores = kitti.evaluate_device(d, c, names, lab)
      t1.record()
      t1.synchronize()
      times.append(t0.elapsed_time(t1))
    res['device_ms'] = {'median': float(np.median(times)), 'min': float(np.min(times)),
                        'max': float(np.max(times))}
    res['ap'] = {k: v[2] for k, v in scores.items()}
    dev_dir = os.path.join(tmp, 'device')
    kitti.write_stats(dev_dir, scores)
    if os.path.exists(EVAL_TOOL):
      all_boxes = [[None] * args.images for _ in names]
      for i, r in enumerate(records):
        per = detections_to_all_boxes(r, len(r), None, len(names))
        for k in range(len(names)):
          all_boxes[k][i] = per[k]
      result = write_kitti_detections(os.path.join(tmp, 'result', 'data'), ids, names, all_boxes)
      image_set = os.path.join(tmp, 'val.txt')
      with open(image_set, 'w') as f:
        f.write('\n'.join(ids) + '\n')
      bt = []
      for _ in range(args.binary_runs):
        t = time.perf_counter()
        subprocess.run([EVAL_TOOL, os.path.join(tmp, 'training'), image_set, result,
                        str(args.images)], check=True, stdout=subprocess.DEVNULL,
                       stderr=subprocess.DEVNULL)
        bt.append(time.perf_counter() - t)
      res['binary_s'] = {'median': float(np.median(bt)), 'min': float(np.min(bt))}
      want, got = _files(result), _files(dev_dir)
      res['files_identical'] = bool(want == got and len(want) > 0)
    else:
      res['binary_s'] = None
      res['files_identical'] = None
  return res


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
