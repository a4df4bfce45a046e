"""Labelled sets for the KITTI scorer: one small set per rule of evaluate_object.cpp that a
restatement could get wrong (traps()), seeded KITTI-like sets of any size (random_set()), and the
files both scorers read.  A set is (labels, records): labels[i] the text of image i's label file,
records[i] a DET_DTYPE array of its filtered detections, as the engine writes them.
tests/test_oracle_kitti_eval.py shows that each trap's case occurs."""
import os
import subprocess

import numpy as np

from squeezedet_b200._lib import DET_DTYPE
from squeezedet_b200.bench_kitti_eval import label_line, synthetic_set
from squeezedet_b200.eval import EVAL_TOOL, detections_to_all_boxes
from squeezedet_b200.utils.viz import write_kitti_detections

CLASS_NAMES = ('car', 'pedestrian', 'cyclist')


label = label_line


def rec(cls, x1, y1, x2, y2, prob):
  """A record whose corners, after bbox_transform in float32, print as x1 y1 x2 y2 when they are
  multiples of 1/4."""
  r = np.zeros((), DET_DTYPE)
  w, h = np.float32(x2 - x1), np.float32(y2 - y1)
  r['cls'], r['prob'] = cls, np.float32(prob)
  r['cx'], r['cy'] = np.float32(x1) + w / np.float32(2), np.float32(y1) + h / np.float32(2)
  r['w'], r['h'] = w, h
  return r


def recs(*rs):
  out = np.zeros((len(rs),), DET_DTYPE)
  for j, r in enumerate(rs):
    out[j] = r
  return out


CAR, PED, CYC = 0, 1, 2


def traps():
  """[(name, labels, records)]: each set isolates one rule."""
  out = []

  def add(name, images):
    out.append((name, [''.join(l) for l, _ in images], [recs(*r) for _, r in images]))

  # heights of exactly 40 and 25 pass easy / moderate (strict < ignores); 39.99 and 24.99 fail
  add('heights', [([label('Car', 0, 0, 50, 40), label('Car', 100, 0, 150, 25),
                    label('Car', 200, 0, 250, 39.99), label('Pedestrian', 300, 0, 320, 25),
                    label('Pedestrian', 400, 0, 420, 24.99)],
                   [rec(CAR, 0, 0, 50, 40, 0.9), rec(CAR, 100, 0, 150, 25, 0.8),
                    rec(CAR, 200, 0, 250, 40, 0.7), rec(PED, 300, 0, 320, 25, 0.6),
                    rec(PED, 400, 0, 420, 25, 0.5)])])
  # truncations of exactly 0.15, 0.3, 0.5 pass (strict > ignores); occlusion 3 fails everything
  add('truncation_occlusion', [([label('Car', 0, 0, 100, 50, trunc=0.15),
                                 label('Car', 200, 0, 300, 50, trunc=0.3),
                                 label('Car', 400, 0, 500, 50, trunc=0.5),
                                 label('Car', 600, 0, 700, 50, trunc=0.51),
                                 label('Car', 800, 0, 900, 50, occ=3),
                                 label('Car', 0, 100, 100, 150, occ=1),
                                 label('Car', 200, 100, 300, 150, occ=2)],
                                [rec(CAR, 0, 0, 100, 50, 0.9), rec(CAR, 200, 0, 300, 50, 0.8),
                                 rec(CAR, 400, 0, 500, 50, 0.7), rec(CAR, 600, 0, 700, 50, 0.6),
                                 rec(CAR, 800, 0, 900, 50, 0.5), rec(CAR, 0, 100, 100, 150, 0.4),
                                 rec(CAR, 200, 100, 300, 150, 0.3)])])
  # neighbour classes: a Van takes a car detection without counting, as does a Person_sitting
  add('neighbours', [([label('Van', 0, 0, 100, 60), label('Person_sitting', 200, 0, 230, 60),
                       label('Car', 300, 0, 400, 60), label('Truck', 500, 0, 600, 60)],
                      [rec(CAR, 0, 0, 100, 60, 0.9), rec(PED, 200, 0, 230, 60, 0.8),
                       rec(CAR, 300, 0, 400, 60, 0.7), rec(CAR, 500, 0, 600, 60, 0.6)])])
  # IoU exactly 7/10 (car) and 5/10 (pedestrian) from integer corners is not > the minimum:
  # gt 0..100 x 0..100, detection 0..70 x 0..100 -> 7000 / 10000; 0..50 -> 5000 / 10000
  add('iou_exact', [([label('Car', 0, 0, 100, 100), label('Pedestrian', 200, 0, 300, 100)],
                     [rec(CAR, 0, 0, 70, 100, 0.9), rec(PED, 200, 0, 250, 100, 0.8),
                      rec(CAR, 0, 0, 71, 100, 0.7)])])
  # equal scores and equal overlaps, where the first detection index wins and the other choice
  # changes the counts.  Two cars, 0..100 and 20..120; detections -10..90 and 10..110 overlap
  # the first car equally (9000 / 11000), and only 10..110 matches the second car.
  cars = [label('Car', 0, 0, 100, 100), label('Car', 20, 0, 120, 100)]
  # recall pass: equal scores, so the first car takes the first detection: -10..90 leaves the
  # second car its match (2 TPs), 10..110 first does not (1 TP)
  add('ties_recall', [(cars, [rec(CAR, -10, 0, 90, 100, 0.5), rec(CAR, 10, 0, 110, 100, 0.5)])])
  add('ties_recall_swapped', [(cars, [rec(CAR, 10, 0, 110, 100, 0.5),
                                      rec(CAR, -10, 0, 90, 100, 0.5)])])
  # PR pass: the scores differ (the recall pass has no tie and gives thresholds 0.6 and 0.5), and
  # at 0.5 the first car takes the first of its two equal overlaps
  add('ties_pr', [(cars, [rec(CAR, -10, 0, 90, 100, 0.6), rec(CAR, 10, 0, 110, 100, 0.5)])])
  add('ties_pr_swapped', [(cars, [rec(CAR, 10, 0, 110, 100, 0.5),
                                  rec(CAR, -10, 0, 90, 100, 0.6)])])
  # identical boxes and scores: either choice gives the same counts
  add('ties', [([label('Car', 0, 0, 100, 100), label('Car', 300, 0, 400, 100)],
                [rec(CAR, 5, 0, 105, 100, 0.5), rec(CAR, -5, 0, 95, 100, 0.5),
                 rec(CAR, 300, 0, 400, 100, 0.5), rec(CAR, 300, 0, 400, 100, 0.5)])])
  # a DontCare box absorbs a false positive (inter / det_area > minimum); one outside does not,
  # nor one whose stuff overlap is exactly 7/10 (130..230 x 0..100 in 0..200: 7000 / 10000)
  add('dontcare', [([label('DontCare', 0, 0, 200, 200, trunc=-1, occ=-1, alpha=-10),
                     label('Car', 400, 0, 500, 100)],
                    [rec(CAR, 10, 10, 100, 100, 0.9), rec(CAR, 150, 150, 250, 250, 0.8),
                     rec(CAR, 130, 0, 230, 100, 0.75), rec(CAR, 400, 0, 500, 100, 0.7)])])
  # 0/0 precision: in the recall pass a Van takes the higher-scoring detection A and the Car
  # after it takes B (a TP); in the PR pass the Van takes B, its higher overlap, A misses the Car
  # and lies in a DontCare box, so the only threshold has TP + FP = 0 -> -nan, kept by suffix max
  add('nan_precision', [([label('Van', 0, 0, 100, 100), label('Car', 20, 0, 120, 100),
                          label('DontCare', 0, 0, 90, 110, trunc=-1, occ=-1, alpha=-10)],
                         [rec(CAR, 0, 0, 80, 100, 0.9), rec(CAR, 10, 0, 110, 100, 0.5)]),
                        ([label('Car', 0, 0, 100, 100)], [rec(CAR, 0, 0, 100, 100, 0.3)])])
  # n_gt of 0 (pedestrian), under 41 (car, 7) and well over 41 (cyclist, 120)
  imgs = []
  for k in range(12):
    ls, rs = [], []
    for m in range(10):
      x = 60 * m
      ls.append(label('Cyclist', x, 0, x + 50, 60))
      if (k + m) % 3:
        rs.append(rec(CYC, x, 0, x + 50, 60, ((k * 10 + m) * 7 % 1000) / 1000.0))
    if k < 7:
      ls.append(label('Car', 0, 100, 100, 200))
      rs.append(rec(CAR, 0, 100, 100, 200, 0.1 * (k + 1)))
    rs.append(rec(PED, 700, 0, 720, 50, 0.3))
    imgs.append((ls, rs))
  add('n_gt', imgs)
  # scores of exactly 0.000 and 1.000, and 0.0004 and 0.9995 (a float32 just below), which print
  # as 0.000 and 0.999
  add('score_ends', [([label('Car', 0, 0, 100, 100), label('Car', 200, 0, 300, 100)],
                      [rec(CAR, 0, 0, 100, 100, 0.0), rec(CAR, 200, 0, 300, 100, 1.0),
                       rec(CAR, 400, 0, 500, 100, 0.0004), rec(CAR, 600, 0, 700, 100, 0.9995)])])
  # empty label files, an image with no detections, a class never detected (cyclist: no files)
  add('empty', [([], [rec(CAR, 0, 0, 100, 100, 0.5)]),
                ([label('Car', 0, 0, 100, 100), label('Cyclist', 200, 0, 250, 100)], []),
                ([label('Car', 0, 0, 100, 100)], [rec(CAR, 0, 0, 100, 100, 0.6),
                                                  rec(PED, 0, 0, 20, 50, 0.2)])])
  # degenerate (zero, negative size) and negative-coordinate boxes, gt and detection
  add('degenerate', [([label('Car', -50, -40, 50, 60), label('Car', 100, 100, 100, 200),
                       label('Car', 300, 300, 200, 400), label('DontCare', -10, -10, -10, 50)],
                      [rec(CAR, -50, -40, 50, 60, 0.9), rec(CAR, 100, 100, 100, 200, 0.8),
                       rec(CAR, 300, 300, 200, 400, 0.7), rec(CAR, -30, -30, 0, 0, 0.6)])])
  return out


random_set = synthetic_set


def write_set(root, labels, records, class_names=CLASS_NAMES):
  """The KITTI tree of a set under `root`, as eval.py leaves it: training/label_2/<id>.txt,
  ImageSets/val.txt and result/data/<id>.txt (written by eval.py's own writer).  Returns
  (kitti_dir, image_set_file, result_dir, image ids)."""
  root = str(root)
  ids = ['%06d' % i for i in range(len(labels))]
  lab = os.path.join(root, 'training', 'label_2')
  os.makedirs(lab, exist_ok=True)
  os.makedirs(os.path.join(root, 'ImageSets'), exist_ok=True)
  for i, text in zip(ids, labels):
    with open(os.path.join(lab, i + '.txt'), 'w') as f:
      f.write(text)
  image_set = os.path.join(root, 'ImageSets', 'val.txt')
  with open(image_set, 'w') as f:
    f.write('\n'.join(ids) + '\n')
  all_boxes = [[None] * len(ids) for _ in class_names]
  for i, r in enumerate(records):
    per = detections_to_all_boxes(r, len(r), None, len(class_names))
    for c in range(len(class_names)):
      all_boxes[c][i] = per[c]
  result = write_kitti_detections(os.path.join(root, 'result', 'data'), ids, class_names, all_boxes)
  return os.path.join(root, 'training'), image_set, result, ids


def output_files(result_dir):
  """{relative path: bytes} of the scorer's text outputs under result_dir (stats_*.txt and
  plot/*.txt)."""
  out = {}
  for name in sorted(os.listdir(result_dir)):
    if name.startswith('stats_') and name.endswith('.txt'):
      out[name] = open(os.path.join(result_dir, name), 'rb').read()
  plot = os.path.join(result_dir, 'plot')
  if os.path.isdir(plot):
    for name in sorted(os.listdir(plot)):
      if name.endswith('.txt'):
        out[os.path.join('plot', name)] = open(os.path.join(plot, name), 'rb').read()
  return out


def run_binary(kitti_dir, image_set, result_dir, n):
  """evaluate_object on the set, its gnuplot and ps2pdf calls left to fail quietly; -> its files."""
  subprocess.run([EVAL_TOOL, kitti_dir, image_set, result_dir, str(n)], check=True,
                 stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
  return output_files(result_dir)
