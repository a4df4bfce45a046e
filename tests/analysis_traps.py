"""Labelled sets for the detection error analysis: one small set per rule of the reference's
analyze_detections that a restatement could get wrong (traps()), and the KITTI tree both the
oracle and the reference read.  A set is (labels, records) as in tests/kitti_traps.py.
tests/test_oracle_kitti_analysis.py shows that each trap's case occurs."""
import os

import numpy as np

import kitti_traps as kt
from kitti_traps import CAR, CYC, PED, label, rec, recs
from oracle import kitti_analysis as ka
from squeezedet_b200.bench_kitti_eval import synthetic_set

CLASS_NAMES = kt.CLASS_NAMES
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'analysis_kat.npz')
STAT_KEYS = ('num of detections', 'num of objects', '% correct detections',
             '% localization error', '% classification error', '% background error', '% repeated error', '% recall')


def golden_sets():
  """[(name, labels, records, error bytes, stats, printed text)] of the golden fixture."""
  z = np.load(GOLDEN)
  out = []
  for name in z['names'].tolist():
    text, off = z['labels_' + name].tobytes(), z['label_offsets_' + name]
    labels = [text[a:b].decode() for a, b in zip(off[:-1], off[1:])]
    dets, counts = z['dets_' + name], z['counts_' + name]
    ends = np.cumsum(counts)
    records = [dets[e - c:e] for c, e in zip(counts, ends)]
    out.append((name, labels, records, z['error_' + name].tobytes(),
                dict(zip(STAT_KEYS, z['stats_' + name].tolist())),
                z['printed_' + name].tobytes().decode()))
  return out


def random_set(seed, n, dets=64, **kw):
  """A seeded KITTI-like set whose analyzed labels the reference accepts."""
  return synthetic_set(seed, n, dets, analyzable=True, **kw)


def traps():
  """[(name, labels, records)]: each set isolates one rule."""
  out = []

  def add(name, images):
    out.append((name, [''.join(l) for l, _ in images], [recs(*r) for _, r in images]))

  # G = 2: only the two best-scoring detections count; the third (a perfect match of the second
  # car) and the fourth (background) are neither counted nor written, so the second car is missed
  add('past_g', [([label('Car', 0, 0, 99, 99), label('Car', 200, 0, 299, 99)],
                  [rec(CAR, 0, 0, 99, 99, 0.9), rec(CAR, 500, 0, 599, 99, 0.8),
                   rec(CAR, 200, 0, 299, 99, 0.7), rec(CAR, 700, 0, 799, 99, 0.6)])])
  # detections on an image with no analyzed object (a Van only) and on an empty label file:
  # nothing counted, nothing written; then an image that counts
  add('no_objects', [([label('Van', 0, 0, 99, 99)], [rec(CAR, 0, 0, 99, 99, 0.9)]),
                     ([], [rec(PED, 0, 0, 20, 50, 0.5), rec(CAR, 0, 0, 99, 99, 0.4)]),
                     ([label('Car', 0, 0, 99, 99)], [rec(CAR, 300, 0, 399, 99, 0.5)])])
  # scores that print alike ('0.500'): the file order decides, car lines before pedestrian lines
  # (the pedestrian record comes first and would be correct), then record order within a class
  # (the first car record is background, the second a hit)
  add('score_ties', [([label('Pedestrian', 0, 0, 30, 80)],
                      [rec(PED, 0, 0, 30, 80, 0.5004), rec(CAR, 400, 0, 499, 99, 0.4996)]),
                     ([label('Car', 0, 0, 99, 99)],
                      [rec(CAR, 600, 0, 699, 99, 0.5001), rec(CAR, 0, 0, 99, 99, 0.4999)])])
  # IoU of exactly 0.5 (correct: >= 0.5) and exactly 0.1 (bg: not > 0.1), with their neighbours
  # 0.49 (loc) and 0.11 (loc); widths are x2 - x1 + 1, so 0..99 is 100 wide
  add('iou_exact', [([label('Car', 0, 0, 99, 99), label('Car', 200, 0, 299, 99),
                      label('Car', 400, 0, 499, 99), label('Car', 600, 0, 699, 99)],
                     [rec(CAR, 0, 0, 49, 99, 0.9), rec(CAR, 200, 0, 209, 99, 0.8),
                      rec(CAR, 400, 0, 448, 99, 0.7), rec(CAR, 600, 0, 610, 99, 0.6)])])
  # one detection overlapping two objects equally (0.6 each): the first in label order takes it,
  # a pedestrian (cls) here and a car (correct) in the swapped file
  tie = [label('Pedestrian', 0, 0, 99, 99), label('Car', 50, 0, 149, 99)]
  add('argmax_tie', [(tie, [rec(CAR, 25, 0, 124, 99, 0.9)])])
  add('argmax_tie_swapped', [(tie[::-1], [rec(CAR, 25, 0, 124, 99, 0.9)])])
  # three hits on one car: the best-scoring is correct, the other two repeated (G = 3)
  add('repeated', [([label('Car', 0, 0, 99, 99), label('Car', 300, 0, 399, 99),
                     label('Cyclist', 600, 0, 640, 80)],
                    [rec(CAR, 2, 0, 99, 99, 0.5), rec(CAR, 0, 0, 99, 99, 0.9),
                     rec(CAR, 0, 2, 99, 99, 0.7)])])
  # a car detection whose best object is a pedestrian (0.9) though a car overlaps it by 0.6:
  # a classification error
  add('cls_over_same', [([label('Car', 10, 0, 109, 99), label('Pedestrian', 40, 0, 139, 99)],
                         [rec(CAR, 40, 0, 129, 99, 0.8), rec(PED, 800, 0, 830, 80, 0.1)])])
  # Van, DontCare, Person_sitting, Truck are not ground truth, even with x1 < 0, which the
  # reference would assert against in an analyzed class; 'CAR' and 'cyclist' lowercase to classes
  add('ignored_types', [([label('Van', -10, 0, 50, 60), label('DontCare', -5, -5, 40, 40,
                                                                trunc=-1, occ=-1, alpha=-10),
                          label('Person_sitting', -3, 10, 30, 90), label('Truck', -20, 0, 9, 9),
                          label('CAR', 100, 0, 199, 99), label('cyclist', 300, 0, 340, 80)],
                         [rec(CAR, -10, 0, 50, 60, 0.9), rec(PED, -3, 10, 30, 90, 0.8),
                          rec(CAR, 100, 0, 199, 99, 0.7)])])
  # a detection at x1 = -0.04 prints '-0.0'; corners on quarters print .1f ties (10.25 -> '10.2',
  # 31.75 -> '31.8', the x-max being the corner plus 1)
  add('print_edges', [([label('Car', 500, 0, 599, 99), label('Car', 700, 0, 799, 99)],
                       [rec(CAR, -0.04, 3.25, 20.5, 40.75, 0.6),
                        rec(PED, 10.25, 0.75, 30.75, 60.25, 0.55)])])
  return out


def write_tree(root, labels, records, class_names=CLASS_NAMES):
  """The set's KITTI tree under root, as eval.py leaves it (tests/kitti_traps.write_set) ->
  (label_dir, detection data dir, image ids)."""
  kitti_dir, _, result, ids = kt.write_set(root, labels, records, class_names)
  return os.path.join(kitti_dir, 'label_2'), os.path.join(result, 'data'), ids


def oracle(root, labels, records):
  """(error file text, counts) of the oracle on the set's files."""
  lab, det, ids = write_tree(root, labels, records)
  return ka.analyze(lab, det, ids, CLASS_NAMES)


def stacked(records, max_dets=None):
  m = max_dets or max(1, max(len(r) for r in records))
  dets = np.zeros((len(records), m), records[0].dtype if records else kt.DET_DTYPE)
  for i, r in enumerate(records):
    dets[i, :len(r)] = r
  return dets, np.array([len(r) for r in records], np.int32)
