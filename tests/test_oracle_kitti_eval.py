"""oracle/kitti_eval.py against the KITTI devkit's evaluate_object (oracle/_ref/, compiled by
oracle/build_kitti_eval.sh where the reference checkout is present): byte-identical files on every
trap of tests/kitti_traps.py, on seeded random sets and on a val-sized set, with each trap's case
shown to occur; and the decimal identity that lets the GPU scorer skip the text round trip."""
import os

import numpy as np
import pytest

import kitti_traps as kt
from oracle import kitti_eval as ke
from squeezedet_b200.eval import EVAL_TOOL

needs_binary = pytest.mark.skipif(not os.path.exists(EVAL_TOOL),
                                  reason='evaluate_object absent: build() compiles it where the '
                                         'reference checkout exists')
TRAPS = {name: (labels, records) for name, labels, records in kt.traps()}


def oracle_files(tmp_path, labels, records):
  kitti_dir, _, result, ids = kt.write_set(tmp_path, labels, records)
  return ke.run(os.path.join(kitti_dir, 'label_2'), result, ids)


def both(tmp_path, labels, records):
  kitti_dir, image_set, result, ids = kt.write_set(tmp_path, labels, records)
  got = ke.run(os.path.join(kitti_dir, 'label_2'), result, ids)
  want = kt.run_binary(kitti_dir, image_set, result, len(ids))
  return got, want


@needs_binary
@pytest.mark.parametrize('name', sorted(TRAPS))
def test_traps_match_binary(tmp_path, name):
  got, want = both(tmp_path, *TRAPS[name])
  assert sorted(got) == sorted(want)
  for k in want:
    assert got[k] == want[k], (name, k)


@needs_binary
@pytest.mark.parametrize('seed', range(8))
def test_random_sets_match_binary(tmp_path, seed):
  labels, records = kt.random_set(seed, 30 + 20 * seed, dets=int(8 + 20 * seed))
  got, want = both(tmp_path, labels, records)
  assert got == want


@needs_binary
def test_val_sized_set_matches_binary(tmp_path):
  labels, records = kt.random_set(2024, 3769)
  got, want = both(tmp_path, labels, records)
  assert got == want and len(want) == 15


def scores_of(tmp_path, name):
  labels, records = TRAPS[name]
  kitti_dir, _, result, ids = kt.write_set(tmp_path, labels, records)
  gts = [ke.read_groundtruth(os.path.join(kitti_dir, 'label_2', i + '.txt')) for i in ids]
  dets = [ke.read_detections(os.path.join(result, 'data', i + '.txt')) for i in ids]
  return gts, dets, ke.evaluate(gts, dets)


def test_trap_cases_occur(tmp_path):
  # heights 40 / 25 and truncations 0.15 / 0.3 / 0.5 sit exactly on the limits, and are counted
  gts, _, _ = scores_of(tmp_path / 'h', 'heights')
  assert [ke.gt_state(g, 0, 0) for g in gts[0][:3]] == [0, 1, 1]
  assert [ke.gt_state(g, 0, 1) for g in gts[0][:3]] == [0, 0, 0]
  assert [ke.gt_state(g, 1, 1) for g in gts[0][3:]] == [0, 1]
  gts, _, _ = scores_of(tmp_path / 't', 'truncation_occlusion')
  assert [g[1] for g in gts[0][:3]] == [0.15, 0.3, 0.5]
  assert [ke.gt_state(g, 0, d) for d, g in enumerate(gts[0][:3])] == [0, 0, 0]
  assert ke.gt_state(gts[0][3], 0, 2) == 1 and all(ke.gt_state(gts[0][4], 0, d) == 1 for d in range(3))
  # neighbours are ignored (1), other types skipped (-1)
  gts, _, _ = scores_of(tmp_path / 'n', 'neighbours')
  assert [ke.gt_state(g, 0, 0) for g in gts[0]] == [1, -1, 0, -1]
  assert ke.gt_state(gts[0][1], 1, 0) == 1
  # IoU of exactly 7/10 and 5/10, which strict > rejects
  gts, dets, _ = scores_of(tmp_path / 'i', 'iou_exact')
  assert ke.boxoverlap(dets[0][0][2:6], gts[0][0][4:8]) == 0.7
  assert ke.boxoverlap(dets[0][2][2:6], gts[0][1][4:8]) == 0.5
  # equal scores and equal overlaps: swapping the two tied detections is what a last-index rule
  # would do, and it changes the files, so matching the binary in both orders pins the first index
  for name in ('ties_recall', 'ties_pr'):
    gts, dets, _ = scores_of(tmp_path / name, name)
    a, b = dets[0][0][2:6], dets[0][1][2:6]
    assert ke.boxoverlap(a, gts[0][0][4:8]) == ke.boxoverlap(b, gts[0][0][4:8]) > 0.7
    assert ke.boxoverlap(b, gts[0][1][4:8]) > 0.7 > ke.boxoverlap(a, gts[0][1][4:8])
    assert oracle_files(tmp_path / (name + '_f'), *TRAPS[name]) != \
        oracle_files(tmp_path / (name + '_s'), *TRAPS[name + '_swapped'])
  # in ties_recall the recall pass decides: equal scores, and the first choice gives 2 TPs
  gts, dets, _ = scores_of(tmp_path / 'r', 'ties_recall')
  img = ke._Image(gts[0], dets[0])
  states = [ke.gt_state(g, 0, 0) for g in gts[0]]
  assert dets[0][0][6] == dets[0][1][6] and len(ke._recall(img, 0, states)) == 2
  gts, dets, _ = scores_of(tmp_path / 'rs', 'ties_recall_swapped')
  assert len(ke._recall(ke._Image(gts[0], dets[0]), 0, states)) == 1
  # in ties_pr the scores differ, so only the PR pass has a tie: at 0.5 two TPs, swapped one
  gts, dets, _ = scores_of(tmp_path / 'p', 'ties_pr')
  assert dets[0][0][6] != dets[0][1][6]
  assert ke._pr(ke._Image(gts[0], dets[0]), 0, states, 0.5, True)[:3] == (2, 0, 0)
  gts, dets, _ = scores_of(tmp_path / 'ps', 'ties_pr_swapped')
  assert ke._pr(ke._Image(gts[0], dets[0]), 0, states, 0.5, True)[:3] == (1, 1, 1)
  # a DontCare box absorbs a false positive, but not one whose stuff overlap is exactly 7/10
  gts, dets, _ = scores_of(tmp_path / 'd', 'dontcare')
  assert ke.boxoverlap(dets[0][0][2:6], gts[0][0][4:8], 0) > 0.7
  assert ke.boxoverlap(dets[0][2][2:6], gts[0][0][4:8], 0) == 0.7
  assert ke._pr(ke._Image(gts[0], dets[0]), 0, [-1, 0], 0.7, True)[:3] == (1, 2, 0)
  # 0/0 precision: -nan in the first threshold, kept by the suffix maximum, and in the AP
  _, _, s = scores_of(tmp_path / 'z', 'nan_precision')
  p = s['car'][0][0]
  assert np.isnan(p[0]) and not np.isnan(p[1]) and ke.fmt_g(ke.ap_of(p)) == '-nan'
  # n_gt of 0, under 41 and well over 41; more TPs than 41 still give at most 41 thresholds
  gts, _, s = scores_of(tmp_path / 'g', 'n_gt')
  n_gt = [sum(ke.gt_state(g, c, 0) == 0 for img in gts for g in img) for c in range(3)]
  assert n_gt == [7, 0, 120] and set(s) == {'car', 'pedestrian', 'cyclist'}
  # scores 0.000 and 1.000
  _, dets, _ = scores_of(tmp_path / 's', 'score_ends')
  assert [d[6] for d in dets[0]] == [0.0, 1.0, 0.0, 0.999]
  # empty label file, image without detections, a class never detected has no files
  gts, dets, s = scores_of(tmp_path / 'm', 'empty')
  assert gts[0] == [] and dets[1] == [] and 'cyclist' not in s
  assert not any(k.startswith('stats_cyclist') for k in ke.stats_files(s))
  # degenerate and negative boxes
  gts, _, _ = scores_of(tmp_path / 'x', 'degenerate')
  assert gts[0][0][4] < 0 and gts[0][1][4] == gts[0][1][6] and gts[0][2][6] < gts[0][2][4]


def test_at_most_41_thresholds():
  for n in (1, 2, 40, 41, 42, 80, 81, 1000, 12345):
    for tps in {1, n // 2 + 1, n}:
      assert len(ke.get_thresholds(list(np.linspace(1, 0, tps)), n)) <= 41


def test_nan_is_printed_as_glibc_prints_it():
  assert ke.fmt_f(float('-nan')) == '-nan' and ke.fmt_g(float('-nan')) == '-nan'
  assert ke.fmt_f(0.5) == '0.500000' and ke.fmt_g(1 / 11) == '0.0909091' and ke.fmt_g(0.0) == '0'


def test_decimal_identity():
  """'{:.2f}' / '{:.3f}' of a float32 read back as a double is rint(v * 100) / 100 and
  rint(p * 1000) / 1000: v * 100 and v * 1000 are exact in double, and both sides round exact ties
  to even.  A tie of v * 100 is v = (2k + 1) / 200, a float32 only when 25 divides 2k + 1: v is an odd
  multiple of 1/8; likewise a tie of p * 1000 is an odd multiple of 1/16.  Checked on random
  values, on every multiple of 1/8 in [-50000, 50000) and every multiple of 1/16 in [0, 1]."""
  rng = np.random.default_rng(0)
  vals = np.concatenate([rng.uniform(-2000, 3000, 400000).astype(np.float32),
                         rng.uniform(0, 1, 200000).astype(np.float32),
                         (np.arange(-400000, 400000) / np.float32(8)).astype(np.float32)])
  ties = 0
  for v in vals.tolist():
    d = float(np.float32(v))
    ties += (d * 100) % 1 == 0.5
    assert float('%.2f' % d) == np.rint(d * 100.0) / 100.0, d
    if 0 <= d <= 1:
      assert float('%.3f' % d) == np.rint(d * 1000.0) / 1000.0, d
  assert ties > 1000
  for k in range(0, 17):
    d = k / 16
    assert float('%.3f' % d) == np.rint(d * 1000.0) / 1000.0, d
