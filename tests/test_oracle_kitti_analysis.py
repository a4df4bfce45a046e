"""oracle/kitti_analysis.py against the reference's own analyze_detections (imported unmodified
where the reference checkout is present): the same error file bytes and counts on every trap of
tests/analysis_traps.py, on seeded random sets and on a val-sized set, with each trap's case shown
to occur; and, everywhere, against tests/golden/analysis_kat.npz, the reference's stored output."""
import math
import os

import numpy as np
import pytest

import analysis_traps as at
from analysis_traps import golden_sets
from oracle import kitti_analysis as ka
from oracle import ref_import
from squeezedet_b200 import kitti

needs_reference = pytest.mark.skipif(not ref_import.available(),
                                     reason='the reference checkout is absent')
TRAPS = {name: (labels, records) for name, labels, records in at.traps()}


def both(tmp_path, labels, records):
  lab, det, ids = at.write_tree(tmp_path, labels, records)
  text, counts = ka.analyze(lab, det, ids, at.CLASS_NAMES)
  err = str(tmp_path / 'det_error_file.txt')
  out, printed = ka.run_reference(lab, det, ids, at.CLASS_NAMES, err)
  with open(err) as f:
    return (text, counts), (f.read(), out, printed)


def check(got, want):
  (text, counts), (ref_text, out, printed) = got, want
  assert text == ref_text
  stats = kitti.analysis_stats(counts)
  assert list(stats) == list(out) and stats == out
  assert kitti.analysis_text(stats) == printed


@needs_reference
@pytest.mark.parametrize('name', sorted(TRAPS))
def test_traps_match_reference(tmp_path, name):
  check(*both(tmp_path, *TRAPS[name]))


@needs_reference
@pytest.mark.parametrize('seed', range(6))
def test_random_sets_match_reference(tmp_path, seed):
  labels, records = at.random_set(seed, 20 + 15 * seed, dets=[1, 5, 16, 64, 200, 1024][seed])
  check(*both(tmp_path, labels, records))


@needs_reference
def test_val_sized_set_matches_reference(tmp_path):
  labels, records = at.random_set(2024, 3769)
  got, want = both(tmp_path, labels, records)
  check(got, want)
  counts = got[1]
  assert counts['num_objs'] > 10000 and all(counts[k] > 0 for k in ka.COUNT_FIELDS)


@pytest.mark.parametrize('name', [s[0] for s in golden_sets()])
def test_oracle_matches_golden(tmp_path, name):
  _, labels, records, error, stats, printed = next(s for s in golden_sets() if s[0] == name)
  text, counts = at.oracle(tmp_path, labels, records)
  assert text.encode() == error
  got = kitti.analysis_stats(counts)
  assert got == stats and kitti.analysis_text(got) == printed


def test_golden_covers_every_trap():
  assert {s[0] for s in golden_sets()} >= set(TRAPS)


def lines_of(tmp_path, name):
  text, counts = at.oracle(tmp_path, *TRAPS[name])
  return text.splitlines(), counts


def ranked(tmp_path, name, image=0):
  """The oracle's ground truth and sorted detections of one trap image."""
  lab, det, ids = at.write_tree(tmp_path, *TRAPS[name])
  idx = {c: k for k, c in enumerate(at.CLASS_NAMES)}
  return (ka.read_ground_truth(os.path.join(lab, ids[image] + '.txt'), idx),
          ka.read_detections(os.path.join(det, ids[image] + '.txt'), idx))


def test_trap_cases_occur(tmp_path):
  # past G: a perfect match ranked third of two objects is not counted, its car is missed
  lines, c = lines_of(tmp_path / 'g', 'past_g')
  gts, dets = ranked(tmp_path / 'g2', 'past_g')
  assert len(dets) > len(gts) == 2 and max(ka.iou_row(np.array(gts), dets[2][:4])) == 1.0
  assert c['num_dets'] == 2 and lines[-1].startswith('000000 missed 200.0')
  # detections and no objects (a Van, an empty file): nothing counted or written
  lines, c = lines_of(tmp_path / 'n', 'no_objects')
  assert all(ln.startswith('000002') for ln in lines) and c['num_dets'] == 1
  assert ranked(tmp_path / 'n2', 'no_objects', 0)[0] == [] != ranked(tmp_path / 'n3', 'no_objects', 0)[1]
  # .3f ties across classes and within a class: the file order decides which one counts
  for image in (0, 1):
    _, dets = ranked(tmp_path / ('t%d' % image), 'score_ties', image)
    assert dets[0][5] == dets[1][5] == 0.5
  assert ranked(tmp_path / 't3', 'score_ties', 0)[1][0][4] == 0      # the car line, filed first
  lines, c = lines_of(tmp_path / 't', 'score_ties')
  assert c['bg'] == 2 and c['correct'] == 0
  # IoU of exactly 0.5 (correct) and exactly 0.1 (bg)
  gts, dets = ranked(tmp_path / 'i', 'iou_exact')
  ious = [max(ka.iou_row(np.array(gts), d[:4])) for d in dets]
  assert ious[0] == 0.5 and ious[1] == 0.1 and 0.1 < ious[3] < ious[2] < 0.5
  lines, c = lines_of(tmp_path / 'i2', 'iou_exact')
  assert (c['correct'], c['bg'], c['loc']) == (1, 1, 2)
  # argmax ties: the first object in label order wins, and swapping the labels changes the kind
  gts, dets = ranked(tmp_path / 'a', 'argmax_tie')
  row = ka.iou_row(np.array(gts), dets[0][:4])
  assert row[0] == row[1] > 0.5 and gts[0][4] != gts[1][4]
  assert lines_of(tmp_path / 'a2', 'argmax_tie')[1]['cls'] == 1
  assert lines_of(tmp_path / 'a3', 'argmax_tie_swapped')[1]['correct'] == 1
  # repeated hits on one object
  assert lines_of(tmp_path / 'r', 'repeated')[1]['repeated'] == 2
  # a cls error beats a same-class overlap of 0.5 or more
  gts, dets = ranked(tmp_path / 'c', 'cls_over_same')
  row = ka.iou_row(np.array(gts), dets[0][:4])
  assert gts[0][4] == dets[0][4] and row[0] >= 0.5 and row[1] > row[0] and gts[1][4] != dets[0][4]
  assert lines_of(tmp_path / 'c2', 'cls_over_same')[1]['cls'] == 1
  # Van / DontCare / Person_sitting / Truck with x1 < 0 are no ground truth; 'CAR' is a car
  labels = TRAPS['ignored_types'][0][0]
  assert all(float(ln.split()[4]) < 0 for ln in labels.splitlines()[:4])
  assert 'CAR ' in labels
  gts, _ = ranked(tmp_path / 'v', 'ignored_types')
  assert [g[4] for g in gts] == [0, 2]
  # a -0.0 print, .1f ties (10.25 -> 10.2, 0.75 -> 0.8) and x-max printed as the corner plus 1
  lines, _ = lines_of(tmp_path / 'p', 'print_edges')
  assert lines[0].split()[2] == '-0.0' and lines[1].split()[2:6] == ['10.2', '0.8', '31.8', '61.2']


def test_shares_of_nothing_are_nan():
  """The reference raises ZeroDivisionError with no counted detection or no object; the shares
  are nan instead."""
  s = kitti.analysis_stats(dict.fromkeys(ka.COUNT_FIELDS, 0))
  assert s['num of detections'] == 0.0 and all(math.isnan(v) for k, v in s.items() if '%' in k)
  assert kitti.analysis_text(s).splitlines()[3] == '    Percentage of correct detections: nan'
