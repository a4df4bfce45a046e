"""The GPU detection analysis (squeezedet_b200.kitti.analyze_device) against oracle/kitti_analysis.py
and the reference's stored output (tests/golden/analysis_kat.npz): the same error file bytes and
counts on every trap, on random sets of 1 to 1024 records per image and on a val-sized set;
refusals naming the first bad image; bitwise repeatability; and eval.py's block and error file on
a generated KITTI tree."""
import os

import numpy as np
import pytest

import analysis_traps as at
from analysis_traps import golden_sets
from gpu_util import make_kitti
from oracle import kitti_analysis as ka
from squeezedet_b200 import kitti
from squeezedet_b200 import eval as sq_eval

pytestmark = pytest.mark.gpu


def device_text(tmp_path, labels, records, device, max_dets=None):
  """(GPU error file text, GPU stats, oracle text, oracle stats) of one set."""
  lab_dir, det_dir, ids = at.write_tree(tmp_path, labels, records)
  lab = kitti.read_labels(lab_dir, ids)
  dets, counts = at.stacked(records, max_dets)
  stats, lines = kitti.analyze_device(dets, counts, at.CLASS_NAMES, lab, device='cuda:%d' % device)
  text, want = ka.analyze(lab_dir, det_dir, ids, at.CLASS_NAMES)
  return kitti.error_file_text(ids, at.CLASS_NAMES, lines), stats, text, kitti.analysis_stats(want)


def same(a, b):
  return repr(a) == repr(b)          # nan == nan


@pytest.mark.parametrize('name', [t[0] for t in at.traps()])
def test_traps(tmp_path, name, gpu_device):
  _, labels, records = next(t for t in at.traps() if t[0] == name)
  got, stats, want, want_stats = device_text(tmp_path, labels, records, gpu_device)
  assert got == want and same(stats, want_stats)


@pytest.mark.parametrize('name', [s[0] for s in golden_sets()])
def test_golden(tmp_path, name, gpu_device):
  _, labels, records, error, stats, printed = next(s for s in golden_sets() if s[0] == name)
  got, got_stats, _, _ = device_text(tmp_path, labels, records, gpu_device)
  assert got.encode() == error
  assert got_stats == stats and kitti.analysis_text(got_stats) == printed


@pytest.mark.parametrize('seed, dets', [(0, 1), (1, 7), (2, 33), (3, 64), (4, 300), (5, 1024)])
def test_random_sets(tmp_path, seed, dets, gpu_device):
  labels, records = at.random_set(200 + seed, max(8, 200 // (1 + dets // 64)), dets=dets)
  got, stats, want, want_stats = device_text(tmp_path, labels, records, gpu_device)
  assert got == want and same(stats, want_stats) and len(want) > 0


def test_more_objects_than_threads(tmp_path, gpu_device):
  """600 labels in an image and 400 records: the label loops, the ranks and the line scans
  each run over more than one CTA-wide chunk."""
  labels, records = at.random_set(9, 3, dets=400, min_labels=600, max_labels=600)
  got, stats, want, want_stats = device_text(tmp_path, labels, records, gpu_device)
  assert got == want and same(stats, want_stats) and stats['num of detections'] > 256


def test_val_sized_set(tmp_path, gpu_device):
  labels, records = at.random_set(2024, 3769)
  got, stats, want, want_stats = device_text(tmp_path, labels, records, gpu_device)
  assert got == want and same(stats, want_stats)
  assert got.count('\n') > 1024 and all(v > 0 for v in stats.values())


def test_twice_bitwise(tmp_path, gpu_device):
  labels, records = at.random_set(7, 300)
  lab_dir, _, ids = at.write_tree(tmp_path, labels, records)
  lab = kitti.read_labels(lab_dir, ids)
  dets, counts = at.stacked(records)
  runs = [kitti.analyze_device(dets, counts, at.CLASS_NAMES, lab, device='cuda:%d' % gpu_device)
          for _ in range(2)]
  assert repr(runs[0][0]) == repr(runs[1][0])
  assert runs[0][1].tobytes() == runs[1][1].tobytes() and len(runs[0][1]) > 0


@pytest.mark.parametrize('field, value, reason', [
    ('count', -1, 'count'), ('count', 9, 'count'), ('cls', 3, 'class id'), ('cls', -1, 'class id'),
    ('prob', np.nan, 'non-finite'), ('cx', np.inf, 'non-finite'), ('prob', 1.0001, 'outside'),
    ('w', -0.5, 'w < 0'), ('h', -1e-3, 'w < 0')])
def test_record_refusals_name_the_image(tmp_path, field, value, reason, gpu_device):
  labels, records = at.random_set(3, 6, dets=8)
  lab_dir, _, ids = at.write_tree(tmp_path, labels, records)
  lab = kitti.read_labels(lab_dir, ids)
  dets, counts = at.stacked(records)
  for i in (4, 2):                       # the first bad image is named
    if field == 'count':
      counts[i] = value
    else:
      dets[i, 5][field] = value
  with pytest.raises(ValueError, match='image 2: .*' + reason):
    kitti.analyze_device(dets, counts, at.CLASS_NAMES, lab, device='cuda:%d' % gpu_device)


@pytest.mark.parametrize('box', [(-0.5, 0, 10, 10), (5, 0, 4, 10), (0, -1, 10, 10), (0, 5, 10, 4),
                                 (0, 0, np.inf, 10), (np.nan, 0, 10, 10)])
def test_label_refusals_name_the_image(tmp_path, box, gpu_device):
  """A car box the reference asserts against (or one not finite) is refused; the same box on a
  Van is not ground truth and is fine."""
  labels, records = at.random_set(4, 5, dets=8)
  lab_dir, _, ids = at.write_tree(tmp_path, labels, records)
  lab = kitti.read_labels(lab_dir, ids)
  dets, counts = at.stacked(records)
  dev = 'cuda:%d' % gpu_device
  objs = lab.objs.copy()
  for i in (3, 1):
    g = lab.offsets[i]
    objs[g]['x1'], objs[g]['y1'], objs[g]['x2'], objs[g]['y2'] = box
    objs[g]['type'] = kitti.TYPE_CODES['van']
  kitti.analyze_device(dets, counts, at.CLASS_NAMES, kitti.Labels(objs, lab.offsets), device=dev)
  for i in (3, 1):
    objs[lab.offsets[i]]['type'] = kitti.TYPE_CODES['car']
  with pytest.raises(ValueError, match="image 1: a label box .* reference's assertions"):
    kitti.analyze_device(dets, counts, at.CLASS_NAMES, kitti.Labels(objs, lab.offsets), device=dev)


def test_bad_offsets_are_refused(tmp_path, gpu_device):
  labels, records = at.random_set(4, 3, dets=8, min_labels=2, max_labels=2)
  lab_dir, _, ids = at.write_tree(tmp_path, labels, records)
  lab = kitti.read_labels(lab_dir, ids)
  dets, counts = at.stacked(records)
  with pytest.raises(ValueError, match='image 1: its label offsets'):
    kitti.analyze_device(dets, counts, at.CLASS_NAMES,
                         kitti.Labels(lab.objs[:5], np.array([0, 3, 2, 5], np.int64)),
                         device='cuda:%d' % gpu_device)


def test_no_objects_at_all(tmp_path, gpu_device):
  """No label lines anywhere: objs and the line buffer are empty, nothing is counted and every
  share is nan."""
  _, records = at.random_set(5, 4, dets=16)
  got, stats, want, want_stats = device_text(tmp_path, [''] * 4, records, gpu_device)
  assert got == want == '' and same(stats, want_stats)
  assert stats['num of detections'] == 0.0 and np.isnan(stats['% recall'])


def test_capacity_above_1024(tmp_path, gpu_device):
  """A record capacity above 1024 is cut to the largest count: the same lines as a tight one."""
  labels, records = at.random_set(6, 50, dets=40)
  tight, s1, want, _ = device_text(tmp_path / 'a', labels, records, gpu_device)
  wide, s2, _, _ = device_text(tmp_path / 'b', labels, records, gpu_device, max_dets=2000)
  assert tight == wide == want and same(s1, s2)


def test_eval_once_prints_and_writes_the_analysis(tmp_path, gpu_device, capsys):
  data, ids, _ = make_kitti(tmp_path)
  flags = sq_eval.parse_flags(['--data_path', str(data), '--image_set', 'val',
                               '--eval_dir', str(tmp_path / 'eval'), '--checkpoint_path',
                               'synthetic', '--net', 'squeezeDet', '--gpu', str(gpu_device)])
  capsys.readouterr()
  sq_eval.eval_once(flags)
  printed = capsys.readouterr().out
  res = tmp_path / 'eval' / 'detection_files_0'
  text, counts = ka.analyze(str(data / 'training' / 'label_2'), str(res / 'data'), ids,
                            ('car', 'pedestrian', 'cyclist'))
  assert (res / 'error_analysis' / 'det_error_file.txt').read_text() == text
  block = 'Analyzing detections...\n' + kitti.analysis_text(kitti.analysis_stats(counts))
  assert printed.index('Mean average precision') < printed.index(block)
  assert counts['num_objs'] == 3
  # a car box the reference asserts against: an error naming the image, no error file
  (data / 'training' / 'label_2' / (ids[1] + '.txt')).write_text(
      'Car 0.00 0 -1.57 -5.00 120.00 300.00 250.00 1.5 1.6 3.9 1.0 1.7 10.0 -1.5\n')
  flags.eval_dir = str(tmp_path / 'eval2')
  sq_eval.eval_once(flags)
  printed = capsys.readouterr().out
  assert "Couldn't analyze the detections: image 1 (%s.txt): a label box" % ids[1] in printed
  assert not (tmp_path / 'eval2' / 'detection_files_0' / 'error_analysis').exists()
  # an unreadable label file: no analysis at all
  os.remove(data / 'training' / 'label_2' / (ids[1] + '.txt'))
  flags.eval_dir = str(tmp_path / 'eval3')
  sq_eval.eval_once(flags)
  assert 'Analyzing detections' not in capsys.readouterr().out
  # an empty image set: nothing launched, zero counts printed
  (data / 'ImageSets' / 'val.txt').write_text('')
  flags.eval_dir = str(tmp_path / 'eval4')
  sq_eval.eval_once(flags)
  printed = capsys.readouterr().out
  assert '    Number of detections: 0.0\n    Number of objects: 0.0\n' in printed
  assert (tmp_path / 'eval4' / 'detection_files_0' / 'error_analysis' /
          'det_error_file.txt').read_text() == ''
