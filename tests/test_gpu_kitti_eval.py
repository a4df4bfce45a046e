"""The GPU KITTI scorer (squeezedet_b200.kitti) against oracle/kitti_eval.py and, where
oracle/_ref/evaluate_object exists, the devkit's binary: byte-identical files on every trap, on
seeded random sets and on a val-sized set; refusals naming the image; bitwise repeatability; and
eval.py's stats files on a generated KITTI tree."""
import os

import numpy as np
import pytest

import kitti_traps as kt
from gpu_util import make_kitti
from oracle import kitti_eval as ke
from squeezedet_b200 import _lib, kitti
from squeezedet_b200 import eval as sq_eval

pytestmark = pytest.mark.gpu


def stacked(records, max_dets=None):
  m = max_dets or max(1, max(len(r) for r in records))
  dets = np.zeros((len(records), m), _lib.DET_DTYPE)
  for i, r in enumerate(records):
    dets[i, :len(r)] = r
  return dets, np.array([len(r) for r in records], np.int32)


def device_files(tmp_path, labels, records, device, max_dets=None):
  kitti_dir, image_set, result, ids = kt.write_set(tmp_path, labels, records)
  lab = kitti.read_labels(os.path.join(kitti_dir, 'label_2'), ids)
  dets, counts = stacked(records, max_dets)
  scores = kitti.evaluate_device(dets, counts, kt.CLASS_NAMES, lab, device='cuda:%d' % device)
  out = str(tmp_path / 'device')
  kitti.write_stats(out, scores)
  got = kt.output_files(out)
  want = ke.run(os.path.join(kitti_dir, 'label_2'), result, ids)
  if os.path.exists(sq_eval.EVAL_TOOL):
    assert kt.run_binary(kitti_dir, image_set, result, len(ids)) == want
  return got, want, scores


@pytest.mark.parametrize('name', [t[0] for t in kt.traps()])
def test_traps(tmp_path, name, gpu_device):
  _, labels, records = next(t for t in kt.traps() if t[0] == name)
  got, want, _ = device_files(tmp_path, labels, records, gpu_device)
  assert sorted(got) == sorted(want)
  for k in want:
    assert got[k] == want[k], (name, k, got[k], want[k])


@pytest.mark.parametrize('seed', range(6))
def test_random_sets(tmp_path, seed, gpu_device):
  labels, records = kt.random_set(100 + seed, 20 + 30 * seed, dets=[1, 8, 33, 64, 200, 1024][seed])
  got, want, _ = device_files(tmp_path, labels, records, gpu_device)
  assert got == want


def test_val_sized_set(tmp_path, gpu_device):
  labels, records = kt.random_set(2024, 3769)
  got, want, scores = device_files(tmp_path, labels, records, gpu_device)
  assert got == want and len(want) == 15
  assert all(0 < ap < 1 for _, _, aps in scores.values() for ap in aps)


def test_twice_bitwise(tmp_path, gpu_device):
  labels, records = kt.random_set(7, 300)
  kitti_dir, _, _, ids = kt.write_set(tmp_path, labels, records)
  lab = kitti.read_labels(os.path.join(kitti_dir, 'label_2'), ids)
  dets, counts = stacked(records)
  runs = [kitti.evaluate_device(dets, counts, kt.CLASS_NAMES, lab, device='cuda:%d' % gpu_device)
          for _ in range(2)]
  a, b = (np.array([v for s in r.values() for part in s for v in np.ravel(part)]) for r in runs)
  assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize('field, value, reason', [
    ('count', -1, 'count'), ('count', 9, 'count'), ('cls', 3, 'class id'), ('cls', -1, 'class id'),
    ('prob', np.nan, 'non-finite'), ('cx', np.inf, 'non-finite'), ('h', -np.inf, 'non-finite'),
    ('prob', 1.0001, 'outside'), ('prob', -0.001, 'outside')])
def test_refusals_name_the_image(tmp_path, field, value, reason, gpu_device):
  labels, records = kt.random_set(3, 6, dets=8)
  kitti_dir, _, _, ids = kt.write_set(tmp_path, labels, records)
  lab = kitti.read_labels(os.path.join(kitti_dir, 'label_2'), ids)
  dets, counts = stacked(records)
  for i in (4, 2):                       # the first bad image is named
    if field == 'count':
      counts[i] = value
    else:
      dets[i, 5][field] = value
  with pytest.raises(ValueError, match='image 2: .*' + reason):
    kitti.evaluate_device(dets, counts, kt.CLASS_NAMES, lab, device='cuda:%d' % gpu_device)


@pytest.mark.parametrize('offsets', [[0, 3, -1, 5], [0, 3, 2, 5], [0, 3, 9, 5], [0, 3, 3, 9]])
def test_bad_label_offsets_are_refused(tmp_path, offsets, gpu_device):
  """Offsets outside [0, n_objects] or decreasing set the status word only: the kernels score such
  an image as having no objects, so nothing outside objs is read."""
  labels, records = kt.random_set(4, 3, dets=8, min_labels=2, max_labels=2)
  kitti_dir, _, _, ids = kt.write_set(tmp_path, labels, records)
  lab = kitti.read_labels(os.path.join(kitti_dir, 'label_2'), ids)
  assert len(lab.objs) == 6
  lab = kitti.Labels(lab.objs[:5], np.array(offsets, np.int64))
  dets, counts = stacked(records)
  first = next(i for i in range(3) if not 0 <= offsets[i] <= offsets[i + 1] <= 5)
  with pytest.raises(ValueError, match='image %d: its label offsets' % first):
    kitti.evaluate_device(dets, counts, kt.CLASS_NAMES, lab, device='cuda:%d' % gpu_device)


def test_no_objects_at_all(tmp_path, gpu_device):
  """No label lines anywhere: objs is not even allocated, and every detection is a false positive."""
  _, records = kt.random_set(5, 4, dets=16)
  got, want, _ = device_files(tmp_path, [''] * 4, records, gpu_device)
  assert got == want


def test_capacity_above_1024(tmp_path, gpu_device):
  """A record capacity above 1024 is cut to the largest count: the same scores as a tight one."""
  labels, records = kt.random_set(6, 50, dets=40)
  kitti_dir, _, _, ids = kt.write_set(tmp_path, labels, records)
  lab = kitti.read_labels(os.path.join(kitti_dir, 'label_2'), ids)
  dev = 'cuda:%d' % gpu_device
  tight = kitti.evaluate_device(*stacked(records), kt.CLASS_NAMES, lab, device=dev)
  wide = kitti.evaluate_device(*stacked(records, 2000), kt.CLASS_NAMES, lab, device=dev)
  assert repr(tight) == repr(wide)


def test_eval_once_writes_the_binarys_stats(tmp_path, gpu_device):
  data, ids, _ = make_kitti(tmp_path)
  flags = sq_eval.parse_flags(['--data_path', str(data), '--image_set', 'val',
                               '--eval_dir', str(tmp_path / 'eval'), '--checkpoint_path',
                               'synthetic', '--net', 'squeezeDet', '--gpu', str(gpu_device)])
  all_boxes, aps, names = sq_eval.eval_once(flags)
  assert aps is not None and len(aps) == 9 and names[0] == 'car_easy'
  res = str(tmp_path / 'eval' / 'detection_files_0')
  got = kt.output_files(res)
  want = ke.run(str(data / 'training' / 'label_2'), res, ids)
  assert got == want
  if os.path.exists(sq_eval.EVAL_TOOL):
    for f in list(os.listdir(res)):
      if f.startswith('stats_'):
        os.remove(os.path.join(res, f))
    assert kt.run_binary(str(data / 'training'), str(data / 'ImageSets' / 'val.txt'), res,
                         len(ids)) == got
  # an unreadable label file: an error naming it, no stats files, APs of 0
  os.remove(data / 'training' / 'label_2' / (ids[1] + '.txt'))
  flags.eval_dir = str(tmp_path / 'eval2')
  _, aps, _ = sq_eval.eval_once(flags)
  assert aps == [0.0] * 9
  assert not any(f.startswith('stats_') for f in os.listdir(tmp_path / 'eval2' / 'detection_files_0'))
  # an empty image set: nothing scored, no stats files, APs of 0
  (data / 'ImageSets' / 'val.txt').write_text('')
  flags.eval_dir = str(tmp_path / 'eval3')
  _, aps, _ = sq_eval.eval_once(flags)
  assert aps == [0.0] * 9
  assert not any(f.startswith('stats_') for f in os.listdir(tmp_path / 'eval3' / 'detection_files_0'))
