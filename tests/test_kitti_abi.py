"""The KITTI scorer's C ABI refusals without a device, read_labels' refusals, and kitti_eval.cu
compiled with the Makefile's flags to kernels with no spills and no stack frame."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from squeezedet_b200 import _lib, kitti
from test_png_build import CSRC, makefile_flags

KERNELS = ('prepare_kernel', 'recall_kernel', 'threshold_kernel', 'pr_kernel', 'sum_kernel')


def lib():
  try:
    return _lib.load()
  except _lib.SqdetError as e:
    pytest.skip(str(e))


def last_error():
  return lib().sqdet_last_error().decode()


def test_scratch_bytes_refusals():
  L = lib()
  assert L.sqdet_kitti_eval_scratch_bytes(3769, 64, 30000) > 0
  for args in ((0, 64, 0), (-1, 64, 0), (1, 0, 0), (1, 1025, 0), (1, 64, -1)):
    assert L.sqdet_kitti_eval_scratch_bytes(*args) == -1, args
    assert 'sqdet_kitti_eval_scratch_bytes' in last_error()


def test_eval_refusals_before_any_launch():
  L = lib()
  buf = C.create_string_buffer(1 << 16)
  p = (C.cast(buf, C.c_void_p).value + 255) & ~255      # aligned, so only the sizes are wrong
  cmap = (C.c_int32 * 3)(0, 1, 2)

  def call(n=2, max_dets=8, dets=p, counts=p, classes=3, class_map=cmap, objs=p, offsets=p,
           n_obj=1, scratch=p, nbytes=1 << 30, out=p):
    return L.sqdet_kitti_eval(n, max_dets, dets, counts, classes, class_map, objs, offsets, n_obj,
                              scratch, nbytes, out, None)

  cases = [(dict(n=0), 'n must be'), (dict(max_dets=0), 'max_dets'), (dict(max_dets=1025), 'max_dets'),
           (dict(n_obj=-1), 'n_objects'), (dict(dets=None), 'null'), (dict(counts=None), 'null'),
           (dict(class_map=None), 'null'), (dict(offsets=None), 'null'), (dict(scratch=None), 'null'),
           (dict(out=None), 'null'), (dict(objs=None), 'null'), (dict(classes=0), 'classes'),
           (dict(classes=65), 'classes'),
           (dict(class_map=(C.c_int32 * 3)(0, 0, 1)), 'same KITTI class'),
           (dict(class_map=(C.c_int32 * 3)(0, 3, 1)), 'class_map'),
           (dict(nbytes=16), 'scratch_bytes'),
           (dict(), 'one allocation')]          # host memory, or no device at all
  for kw, msg in cases:
    assert call(**kw) == _lib.SqdetError(-1, '').code == -1, kw
    assert msg in last_error(), (kw, last_error())
  # no objects at all is fine for objs = NULL, up to the device checks
  assert call(objs=None, n_obj=0) == -1 and 'one allocation' in last_error()


def test_python_refusals_without_device():
  labels = kitti.Labels(np.zeros((0,), kitti.OBJ_DTYPE), np.zeros((2,), np.int64))
  dets = np.zeros((1, 4), _lib.DET_DTYPE)
  with pytest.raises(ValueError, match='same KITTI class'):
    kitti.evaluate_device(dets, [0], ('car', 'Car'), labels, device='cuda:0')
  with pytest.raises(ValueError, match='CUDA'):
    kitti.evaluate_device(dets, [0], ('car',), labels, device='cpu')
  # no images: nothing to score and no class, as evaluate_object writes no stats for an empty set
  empty = kitti.Labels(np.zeros((0,), kitti.OBJ_DTYPE), np.zeros((1,), np.int64))
  assert kitti.evaluate_device(np.zeros((0, 64), _lib.DET_DTYPE), [], ('car',), empty,
                               device='cuda:0') == {}
  # a capacity above 1024 with an image holding more than 1024 records
  with pytest.raises(ValueError, match='image 1: 1500 records'):
    kitti.evaluate_device(np.zeros((2, 2000), _lib.DET_DTYPE), [3, 1500], ('car',),
                          kitti.Labels(empty.objs, np.zeros((3,), np.int64)), device='cuda:0')


def test_result_layout_matches_the_header():
  assert kitti.RESULT_DTYPE.itemsize == 7472      # 9 * 41 doubles, 3 * 9 * 41 + 9 + 9 + 3 + 2 int32
  assert kitti.RESULT_DTYPE.itemsize % 8 == 0


def test_read_labels(tmp_path):
  (tmp_path / 'a.txt').write_text(
      'Car 0.00 0 -1.57 1.00 2.00 3.00 4.00 1 1 1 1 1 1 1\n\nDontCare -1 -1 -10 5 6 7 8 -1 -1 -1 '
      '-1000 -1000 -1000 -10\nperson_SITTING 0.5 2 0.0 1 2 3 4 0 0 0 0 0 0 0\n')
  (tmp_path / 'b.txt').write_text('')
  lab = kitti.read_labels(str(tmp_path), ['a', 'b', 'a'])
  assert len(lab) == 3 and lab.offsets.tolist() == [0, 3, 3, 6]
  assert lab.objs['type'].tolist() == [0, 5, 4] * 2
  assert lab.objs['occlusion'].tolist()[:3] == [0, -1, 2]
  assert lab.objs['aos_term'][2] == 1.0 and lab.objs['aos_term'][0] == (1 + np.cos(-1.57)) / 2
  (tmp_path / 'c.txt').write_text('Car 0.00 0 -1.57 1 2 3 4 1 1 1 1 1 1 1\nCar 0 0 1 2 3 4\n')
  with pytest.raises(ValueError, match=r'c\.txt:2'):
    kitti.read_labels(str(tmp_path), ['a', 'c'])
  (tmp_path / 'd.txt').write_text('Car 0.00 0.5 -1.57 1 2 3 4 1 1 1 1 1 1 1\n')
  with pytest.raises(ValueError, match=r'd\.txt:1'):
    kitti.read_labels(str(tmp_path), ['d'])
  with pytest.raises(FileNotFoundError, match='missing'):
    kitti.read_labels(str(tmp_path), ['a', 'missing'])


def test_kitti_kernels_do_not_spill():
  nvcc, flags = makefile_flags()
  with tempfile.TemporaryDirectory() as tmp:
    r = subprocess.run([nvcc] + flags + ['-Xptxas', '-v', '-c', 'kitti_eval.cu', '-o',
                                         os.path.join(tmp, 'kitti_eval.o')],
                       cwd=CSRC, capture_output=True, text=True, check=True)
  report = {}
  name = None
  for line in r.stderr.splitlines():
    m = re.search(r"Function properties for (\S+)", line)
    if m:
      name = m.group(1)
    m = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
    if m and name:
      report[name] = tuple(int(v) for v in m.groups())
      name = None
  kernels = {n: v for n, v in report.items() if any(k in n for k in KERNELS)}
  assert all(any(k in n for n in kernels) for k in KERNELS), sorted(report)
  assert all(v == (0, 0, 0) for v in kernels.values()), kernels
