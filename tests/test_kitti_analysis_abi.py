"""The detection analysis's C ABI refusals without a device, analyze_device's refusals before any
launch, the layouts against the header, and the analysis kernels compiled with the Makefile's
flags with no spills and no stack frame."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from squeezedet_b200 import _lib, kitti
from test_png_build import CSRC, makefile_flags

KERNELS = ('rank_kernel', 'line_scan_kernel', 'line_kernel')


def lib():
  try:
    return _lib.load()
  except _lib.SqdetError as e:
    pytest.skip(str(e))


def last_error():
  return lib().sqdet_last_error().decode()


def test_scratch_bytes_refusals():
  L = lib()
  assert L.sqdet_kitti_analyze_scratch_bytes(3769, 64, 30000) > 0
  assert (L.sqdet_kitti_analyze_scratch_bytes(10, 64, 1000) -
          L.sqdet_kitti_analyze_scratch_bytes(10, 64, 0)) >= 4000
  for args in ((0, 64, 0), (1 << 27, 64, 0), (1, 0, 0), (1, 1025, 0), (1, 64, -1)):
    assert L.sqdet_kitti_analyze_scratch_bytes(*args) == -1, args
    assert 'sqdet_kitti_analyze_scratch_bytes' in last_error()


def test_analyze_refusals_before_any_launch():
  L = lib()
  buf = C.create_string_buffer(1 << 16)
  p = (C.cast(buf, C.c_void_p).value + 255) & ~255      # aligned, so only the sizes are wrong
  cmap = (C.c_int32 * 3)(0, 1, 2)

  def call(n=2, max_dets=8, dets=p, counts=p, classes=3, class_map=cmap, objs=p, offsets=p,
           n_obj=1, scratch=p, nbytes=1 << 30, out=p, lines=p, cap=4):
    return L.sqdet_kitti_analyze(n, max_dets, dets, counts, classes, class_map, objs, offsets,
                                 n_obj, scratch, nbytes, out, lines, cap, None)

  cases = [(dict(n=0), 'n must be'), (dict(n=1 << 27), 'below 2^27'), (dict(max_dets=0), 'max_dets'),
           (dict(max_dets=1025), 'max_dets'), (dict(n_obj=-1), 'n_objects'),
           (dict(dets=None), 'null'), (dict(counts=None), 'null'), (dict(class_map=None), 'null'),
           (dict(offsets=None), 'null'), (dict(scratch=None), 'null'), (dict(out=None), 'null'),
           (dict(objs=None), 'null'), (dict(classes=0), 'classes'),
           (dict(class_map=(C.c_int32 * 3)(0, 0, 1)), 'same KITTI class'),
           (dict(class_map=(C.c_int32 * 3)(0, 3, 1)), 'class_map'),
           (dict(class_map=(C.c_int32 * 3)(0, -1, 1)), 'car, pedestrian or cyclist'),
           (dict(classes=4, class_map=(C.c_int32 * 4)(0, 1, 2, -1)), 'car, pedestrian or cyclist'),
           (dict(cap=-1), 'line_capacity'), (dict(lines=None), 'line_capacity'),
           (dict(lines=p + 4), 'misaligned'), (dict(scratch=p + 8), '256-byte'),
           (dict(nbytes=16), 'scratch_bytes'),
           (dict(), 'one allocation')]          # host memory, or no device at all
  for kw, msg in cases:
    assert call(**kw) == -1, kw
    assert msg in last_error(), (kw, last_error())
    assert last_error().startswith('sqdet_kitti_analyze'), kw
  # no objects and no lines at all are fine for null objs and lines, up to the device checks
  assert call(objs=None, n_obj=0, lines=None, cap=0) == -1 and 'one allocation' in last_error()


def test_python_refusals_before_any_launch():
  labels = kitti.Labels(np.zeros((0,), kitti.OBJ_DTYPE), np.zeros((2,), np.int64))
  dets = np.zeros((1, 4), _lib.DET_DTYPE)
  for names in (('Car',), ('car', 'car'), ('car', 'pedestrian', 'cyclist', 'van'), ('truck',), ()):
    with pytest.raises(ValueError, match='distinct class names'):
      kitti.analyze_device(dets, [0], names, labels, device='cuda:0')
  with pytest.raises(ValueError, match='CUDA'):
    kitti.analyze_device(dets, [0], ('car',), labels, device='cpu')
  # no images: nothing launched, zero counts, nan shares, no lines
  empty = kitti.Labels(np.zeros((0,), kitti.OBJ_DTYPE), np.zeros((1,), np.int64))
  stats, lines = kitti.analyze_device(np.zeros((0, 64), _lib.DET_DTYPE), [], ('car',), empty,
                                      device='cuda:0')
  assert stats['num of detections'] == stats['num of objects'] == 0.0 and len(lines) == 0
  assert kitti.error_file_text([], ('car',), lines) == ''
  with pytest.raises(ValueError, match='image 1: 1500 records'):
    kitti.analyze_device(np.zeros((2, 2000), _lib.DET_DTYPE), [3, 1500], ('car',),
                         kitti.Labels(empty.objs, np.zeros((3,), np.int64)), device='cuda:0')


def test_layouts_match_the_header():
  assert kitti.LINE_DTYPE.itemsize == 56 and kitti.ANALYSIS_DTYPE.itemsize == 80
  assert kitti.ERROR_TYPES == ('loc', 'cls', 'bg', 'missed')


def test_error_file_text_formats_as_the_reference():
  lines = np.zeros((2,), kitti.LINE_DTYPE)
  lines[0] = (0, 2, 1, 0, -0.04000000000000001, 10.25, 31.75, 2.0, 0.5)
  lines[1] = (1, 3, 0, 0, 0.0, 0.0, 100.0, 100.0, -1.0)
  assert kitti.error_file_text(['a', 'b'], ('car', 'pedestrian'), lines) == (
      'a bg -0.0 10.2 31.8 2.0 pedestrian 0.500\nb missed 0.0 0.0 100.0 100.0 car -1.000\n')


def test_analysis_kernels_do_not_spill():
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
  kernels = {n: v for n, v in report.items() if any(re.search(r'\d' + k, n) for k in KERNELS)}
  assert all(any(re.search(r'\d' + k, n) for n in kernels) for k in KERNELS), sorted(report)
  assert all(v == (0, 0, 0) for v in kernels.values()), kernels
