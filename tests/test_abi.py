"""The C-ABI library loads without a GPU and exports every symbol that
include/sqdet_b200.h declares; the ctypes table covers exactly that set; and without
a device the product path fails loudly (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

from squeezedet_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
  names = set()
  inc = os.path.join(ROOT, 'include')
  for fn in os.listdir(inc):
    if fn.endswith('.h'):
      src = open(os.path.join(inc, fn)).read()
      src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
      names |= set(re.findall(r'\b(sqdet_[a-z0-9_]+)\s*\(', src))
  return names


def test_library_exports_every_declared_symbol():
  lib = ctypes.CDLL(_lib.LIB_PATH)
  declared = _declared_symbols()
  assert len(declared) >= 30
  for name in sorted(declared):
    assert hasattr(lib, name), 'missing export: ' + name


def test_ctypes_table_matches_header():
  assert set(_lib.SIGNATURES) == _declared_symbols()


def test_struct_layouts():
  assert ctypes.sizeof(_lib.Det) == 28
  assert _lib.DET_DTYPE.itemsize == 28
  assert ctypes.sizeof(_lib.Config) == 12 * 4


def test_no_cpu_fallback_without_device():
  lib = _lib.load()
  if lib.sqdet_device_count() > 0:
    pytest.skip('a GPU is visible; the no-device behaviour is checked on CPU boxes')
  from squeezedet_b200.config import kitti_squeezeDet_config
  from squeezedet_b200.nets import SqueezeDet
  with pytest.raises(_lib.SqdetError) as ei:
    SqueezeDet(kitti_squeezeDet_config())
  assert 'no CPU fallback' in str(ei.value) or 'CUDA' in str(ei.value)


def test_argument_validation_needs_no_gpu():
  lib = _lib.load()
  h = ctypes.c_void_p()
  assert lib.sqdet_create(None, 0, ctypes.byref(h)) == -1
  assert b'null' in lib.sqdet_last_error()
  cfg = _lib.Config(batch_size=0, image_height=8, image_width=8, classes=3,
                    anchors_per_grid=9, top_n_detection=64, math_mode=0)
  assert lib.sqdet_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == -1
  # stage-isolated entry points reject null pointers before touching the device
  assert lib.sqdet_maxpool_nhwc(None, None, 1, 4, 4, 4, 3, 2, 0, None) == -1
  assert lib.sqdet_topk_nms(None, None, None, 1, 8, 3, 64, 0.005, 0.4, None, None, 64, None) == -1


def test_conv_epilogue_validation_needs_no_gpu():
  """sqdet_conv2d (both math modes) rejects a channel window outside
  [0, y_cstride) and a scale without a shift (or the reverse) before any device work: on a box
  with no device that is SQDET_ERR_INVALID_ARG, not a CUDA error.  The pointers are never
  dereferenced, so the test only runs where no device could be handed them."""
  lib = _lib.load()
  if lib.sqdet_device_count() > 0:
    pytest.skip('a GPU is visible; the no-device behaviour is checked on CPU boxes')
  p = ctypes.c_void_p(4096)
  B, H, W, Cin, Cout = 1, 12, 20, 32, 72        # a shape the tensor-core path plans
  bad = [(72, 1, None, None), (80, -1, None, None), (71, 0, None, None),
         (72, 0, p, None), (72, 0, None, p)]
  for cs, coff, sc, sh in bad:
    for mode in (_lib.MATH_FP32_SIMT, _lib.MATH_TF32X3_TC):
      assert lib.sqdet_conv2d(p, p, p, sc, sh, p, B, H, W, Cin, Cout, 3, 1, 0, 1, cs, coff, mode,
                              None) == -1, (cs, coff, sc, sh, mode)


def test_padding_code():
  assert _lib.pad_code('same') == 0 and _lib.pad_code('VALID') == 1
  with pytest.raises(ValueError):
    _lib.pad_code('full')
