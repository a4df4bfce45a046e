import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
  config.addinivalue_line('markers', 'gpu: needs an H100 (run with -m gpu on a GPU machine)')


@pytest.fixture(scope='session')
def postproc_kat():
  z = np.load(os.path.join(GOLDEN, 'postproc_kat.npz'))
  meta = json.loads(bytes(z['meta_json']).decode())
  cases = []
  for i, m in enumerate(meta):
    c = dict(m)
    for k in ('boxes', 'probs', 'cls', 'out_boxes', 'out_probs', 'out_cls', 'nms_keep'):
      c[k] = z['c%d_%s' % (i, k)]
    cases.append(c)
  return dict(cases=cases, iou_boxes=z['iou_boxes'], iou_out=z['iou_out'])


@pytest.fixture(scope='session')
def anchors_golden():
  with open(os.path.join(GOLDEN, 'anchors.json')) as f:
    return json.load(f)


@pytest.fixture(scope='session')
def gpu_device():
  """Device index for GPU tests; fails loudly (never skips to a CPU path)."""
  from squeezedet_b200 import _lib
  n = _lib.device_count()
  assert n > 0, 'GPU test selected but no CUDA device is visible'
  return 0
