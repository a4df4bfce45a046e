"""More than one device: (1) two engines on two devices of ONE process (the per-device opt-in of
the >48 KB dynamic shared memory); (2) N ranks, NCCL all-gather captured in the forward graph:
the gathered records are byte-equal to a 1-rank run of the same global batch.
Both skip on a machine with fewer than 2 visible GPUs."""
import os
import subprocess
import sys

import numpy as np
import pytest

from squeezedet_b200 import _lib
from squeezedet_b200.utils import synth
from gpu_util import make_net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def need_gpus(n):
  have = _lib.device_count()
  if have < n:
    pytest.skip('needs %d GPUs, %d visible' % (n, have))


def test_two_devices_one_process():
  need_gpus(2)
  imgs = synth.synthetic_images(2, 96, 320, seed=4)
  outs = []
  for dev in (0, 1):
    m, _ = make_net('squeezeDet', 320, 96, 2, dev, seed=8)
    outs.append((m, m.detect(imgs)))
  (m0, (b0, p0, c0)), (m1, (b1, p1, c1)) = outs
  assert np.array_equal(p0, p1) and np.array_equal(b0, b1) and np.array_equal(c0, c1)
  # and again on device 0 after device 1 was used (device guard restores the context)
  b2, p2, c2 = m0.detect(imgs)
  assert np.array_equal(p0, p2)


@pytest.mark.parametrize('world,global_batch', [(2, 5), (2, 4)])
def test_nccl_gather_in_graph_matches_single_rank(world, global_batch, tmp_path):
  need_gpus(world)
  port = 29600 + (os.getpid() % 300)
  env = dict(os.environ, OUT_DIR=str(tmp_path), GLOBAL_BATCH=str(global_batch))
  cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1',
         '--nproc-per-node', str(world), '--master-addr', '127.0.0.1', '--master-port',
         str(port), os.path.join(ROOT, 'tests', 'nccl_worker.py')]
  r = subprocess.run(cmd, env=env, cwd=ROOT, timeout=600, capture_output=True, text=True)
  errs = ''.join(open(tmp_path / f).read() for f in sorted(os.listdir(tmp_path)) if f.startswith('err_rank'))
  assert r.returncode == 0, errs[-3000:] + r.stdout[-1000:] + r.stderr[-1000:]
  a = np.load(tmp_path / 'rank0.npz')
  b = np.load(tmp_path / 'rank1.npz')
  assert np.array_equal(a['dets'], b['dets']) and np.array_equal(a['counts'], b['counts'])
  assert 'byte-equal True' in r.stdout
