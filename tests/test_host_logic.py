"""Host-side logic that needs no GPU: config parity with the reference fixtures,
synthetic generators, util helpers, batch sharding + the world_size-2 gloo all-gather."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from squeezedet_b200 import config as cfg
from squeezedet_b200.utils import synth, util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('fn', ['kitti_squeezeDet_config', 'kitti_squeezeDetPlus_config',
                                'kitti_vgg16_config', 'kitti_res50_config'])
def test_config_matches_reference_fixture(fn, anchors_golden):
  mc = getattr(cfg, fn)()
  g = anchors_golden[fn]
  ab = np.ascontiguousarray(mc.ANCHOR_BOX, dtype=np.float64)
  assert hashlib.sha256(ab.tobytes()).hexdigest() == g['sha256']
  assert mc.ANCHORS == g['shape'][0] and mc.ANCHOR_PER_GRID == 9
  assert list(mc.CLASS_NAMES) == g['class_names']
  assert np.asarray(mc.BGR_MEANS).ravel().tolist() == g['bgr_means']
  for k, v in g['scalars'].items():
    assert mc[k] == v, (fn, k, mc[k], v)


def test_set_anchors_after_resize():
  mc = cfg.kitti_squeezeDet_config()
  mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT = 1242, 375
  a = cfg.set_anchors(mc)
  assert a.shape == (16848, 4)
  assert a[0, 0] == 1 * 1242.0 / 79 and a[-1, 1] == 24 * 375.0 / 25


def test_bbox_transforms_roundtrip_grows_by_one():
  box = [np.float32(50.0), np.float32(40.0), np.float32(20.0), np.float32(10.0)]
  back = util.bbox_transform_inv(util.bbox_transform(box))
  assert back == [50.5, 40.5, 21.0, 11.0]          # the reference's +1 (util.py:189-190)


def test_synth_is_deterministic_and_scaled():
  a = synth.synthetic_images(2, 8, 9, seed=5)
  b = synth.synthetic_images(2, 8, 9, seed=5)
  assert a.dtype == np.float32 and a.shape == (2, 8, 9, 3) and np.array_equal(a, b)
  specs = [('conv1/kernels', (3, 3, 3, 64)), ('conv1/biases', (64,)),
           ('fire2/squeeze1x1/kernels', (1, 1, 64, 16)), ('fire2/squeeze1x1/biases', (16,)),
           ('conv12/kernels', (3, 3, 16, 72)), ('conv12/biases', (72,))]
  w = synth.synthetic_weights(specs, seed=3)
  assert set(w) == {n for n, _ in specs}
  assert all(v.dtype == np.float32 for v in w.values())
  assert np.array_equal(w['conv1/kernels'], synth.synthetic_weights(specs, seed=3)['conv1/kernels'])


def test_shard_ranges():
  from squeezedet_b200 import shard
  assert shard.shard_sizes(20, 8) == [3, 3, 3, 3, 2, 2, 2, 2]
  assert shard.shard_sizes(20, 1) == [20]
  assert shard.shard_sizes(5, 8) == [1, 1, 1, 1, 1, 0, 0, 0]
  r = shard.shard_ranges(20, 8)
  assert r[0] == (0, 3) and r[4] == (12, 14) and r[-1] == (18, 20)
  assert sum(b - a for a, b in r) == 20


def test_gloo_world2_allgather_roundtrip(tmp_path):
  """N>1 path on CPU: 2 processes, gloo, 127.0.0.1 — each packs its shard's detection
  blob, one all_gather, both unpack identical global results."""
  script = os.path.join(ROOT, 'tests', 'gloo_worker.py')
  port = 29500 + (os.getpid() % 2000)
  procs = []
  for rank in range(2):
    env = dict(os.environ, RANK=str(rank), WORLD_SIZE='2', LOCAL_RANK=str(rank),
               MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), OUT_DIR=str(tmp_path))
    procs.append(subprocess.Popen([sys.executable, script], env=env, cwd=ROOT))
  for p in procs:
    assert p.wait(timeout=180) == 0
  a = np.load(tmp_path / 'rank0.npz')
  b = np.load(tmp_path / 'rank1.npz')
  assert np.array_equal(a['dets'], b['dets']) and np.array_equal(a['counts'], b['counts'])
  assert a['counts'].tolist() == [2, 0, 5, 1, 3]          # 5 images: shards 3 + 2
  assert a['dets'].shape == (5, 8)
  assert a['dets']['anchor'][2, :5].tolist() == [200, 201, 202, 203, 204]
