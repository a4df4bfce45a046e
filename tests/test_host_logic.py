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


# ---- tensor-core kernel selection, restated from squeezedet_b200/csrc/conv_tc.cu --------------
MAX_CHUNKS = 32          # conv_tc.cu:49   output-channel chunks per conv_tc_kernel launch
MAX_FCHUNKS = 16         # conv_tc.cu:332  64-wide expand chunks per fire_tc_kernel launch


def tc_pick_nt(couts):
  """pick_nt (conv_tc.cu:552-563): the narrowest-cost output tile of 64 / 32 / 16 whose chunk
  count fits one launch; None when none fits (the conv is declined)."""
  best = best_cost = None
  for nt in (64, 32, 16):
    chunks = sum(-(-c // nt) for c in couts)
    if chunks > MAX_CHUNKS:
      continue
    cost = chunks * (nt + 32)
    if best is None or cost < best_cost:
      best, best_cost = nt, cost
  return best


def tc_conv_variant(Cin, Cout, k, stride, padding):
  """conv_tc_kernel<NT, KC, GATHER> that sqdet_conv2d runs with MATH_TF32X3_TC, or None when the
  shape goes to the SIMT kernel: tc_conv_plan (conv_tc.cu:700-711) with tc_conv_eligible
  (conv_tc.cu:694-698) and plan_common's KC rule (conv_tc.cu:581-583)."""
  gather = Cin == 3 and k == 3 and stride in (1, 2)
  eligible = stride == 1 and padding == 'SAME' and k in (1, 3) and Cin % 16 == 0 and Cin >= 16
  if not (gather or eligible):
    return None
  nt = tc_pick_nt([Cout])
  if nt is None:
    return None
  return nt, 32 if gather or Cin % 32 == 0 else 16, gather


def tc_fire_variant(Cin, S, E1, E3):
  """fire_tc_kernel<KCI, SQN, KCE> that sqdet_fire runs with MATH_TF32X3_TC, or None when
  tc_fused_fire_plan declines (conv_tc.cu:798-806) and the fire runs as separate convs."""
  if Cin % 16 or Cin < 16 or S % 16 or not 16 <= S <= 64:
    return None
  if -(-E1 // 64) + -(-E3 // 64) > MAX_FCHUNKS:
    return None
  return (32 if Cin % 32 == 0 else 16, 16 if S <= 16 else 32 if S <= 32 else 64,
          32 if S % 32 == 0 else 16)


ALL_CONV_TC_VARIANTS = {(nt, kc, g) for nt in (64, 32, 16) for kc, g in ((32, True), (32, False),
                                                                        (16, False))}
# fire_tc_instance (conv_tc.cu:512-523)
ALL_FIRE_TC_VARIANTS = {(32, 16, 16), (32, 32, 32), (32, 64, 16), (32, 64, 32),
                        (16, 16, 16), (16, 32, 32), (16, 64, 16), (16, 64, 32)}


def test_gpu_case_tables_reach_every_tc_kernel_variant():
  """The GPU parity tables run every conv_tc_kernel and fire_tc_kernel instantiation, and both
  sides of the chunk limits, by the host rules above."""
  from test_gpu_adversarial import SHAPES
  from test_gpu_fire import FIRE_EDGE_CASES
  from test_gpu_kernels import CONV_CASES
  conv = {tc_conv_variant(Cin, Cout, k, s, pad) for _, _, _, Cin, Cout, k, s, pad in CONV_CASES}
  assert conv - {None} == ALL_CONV_TC_VARIANTS, ALL_CONV_TC_VARIANTS - conv
  adv = {tc_conv_variant(Cin, Cout, k, s, 'SAME') for _, _, _, Cin, Cout, k, s in SHAPES}
  assert {(16, False), (32, True)} <= {(kc, g) for _, kc, g in adv - {None}}
  assert any(v is not None and v[:2] == (32, 16) for v in adv)     # NT = 32 with KC = 16
  fire = {tc_fire_variant(*shape) for shape, _ in FIRE_EDGE_CASES}
  assert fire - {None} == ALL_FIRE_TC_VARIANTS, ALL_FIRE_TC_VARIANTS - fire
  # chunk limits: a 2048-wide 1x1 is 32 chunks of 64 on wgmma, 2049 falls back to SIMT; a fire
  # with 16 expand chunks is one kernel, 17 fall back
  assert tc_conv_variant(32, 2048, 1, 1, 'SAME') == (64, 32, False)
  assert tc_conv_variant(32, 2049, 1, 1, 'SAME') is None
  assert (1, 3, 5, 32, 2048, 1, 1, 'SAME') in CONV_CASES
  assert (1, 3, 5, 32, 2049, 1, 1, 'SAME') in CONV_CASES
  shapes = [s for s, _ in FIRE_EDGE_CASES]
  assert (64, 16, 512, 512) in shapes and tc_fire_variant(64, 16, 512, 512) is not None
  assert (64, 16, 576, 512) in shapes and tc_fire_variant(64, 16, 576, 512) is None


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
