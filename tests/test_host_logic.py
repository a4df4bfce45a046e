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
MAX_CHUNKS = 32          # conv_tc.cu MAX_CHUNKS: output-channel chunks per conv_tc_kernel launch
MAX_FCHUNKS = 16         # conv_tc.cu tc_fire_plan: 64-wide expand chunks of a one-kernel fire


def tc_pick_nt(couts, kc=32, gather=False):
  """pick_nt (conv_tc.cu): the least-cost output tile of 72 / 64 / 32 / 16 whose chunk count fits
  one launch; None when none fits (the conv is declined).  The 72 tile is a candidate only for the
  ConvDet head: one conv of 65..72 channels, not gather mode, K chunks of 32."""
  head = not gather and kc == 32 and len(couts) == 1 and 64 < couts[0] <= 72
  best = best_cost = None
  for nt in (72, 64, 32, 16):
    if nt == 72 and not head:
      continue
    chunks = sum(-(-c // nt) for c in couts)
    if chunks > MAX_CHUNKS:
      continue
    cost = chunks * (nt + 32)
    if best is None or cost < best_cost:
      best, best_cost = nt, cost
  return best


def tc_conv_variant(Cin, Cout, k, stride, padding):
  """conv_tc_kernel<NT, KC, GATHER> that sqdet_conv2d runs with MATH_TF32X3_TC, or None when the
  shape goes to the SIMT kernel: tc_conv_plan (conv_tc.cu) with tc_conv_eligible and
  plan_common's KC rule."""
  gather = Cin == 3 and k == 3 and stride in (1, 2)
  eligible = stride == 1 and padding == 'SAME' and k in (1, 3) and Cin % 16 == 0 and Cin >= 16
  if not (gather or eligible):
    return None
  kc = 32 if gather or Cin % 32 == 0 else 16
  nt = tc_pick_nt([Cout], kc, gather)
  if nt is None:
    return None
  return nt, kc, gather


def tc_fire_variant(Cin, S, E1, E3):
  """KCI of the fire_tc_kernel<KCI> that sqdet_fire runs with MATH_TF32X3_TC, or None when
  tc_fire_plan (conv_tc.cu) declines and the fire runs as separate convs: it takes a 16-channel
  squeeze over Cin % 16 == 0 channels with at most MAX_FCHUNKS expand chunks of 64."""
  if Cin % 16 or Cin < 16 or S != 16:
    return None
  if -(-E1 // 64) + -(-E3 // 64) > MAX_FCHUNKS:
    return None
  return 32 if Cin % 32 == 0 else 16


ALL_CONV_TC_VARIANTS = {(nt, kc, g) for nt in (64, 32, 16) for kc, g in ((32, True), (32, False),
                                                                        (16, False))}
ALL_CONV_TC_VARIANTS.add((72, 32, False))          # conv_tc_instance: the head tile
# the fire_tc_kernel<KCI> instantiations (tc_fire_plan, conv_tc.cu)
ALL_FIRE_TC_VARIANTS = {32, 16}


def test_gpu_case_tables_reach_every_tc_kernel_variant():
  """The GPU parity tables run every conv_tc_kernel and fire_tc_kernel instantiation, and both
  sides of the chunk limits, by the host rules above."""
  from test_gpu_adversarial import SHAPES
  from test_gpu_fire import FIRE_EDGE_CASES
  from test_gpu_halo_tile import HALO_CONV_CASES, WINDOW_CASE
  from test_gpu_kernels import CONV_CASES
  conv = {tc_conv_variant(Cin, Cout, k, s, pad) for _, _, _, Cin, Cout, k, s, pad in CONV_CASES}
  assert conv - {None} == ALL_CONV_TC_VARIANTS, ALL_CONV_TC_VARIANTS - conv
  # sqdet_conv2d would run a declined shape on the SIMT kernel: every halo-conv case is taken
  for _, _, _, Cin, Cout in HALO_CONV_CASES + [WINDOW_CASE]:
    assert tc_conv_variant(Cin, Cout, 3, 1, 'SAME') is not None, (Cin, Cout)
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
  # both sides of the head-tile rule, each a row of CONV_CASES
  by_cout = {}
  for _, _, _, Cin, Cout, k, s, pad in CONV_CASES:
    by_cout.setdefault((Cout, Cin % 32), set()).add(tc_conv_variant(Cin, Cout, k, s, pad))
  assert (64, 32, False) in by_cout[(64, 0)]
  assert by_cout[(65, 0)] == by_cout[(72, 0)] == {(72, 32, False)}
  assert (72, 32, False) not in by_cout[(73, 0)] and by_cout[(73, 0)] - {None}
  assert by_cout[(72, 16)] == {(64, 16, False)}
  # a head-length reduction (K >= 4608) on the 72 tile among the adversarial shapes
  assert any(tc_conv_variant(Cin, Cout, k, s, 'SAME') == (72, 32, False) and k * k * Cin >= 4608
             for _, _, _, Cin, Cout, k, s in SHAPES)


def test_bound_ratio_and_assert_within_bound():
  """The per-element fp64 bound every stage-isolated and layer check goes through: an exact result
  is 0 even on a zero bar, NaN and a non-zero error on a zero bar are inf, and assert_within_bound
  fails at 1.01x the bar, naming the element, and passes at 0.99x it."""
  from gpu_util import adv_tol, assert_within_bound, bound_ratio
  want = np.array([1.0, 0.0, 2.0, -3.0, 5.0, 0.0])
  bar = np.array([1.0, 0.0, 0.0, 2.0, 4.0, 0.0])
  got = np.array([1.5, 0.0, 2.0, np.nan, 5.0, 1e-30], np.float32)
  assert bound_ratio(got, want, bar).tolist() == [0.5, 0.0, 0.0, np.inf, 0.0, np.inf]
  assert_within_bound(got[1:3], want[1:3], bar[1:3], 1, 'exact results on zero bars')
  with pytest.raises(AssertionError):
    assert_within_bound(got[3:5], want[3:5], bar[3:5], 1, 'a NaN')

  K = 9 * 64
  rng = np.random.default_rng(0)
  want = rng.normal(size=(2, 3, 4, 5))
  bar = rng.uniform(0.5, 2.0, want.shape)
  sign = rng.choice([-1.0, 1.0], want.shape)
  for scale, ok in ((0.99, True), (1.01, False)):
    got = want + sign * 0.5 * adv_tol(K) * bar
    got[1, 2, 0, 3] = want[1, 2, 0, 3] + sign[1, 2, 0, 3] * scale * adv_tol(K) * bar[1, 2, 0, 3]
    if ok:
      assert_within_bound(got, want, bar, K, 'at 0.99x')
    else:
      with pytest.raises(AssertionError, match=r'\(1, 2, 0, 3\)'):
        assert_within_bound(got, want, bar, K, 'at 1.01x')


# ---- branches of the other kernels, restated from their launchers -------------------------------
def maxpool_branch(C, size, stride, offset=0):
  """launch_maxpool (pool.cu): float4 kernels need C % 4 == 0 and 16-byte aligned x and y; the
  stride-2 2x2 / 3x3 windows have their own kernel, any other window the generic one."""
  if C % 4 or offset % 4:
    return 'scalar, C % 4' if C % 4 else 'scalar, misaligned'
  if stride == 2 and size in (2, 3):
    return 's2<%d>' % size
  return 'generic vec4'


def add_relu_branch(n, aligned):
  """launch_add_relu / add_relu_kernel (pool.cu): n // 4 float4s when a, b and y are 16-byte
  aligned, then a scalar tail of n % 4; unaligned pointers run all n in the tail loop."""
  if not aligned:
    return 'unaligned'
  return 'vector + tail' if n % 4 else 'vector'


FILTER_THREADS, FILTER_KCACHE, FILTER_CAP = 1024, 24, 1024     # postproc.cu FT, KCACHE, FCAP


def filter_branch(A, top_n, n_above, max_dets):
  """filter_kernel (postproc.cu): the top-n branch when 0 < top_n < A, its scores cached in
  registers while ceil(A / FT) <= KCACHE; else the threshold branch, which reports an overflow
  past min(FCAP, max_dets) records."""
  if 0 < top_n < A:
    per = -(-A // FILTER_THREADS)
    return 'top-n cached' if per <= FILTER_KCACHE else 'top-n uncached'
  return 'threshold overflow' if n_above > min(FILTER_CAP, max_dets) else 'threshold'


def test_gpu_case_tables_reach_every_pool_add_relu_filter_branch():
  """The GPU tables run every branch of the max-pool, add+ReLU and filter launchers, by the host
  rules above, and both sides of the filter's register cache."""
  import test_gpu_branches as br
  from test_gpu_kernels import MAXPOOL_CASES, MAXPOOL_MISALIGNED_CASES
  pool = {maxpool_branch(shape[3], k, s) for shape, k, s, _ in MAXPOOL_CASES}
  pool |= {maxpool_branch(shape[3], k, s, off) for shape, k, s, _, off in MAXPOOL_MISALIGNED_CASES}
  assert pool == {'s2<3>', 's2<2>', 'generic vec4', 'scalar, C % 4', 'scalar, misaligned'}, pool
  # the generic kernel grid-strides past 16 waves of 8 CTAs of 256 threads on a 132-SM H100
  assert any(maxpool_branch(sh[3], k, s) == 'generic vec4' and
             sh[0] * sh[1] * sh[2] * sh[3] // 4 > 132 * 8 * 16 * 256
             for sh, k, s, _ in MAXPOOL_CASES)
  add = {add_relu_branch(B * H * W * br.ADD_RELU_CHANNELS[body], off is None or off % 4 == 0)
         for body, B, H, W, off in br.ADD_RELU_CASES}
  assert add == {'vector', 'vector + tail', 'unaligned'}, add
  assert any(body == 'image' and off is not None for body, _, _, _, off in br.ADD_RELU_CASES)
  filt = {}
  for A, top_n, n_above, max_dets, _, _ in br.FILTER_CASES:
    if max_dets is None:
      max_dets = top_n if 0 < top_n < A else min(A, 1024)
    filt.setdefault(filter_branch(A, top_n, n_above, max_dets), []).append((A, top_n, n_above))
  assert set(filt) == {'top-n cached', 'top-n uncached', 'threshold', 'threshold overflow'}
  cases = [c[:3] for c in br.FILTER_CASES]
  assert (24576, 64, None) in filt['top-n cached'] and (24577, 64, None) in filt['top-n uncached']
  assert {1, 64, 513, 1024} <= {t for _, t, _ in cases}
  assert any(t == A - 1 for A, t, _ in cases)
  assert (3000, 0, 1024) in filt['threshold'] and (3000, 0, 1025) in filt['threshold overflow']
  assert (3000, 0, 100) in filt['threshold'] and (3000, 0, 101) in filt['threshold overflow']
  assert any(c[5] for c in br.FILTER_CASES)                        # class ids == classes


def conv_pool_classes(cout, k, cpad, ppad, bn, height, width):
  """What one first-layer row reaches in conv_pool_simt_kernel (conv_pool_simt.cu): the pooled
  size and its remainders against the 4 x 16 pooled tile (PT_H, PT_W), and the instance
  conv_pool_instance picks (64 threads per 16 channels, NT = 384 above 256 threads)."""
  import oracle
  hc = oracle.conv_geometry(height, k, 2, cpad)[0]
  wc = oracle.conv_geometry(width, k, 2, cpad)[0]
  hp = oracle.conv_geometry(hc, 3, 2, ppad)[0]
  wp = oracle.conv_geometry(wc, 3, 2, ppad)[0]
  return dict(hp=hp, wp=wp, pt_h=hp % 4, pt_w=wp % 16, instance=(k, 4 * cout > 256))


def test_first_layer_table_reaches_every_class():
  """The fused first-layer table of test_gpu_layer_bounds reaches, across its rows: both parities
  of H and W, every pooled height mod 4 and pooled widths with and without a ragged 16-column
  tile, a single pooled pixel, an image smaller than one pooled tile both ways, every ksize x
  conv padding x pool padding, all four kernel instances, and the BN epilogue."""
  from test_gpu_layer_bounds import FIRST_LAYER_ROWS
  rows = [(r, conv_pool_classes(*r)) for r in FIRST_LAYER_ROWS]
  assert {r[5] % 2 for r, _ in rows} == {0, 1} and {r[6] % 2 for r, _ in rows} == {0, 1}
  assert {c['pt_h'] for _, c in rows} == {0, 1, 2, 3}
  assert {c['pt_w'] == 0 for _, c in rows} == {True, False}
  assert any(c['hp'] == c['wp'] == 1 for _, c in rows)
  assert any(c['hp'] < 4 and c['wp'] < 16 and (c['hp'], c['wp']) != (1, 1) for _, c in rows)
  assert {(r[1], r[2], r[3]) for r, _ in rows} == {(k, cp, pp) for k in (3, 7)
                                                     for cp in ('SAME', 'VALID')
                                                     for pp in ('SAME', 'VALID')}
  assert {c['instance'] for _, c in rows} == {(k, wide) for k in (3, 7) for wide in (False, True)}
  assert all(16 <= r[0] <= 96 and r[0] % 16 == 0 for r, _ in rows)     # all fused
  assert any(r[4] for r, _ in rows)
  assert all(r[2] == 'SAME' for r, _ in rows if r[4])                   # _conv_bn_layer: SAME only
  assert all(c['hp'] >= 1 and c['wp'] >= 1 for _, c in rows)


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
