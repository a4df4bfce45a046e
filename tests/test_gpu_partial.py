"""Partial batches: an engine built for B images running n < B of them (sqdet_forward_n,
sqdet_submit_frames_n, eval.py --batch_size).  A short batch runs the kernels planned for B on
smaller grids, so image i of an n-image forward must be bitwise identical to image i of a full
forward over the same first n images; nothing at or past image n is read or written, except that
counts[n, B) are set to 0."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
from squeezedet_b200 import _lib, eval as sq_eval
from squeezedet_b200 import config as cfg
from squeezedet_b200.nets import SqueezeDet
from squeezedet_b200.utils import synth, viz
from squeezedet_b200.utils.util import bbox_transform
from gpu_util import (MODES, RESULTS, TOL, assert_fused_away, assert_rows_equal, build,
                      fetch_results, fire_tiles, forward_n, make_kitti, make_net, oracle_pipeline)

pytestmark = pytest.mark.gpu
ERR_INVALID_ARG = -1


def fill_results(model, device, byte=0xff):
  res = model.results_device()
  for key, arr in fetch_results(model, device).items():
    fill = np.full(arr.nbytes, byte, np.uint8)
    _lib.check(model._lib.sqdet_memcpy_h2d(res[key], fill.ctypes.data, fill.nbytes, None))
  _lib.check(model._lib.sqdet_stream_sync(device, None))


def activations(model):
  """Every materialised activation of the last forward (tensor 0, the engine's own input buffer,
  is not written by forward_device)."""
  out = {}
  for name, t in model._tensors.items():
    if t.id is None or t.id == 0:
      continue
    try:
      out[name] = model.read_tensor(t)
    except _lib.SqdetError as exc:
      assert exc.code == -5, exc              # fused into its consumer
  return out


def assert_rows_match(got, want, n):
  """Rows [0, n) bitwise equal (records up to each image's count); rows [n, B) untouched since
  fill_results (0xff bytes), except counts, which are 0."""
  for key, _, _ in RESULTS:
    assert got[key][:n].tobytes() == want[key][:n].tobytes(), (key, n)
    assert (got[key][n:].view(np.uint8) == 0xff).all(), (key, n)
  assert np.array_equal(got['counts'][:n], want['counts'][:n]), n
  assert (got['counts'][n:] == 0).all(), got['counts']
  for i in range(n):
    c = int(want['counts'][i])
    assert got['dets'][i][:c].tobytes() == want['dets'][i][:c].tobytes(), (i, n)
  assert (got['dets'][n:].view(np.uint8) == 0xff).all(), n


def check_partial_rows(model, images, other, device, stream_for):
  """Full forward of `images`; then n = 1 .. B-1 on buffers of n images, rows against the full
  forward; then `other` at n = 1, after which every activation's rows >= 1 still hold `images`'
  values.  stream_for(n): the stream of the n-image forward (None = legacy, not graph-captured)."""
  B = images.shape[0]
  forward_n(model, images, None, model.engine_stream())
  want = fetch_results(model, device)
  acts = activations(model)
  assert acts
  for n in range(1, B):
    fill_results(model, device)
    forward_n(model, images, n, stream_for(n))
    assert_rows_match(fetch_results(model, device), want, n)
    assert_rows_equal(activations(model), acts, n)
  forward_n(model, other, 1, model.engine_stream())
  for name, a in activations(model).items():
    assert a[1:].tobytes() == acts[name][1:].tobytes(), name
  return want


@pytest.mark.parametrize('math_mode', MODES)
@pytest.mark.parametrize('net,width,height', [
    ('squeezeDet', 208, 112), ('squeezeDet+', 215, 119), ('vgg16', 96, 64),
    ('resnet50', 131, 99)])
def test_forward_n_rows_bitwise(net, width, height, math_mode, gpu_device):
  model, _ = make_net(net, width, height, 3, gpu_device, math_mode, seed=3)
  x = synth.synthetic_images(3, height, width, seed=9)
  y = synth.synthetic_images(3, height, width, seed=10)
  # n = 1 on the legacy stream (launched directly), n = 2 on the engine stream (CUDA graph)
  want = check_partial_rows(model, x, y, gpu_device,
                            lambda n: None if n == 1 else model.engine_stream())
  assert want['counts'].min() >= 0


def test_forward_n_one_kernel_fire_below_its_threshold(gpu_device):
  """B = 3 images of 64 x 352 give the fire 3 x 176 = 528 tiles: one kernel (>= 4 tiles per SM on
  both H100 variants).  At n = 1 and 2 the grid (176, 352 tiles) is below the threshold of either
  variant, and the fire still runs as that one kernel, bitwise equal to the full batch."""
  batch, height, width = 3, 64, 352
  body = [('conv', 'conv1', 32, 3, 1, 'SAME'), ('fire', 'fire2', 16, 64, 64),
          ('pool', 'pool2', 3, 2, 'SAME')]
  assert fire_tiles(batch, height, width) >= 4 * 132
  assert fire_tiles(batch - 1, height, width) < 4 * 114
  _, model, _ = build(body, batch, height, width, _lib.MATH_TF32X3_TC, gpu_device)
  # conv1 + fire2 (one kernel) + pool2 + head + interpret + filter
  assert model.launches_per_forward() == 6
  x = synth.synthetic_images(batch, height, width, seed=11)
  y = synth.synthetic_images(batch, height, width, seed=12)
  check_partial_rows(model, x, y, gpu_device, lambda n: model.engine_stream())
  assert_fused_away(model, 'fire2/squeeze1x1')
  assert model.launches_per_forward() == 6


def submit_n(model, frames, rescale, dets, counts):
  n = len(frames)
  ptrs = (C.c_void_p * n)(*[f.ctypes.data for f in frames])
  hs = (C.c_int32 * n)(*[f.shape[0] for f in frames])
  ws = (C.c_int32 * n)(*[f.shape[1] for f in frames])
  return model._lib.sqdet_submit_frames_n(model._engine, n, ptrs, hs, ws, 1, int(rescale),
                                          dets.ctypes.data, counts.ctypes.data)


def test_submit_frames_n_pipeline(gpu_device):
  """n = B, 1, B, 2 with two submits in flight and rescale alternating: each result equals the
  same frames submitted alone, only n rows come back, and the device counts past n are 0."""
  B = 3
  m, _ = make_net('squeezeDet', 320, 96, B, gpu_device, seed=8)
  rng = np.random.default_rng(4)
  sizes = [(96, 320), (120, 400), (80, 300)]
  plan = [(B, True), (1, False), (B, False), (2, True)]
  subs = [[rng.integers(0, 256, sizes[(j + i) % 3] + (3,), dtype=np.uint8) for j in range(n)]
          for i, (n, _) in enumerate(plan)]
  alone = [m.detect_frames(f, order='eval', rescale=r) for f, (_, r) in zip(subs, plan)]
  assert all(d.shape == (len(f), m.max_dets) and c.shape == (len(f),)
             for f, (d, c) in zip(subs, alone))
  # pinned result buffers: a copy into pageable memory would make each submit wait for its forward
  pinned = [(_lib.PinnedArray((B, m.max_dets), _lib.DET_DTYPE), _lib.PinnedArray((B,), np.int32))
            for _ in plan]
  outs = [(pd.array, pc.array) for pd, pc in pinned]
  for d, c in outs:
    d.view(np.uint8)[...] = 0
    c[...] = -7
  for i, (frames, (_, rescale)) in enumerate(zip(subs, plan)):
    _lib.check(submit_n(m, frames, rescale, *outs[i]))
    if i >= 1:
      m.wait()
  m.wait()
  for frames, (d, c), (wd, wc) in zip(subs, outs, alone):
    n = len(frames)
    assert np.array_equal(c[:n], wc), (c, wc)
    assert (c[n:] == -7).all()                 # only n counts copied back
    for i in range(n):
      assert d[i][:wc[i]].tobytes() == wd[i][:wc[i]].tobytes()
  res = fetch_results(m, gpu_device)
  assert (res['counts'][2:] == 0).all() and np.array_equal(res['counts'][:2], alone[-1][1])
  # n = 0 and n = B + 1 are refused before anything is queued (nothing in flight afterwards)
  d, c = np.zeros((B + 1, m.max_dets), _lib.DET_DTYPE), np.zeros((B + 1,), np.int32)
  ptrs = (C.c_void_p * (B + 1))(*[subs[0][0].ctypes.data] * (B + 1))
  hw = (C.c_int32 * (B + 1))(*[96] * (B + 1))
  ww = (C.c_int32 * (B + 1))(*[320] * (B + 1))
  for bad in (0, B + 1):
    assert m._lib.sqdet_submit_frames_n(m._engine, bad, ptrs, hw, ww, 1, 1, d.ctypes.data,
                                        c.ctypes.data) == ERR_INVALID_ARG
  x = _lib.DeviceBuffer.from_numpy(synth.synthetic_images(B, 96, 320, seed=1), gpu_device)
  for bad in (0, B + 1):
    assert m._lib.sqdet_forward_n(m._engine, x.ptr, bad, None) == ERR_INVALID_ARG
  with pytest.raises(_lib.SqdetError):
    m.wait()
  with pytest.raises(ValueError):
    m.detect_frames([])
  with pytest.raises(ValueError):
    m.detect_frames([subs[0][0]] * (B + 1))


def run_eval(data, eval_dir, batch, device):
  flags = sq_eval.parse_flags(['--data_path', str(data), '--image_set', 'val',
                               '--eval_dir', str(eval_dir), '--checkpoint_path', 'synthetic',
                               '--net', 'squeezeDet', '--gpu', str(device),
                               '--batch_size', str(batch)])
  return sq_eval.eval_once(flags)


def test_eval_once_batch_size_2_with_short_tail(tmp_path, gpu_device):
  """Three frames in groups of 2 (a tail of 1): the same oracle checks as the batch-1 eval, and
  the same all_boxes and detection files as --batch_size 1 - identical where both engines run the
  same plan, within the oracle tolerance where they do not (the one-kernel-fire threshold follows
  the SM count, so on a 114-SM H100 the batch-2 plan differs from batch 1)."""
  data, ids, frames = make_kitti(tmp_path)
  boxes1, _, _ = run_eval(data, tmp_path / 'eval1', 1, gpu_device)
  boxes2, aps2, names2 = run_eval(data, tmp_path / 'eval2', 2, gpu_device)
  mc = cfg.kitti_squeezeDet_config()
  weights = synth.synthetic_weights(oracle.param_specs('squeezeDet'), seed=0)
  launches = []
  for b in (1, 2):
    mcb = cfg.kitti_squeezeDet_config()
    mcb.BATCH_SIZE = b
    launches.append(SqueezeDet(mcb, gpu_device).launches_per_forward())
  same_plan = launches[0] == launches[1]
  dirs = [tmp_path / d / 'detection_files_0' / 'data' for d in ('eval1', 'eval2')]
  for i, idx in enumerate(ids):
    fb, fp, fc, near = oracle_pipeline('squeezeDet', mc, weights, frames[idx], 'eval', True)
    lines = (dirs[1] / (idx + '.txt')).read_text().splitlines()
    assert len(lines) == sum(len(boxes2[c][i]) for c in range(mc.CLASSES))
    if same_plan:
      assert (dirs[0] / (idx + '.txt')).read_bytes() == (dirs[1] / (idx + '.txt')).read_bytes()
      assert all(boxes1[c][i] == boxes2[c][i] for c in range(mc.CLASSES)), idx
    if near:
      continue
    want = [[] for _ in range(mc.CLASSES)]
    for c, b, s in zip(fc, fb, fp):
      want[c].append(bbox_transform(b) + [s])
    k = 0
    for c in range(mc.CLASSES):
      assert len(boxes2[c][i]) == len(want[c]) == len(boxes1[c][i]), (idx, c)
      for g, g1, w in zip(boxes2[c][i], boxes1[c][i], want[c]):
        np.testing.assert_allclose(np.asarray(g, np.float64), np.asarray(w, np.float64),
                                   rtol=2 * TOL, atol=2e-2)
        np.testing.assert_allclose(np.asarray(g, np.float64), np.asarray(g1, np.float64),
                                   rtol=2 * TOL, atol=2e-2)
        assert lines[k] == viz.kitti_detection_line(mc.CLASS_NAMES[c], g[:4], g[4]).rstrip('\n')
        k += 1
  if os.path.exists(sq_eval.EVAL_TOOL):       # the scorer ran on the batch-2 detection files
    assert aps2 is not None and len(aps2) == 3 * mc.CLASSES and names2[0] == 'car_easy'
