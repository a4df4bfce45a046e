"""sqdet_forward_tiles / ModelSkeleton.forward_device_tiles and sqdet_merge_tiles: whole frames run
as tiles, and each frame's detections merged by one top-N and NMS on the GPU.  Every check is
bitwise: the per-tile rows against forward_device_frames_fmt over the tile crops with rescale, the
merged records against oracle.tiles.merge_tiles on the engine's own det_* rows."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from gpu_util import (TableNet, adversarial_rows, assert_merge_matches_oracle, body_grid,
                      fetch_results, merge_gpu)
from squeezedet_b200 import _lib, demo
from squeezedet_b200 import config as cfg
from squeezedet_b200.utils import synth
from squeezedet_b200.utils.util import tile_grid

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_STATE = -1, -4
RESULT_ROWS = ('det_boxes', 'det_probs', 'det_class', 'dets')
BODY = [('conv', 'conv1', 64, 3, 2, 'SAME'), ('pool', 'pool1', 3, 2, 'SAME'),
        ('fire', 'fire2', 16, 64, 64)]
TH, TW = 47, 133                       # the engine's input: tiles of this size run at native scale


def engine(batch, device, top_n=64, prob_thresh=0.005):
  """A SqueezeDet-like engine (conv+pool, fire) at 47 x 133 with the given filter settings."""
  mc = cfg.kitti_squeezeDet_config()
  mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = TW, TH, batch
  mc.TOP_N_DETECTION, mc.PROB_THRESH = top_n, prob_thresh
  mc.GRID_H, mc.GRID_W = body_grid(BODY, TH, TW)
  mc.ANCHOR_BOX = cfg.set_anchors(mc)
  mc.ANCHORS = len(mc.ANCHOR_BOX)
  model = TableNet(mc, BODY, (), device, math_mode=_lib.MATH_TF32X3_TC)
  model.load_weights(synth.synthetic_weights(synth.model_param_specs(model), seed=7))
  return model


def device_frame(fmt, h, w, rng, device):
  """A random h x w frame in `fmt` on the device, in the tensor form the facade takes."""
  if fmt == 'bgr':
    a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
  elif fmt == 'nv12':
    a = rng.integers(0, 256, (3 * h // 2, w), dtype=np.uint8)
  else:
    a = rng.integers(0, 256, (3, h, w), dtype=np.uint8)
  return torch.from_numpy(a).to(device)


def merged(model, n, stream=None):
  return model.tile_results(n, stream)


def by_tile(model, frames, fmt, tiles, order):
  """Every result buffer of forward_device_frames_fmt over the tiles as crops, rescaled."""
  model.forward_device_frames_fmt([frames[t[0]] for t in tiles], fmt,
                                  crops=[t[1:] for t in tiles], order=order, rescale=True)
  torch.cuda.synchronize(model.gpu_id)
  return fetch_results(model, model.gpu_id)


def run_tiles(model, frames, fmt, tiles, order, stream=None):
  model.forward_device_tiles(frames, fmt, tiles, order=order,
                             stream=stream.cuda_stream if stream is not None else None)
  torch.cuda.synchronize(model.gpu_id)
  return fetch_results(model, model.gpu_id), merged(model, len(frames))


def check_case(model, frames, fmt, tiles, order):
  """Rows [0, t) and per-tile records as by_tile, merged records as the oracle, counts of rows
  [n, B) 0."""
  t, n = len(tiles), len(frames)
  want_rows = by_tile(model, frames, fmt, tiles, order)
  got_rows, (dets, counts) = run_tiles(model, frames, fmt, tiles, order)
  for key in RESULT_ROWS:
    assert got_rows[key][:t].tobytes() == want_rows[key][:t].tobytes(), key
  assert np.array_equal(got_rows['counts'][:t], want_rows['counts'][:t])
  want = assert_merge_matches_oracle(dets, counts, {k: v[:t] for k, v in got_rows.items()}, tiles,
                                     n, model.mc)
  B = model.mc.BATCH_SIZE
  all_counts = merged(model, B)[1]
  assert not all_counts[n:].any()
  assert any(len(w[3]) for w in want)
  return got_rows, dets, counts


@pytest.mark.parametrize('fmt', ['bgr', 'nv12', 'rgb_planar'])
@pytest.mark.parametrize('order', ['demo', 'eval'])
def test_grids_with_overview_out_of_order(gpu_device, fmt, order):
  """Two frames of different sizes, each an overlapping tile_grid plus one overview tile of the
  whole frame (resized), the tiles interleaved and shuffled."""
  B = 20
  model = engine(B, gpu_device)
  rng = np.random.default_rng({'bgr': 1, 'nv12': 2, 'rgb_planar': 3}[fmt] + (order == 'eval'))
  sizes = [(120, 300), (94, 200)]
  frames = [device_frame(fmt, h, w, rng, gpu_device) for h, w in sizes]
  tiles = []
  for f, (h, w) in enumerate(sizes):
    tiles += [(f,) + g for g in tile_grid(w, h, TW, TH, 16)]
    tiles.append((f, 0, 0, w, h))
  assert len(tiles) <= B
  tiles = [tiles[i] for i in rng.permutation(len(tiles))]
  check_case(model, frames, fmt, tiles, order)


def test_one_frame_and_one_tile_per_frame(gpu_device):
  """n = 1 (all tiles on one frame, odd offsets) and n = t (one tile per frame, off the origin)."""
  model = engine(6, gpu_device)
  rng = np.random.default_rng(11)
  frame = device_frame('bgr', 101, 211, rng, gpu_device)
  tiles = [(0, 0, 0, TW, TH), (0, 77, 53, TW, TH), (0, 13, 29, 90, 40), (0, 5, 7, 200, 90)]
  check_case(model, [frame], 'bgr', tiles, 'demo')
  frames = [device_frame('nv12', 2 * TH + 2, 2 * TW, rng, gpu_device) for _ in range(6)]
  tiles = [(f, 3 * f, 5 * f, TW + f, TH) for f in range(6)]
  check_case(model, frames, 'nv12', tiles, 'eval')


def test_one_tile_per_frame_at_origin_is_per_tile_records(gpu_device):
  """Adding +0.0 to a box centre changes no bit, so the merge of single whole-frame tiles is the
  per-tile filter."""
  B = 5
  model = engine(B, gpu_device)
  rng = np.random.default_rng(12)
  sizes = [(TH, TW), (60, 150), (30, 90), (47, 300), (200, 133)]
  frames = [device_frame('rgb_planar', h, w, rng, gpu_device) for h, w in sizes]
  tiles = [(f, 0, 0, w, h) for f, (h, w) in enumerate(sizes)]
  rows, dets, counts = check_case(model, frames, 'rgb_planar', tiles, 'eval')
  assert np.array_equal(counts, rows['counts'][:B])
  assert dets.tobytes() == rows['dets'][:B].tobytes()


def test_all_tiles_of_one_frame_exceed_one_table(gpu_device):
  """t = B = 20 tiles of one frame at TOP_N_DETECTION 64: 1280 per-tile candidates, more than
  the 1024 one CTA's table holds."""
  B = 20
  model = engine(B, gpu_device)
  assert model.mc.TOP_N_DETECTION * B > 1024
  rng = np.random.default_rng(13)
  frame = device_frame('bgr', 190, 420, rng, gpu_device)
  xs, ys = rng.integers(0, 420 - TW, B), rng.integers(0, 190 - TH, B)
  tiles = [(0, int(x), int(y), TW, TH) for x, y in zip(xs, ys)]
  check_case(model, [frame], 'bgr', tiles, 'demo')


def test_threshold_branch_and_overflow(gpu_device):
  """TOP_N_DETECTION = 0: PROB_THRESH in union order; more candidates than the table gives
  count -1 and padded records."""
  rng = np.random.default_rng(14)
  frames = [device_frame('bgr', 100, 250, rng, gpu_device) for _ in range(2)]
  tiles = [(0, 0, 0, TW, TH), (1, 50, 20, TW, TH), (0, 117, 53, TW, TH), (1, 0, 0, 250, 100)]
  # the threshold that leaves about 300 candidates in frame 0's union of this input
  probe = engine(4, gpu_device, top_n=0, prob_thresh=0.999)
  rows = by_tile(probe, frames, 'bgr', tiles, 'demo')
  u0 = np.concatenate([rows['det_probs'][0], rows['det_probs'][2]])
  thresh = float(np.sort(u0)[-300])
  for prob_thresh, overflow in [(thresh, False), (0.0, True)]:
    model = engine(4, gpu_device, top_n=0, prob_thresh=prob_thresh)
    assert model.max_dets == 1024
    got, (dets, counts) = run_tiles(model, frames, 'bgr', tiles, 'demo')
    if overflow:
      assert counts.tolist() == [-1, -1]
      assert (dets['anchor'] == -1).all() and (dets['cls'] == -1).all()
      assert not dets['prob'].any() and not dets['cx'].any()
    else:
      assert_merge_matches_oracle(dets, counts, {k: v[:4] for k, v in got.items()}, tiles, 2,
                                  model.mc)
      assert 0 < counts[0]


def test_non_default_stream(gpu_device):
  """The merge runs on the caller's stream, behind the forward, with no host synchronisation."""
  model = engine(12, gpu_device)
  rng = np.random.default_rng(15)
  frames = [device_frame('nv12', 120, 300, rng, gpu_device)]
  tiles = [(0,) + g for g in tile_grid(300, 120, TW, TH, 16)]
  want_rows, (want_dets, want_counts) = run_tiles(model, frames, 'nv12', tiles, 'demo')
  # spoil the merged buffer, then run on a side stream after a long kernel queued there
  res = model.tile_results_device()
  junk = np.full((12 * res['max_dets'] * 28,), 0x5A, np.uint8)
  _lib.check(model._lib.sqdet_memcpy_h2d(res['dets'], junk.ctypes.data, junk.nbytes, None))
  _lib.check(model._lib.sqdet_stream_sync(gpu_device, None))
  s = torch.cuda.Stream(gpu_device)
  with torch.cuda.stream(s):
    x = torch.randn(4096, 4096, device=gpu_device)
    for _ in range(8):
      x = x @ x
      x = x / x.norm()
  model.forward_device_tiles(frames, 'nv12', tiles, stream=s.cuda_stream)
  dets, counts = model.tile_results(1, stream=s.cuda_stream)
  assert np.array_equal(counts, want_counts[:1])
  assert dets.tobytes() == want_dets.tobytes()


# ---- sqdet_merge_tiles on adversarial rows --------------------------------------------------------
@pytest.mark.parametrize('t,n,A,top_n,thresh', [
    (6, 2, 200, 64, 0.005), (20, 1, 200, 64, 0.005), (5, 5, 40, 64, 0.005),
    (4, 2, 150, 0, 0.2), (7, 3, 30, 0, -1.0), (3, 1, 10, 25, 0.3),
    # either side of the per-tile selection's 20 cached keys per thread (A <= 20480) and of the
    # filter's 24 (A <= 24576), with the top-N cut inside a run of tied scores; top_n 1024 is the
    # table's capacity, with t * 1024 stage-1 candidates per frame
    *[(t, t // 4 + 1, A, top_n, 0.005) for A in (20480, 20481, 24576, 24577) for t in (2, 9)
      for top_n in (64, 1024)],
    # 128 tiles, the most one call takes: one frame, one tile per frame, frames of 4 and 2 tiles
    (128, 1, 200, 64, 0.005), (128, 128, 100, 64, 0.005), (128, 40, 150, 64, 0.005)])
def test_merge_tiles_adversarial(gpu_device, t, n, A, top_n, thresh):
  classes, nms = 3, 0.4
  rng = np.random.default_rng(t * 100 + A)
  boxes, probs, cls = adversarial_rows(t, A, classes, rng)
  # tiles 2i and 2i + 1 on one frame where there are tiles enough, so the IoU pairs meet
  frames = [(k // 2) % n if t >= 2 * n else k % n for k in range(t)]
  tiles = [(f, 10 * (k % 2), 3 * (k - k % 2)) for k, f in enumerate(frames)]
  max_dets = 1024 if top_n == 0 else top_n
  dets, counts = merge_gpu(boxes, probs, cls, tiles, n, classes, top_n, thresh, nms, max_dets,
                           gpu_device)
  mc = type('mc', (), dict(CLASSES=classes, TOP_N_DETECTION=top_n, PROB_THRESH=thresh,
                           NMS_THRESH=nms))
  assert_merge_matches_oracle(dets, counts, {'det_boxes': boxes, 'det_probs': probs,
                                             'det_class': cls}, tiles, n, mc)


def test_merge_tiles_iou_exactly_at_threshold_keeps_both(gpu_device):
  boxes = np.zeros((2, 4, 4), np.float32) + np.float32([100, 100, 2, 2])
  probs = np.zeros((2, 4), np.float32)
  cls = np.zeros((2, 4), np.int64)
  boxes[0, 0], boxes[1, 0] = (10.5, 8.5, 7, 7), (3.5, 8.5, 7, 7)
  probs[0, 0], probs[1, 0] = 0.9, 0.8
  tiles = [(0, 0, 0), (0, 10, 0)]
  dets, counts = merge_gpu(boxes, probs, cls, tiles, 1, 1, 2, 0.0, 0.4, 2, gpu_device)
  assert counts[0] == 2 and dets[0]['anchor'].tolist() == [0, 4]
  dets, counts = merge_gpu(boxes, probs, cls, tiles, 1, 1, 2, 0.0, 0.39, 2, gpu_device)
  assert counts[0] == 1 and dets[0]['anchor'].tolist() == [0, -1]


# ---- refusals -------------------------------------------------------------------------------------
def snapshot(model):
  return (model.read_tensor('image_input').tobytes(),
          {k: v.tobytes() for k, v in fetch_results(model, model.gpu_id).items()},
          [a.tobytes() for a in merged(model, model.mc.BATCH_SIZE)])


def test_refusals_before_device_work(gpu_device):
  B = 4
  model = engine(B, gpu_device)
  lib, eng = model._lib, model._engine
  rng = np.random.default_rng(16)
  H, W = 100, 250
  frames = [device_frame('bgr', H, W, rng, gpu_device) for _ in range(2)]
  good = [(0, 0, 0, TW, TH), (1, 10, 10, TW, TH), (0, 100, 40, TW, TH)]
  run_tiles(model, frames, 'bgr', good, 'demo')
  before = snapshot(model)

  planes = [frames[0].data_ptr(), None, None, frames[1].data_ptr(), None, None]

  def call(tiles, n=2, e=eng, pl=planes, hs=(H, H), ws=(W, W), pitches=None, order=0, fmt=0):
    t = len(tiles)
    flat = [v for tl in tiles for v in tl]
    return lib.sqdet_forward_tiles(
        e, n, fmt, (C.c_void_p * 6)(*pl) if pl is not None else None,
        (C.c_int64 * 6)(*pitches) if pitches else None, (C.c_int32 * 2)(*hs),
        (C.c_int32 * 2)(*ws), t, (C.c_int32 * max(1, 5 * t))(*flat), order, None)

  cases = [
      (dict(tiles=good, e=None), b'null'),
      (dict(tiles=good, pl=None), b'null'),
      (dict(tiles=[]), b't must be'),
      (dict(tiles=good * 2), b't must be'),
      (dict(tiles=good[:1], n=2), b'n must be'),
      (dict(tiles=good, n=0), b'n must be'),
      (dict(tiles=[(0, 0, 0, TW, TH), (2, 0, 0, TW, TH)]), b'tile 1: frame index 2'),
      (dict(tiles=[(0, 0, 0, TW, TH), (0, 5, 0, TW, TH)]), b'frame 1 has no tile'),
      (dict(tiles=[(0, 0, 0, TW, TH), (1, 0, 0, 0, TH)]), b'tile 1 (frame 1) is empty'),
      (dict(tiles=[(0, 0, 0, TW, TH), (1, W - TW + 1, 0, TW, TH)]),
       b'tile 1 (frame 1) is outside its frame'),
      (dict(tiles=[(0, -1, 0, TW, TH), (1, 0, 0, TW, TH)]), b'tile 0 (frame 0) is outside'),
      (dict(tiles=good, order=2), b'order'),
      (dict(tiles=good, fmt=9), b'format'),
      (dict(tiles=good, pl=[planes[0], None, None, None, None, None]),
       b'tile 1 (frame 1) is a null pointer'),
      (dict(tiles=good, pitches=[3 * W, 0, 0, 3 * W - 1, 0, 0]),
       b'tile 1 (frame 1): row pitch below'),
      (dict(tiles=good, hs=(H, 1 << 20), ws=(W, W)), b'tile 1 (frame 1) is not inside'),
  ]
  for kw, msg in cases:
    assert call(**kw) == ERR_INVALID_ARG, kw
    assert msg in lib.sqdet_last_error(), (kw, lib.sqdet_last_error())
  assert snapshot(model) == before

  hd = C.c_void_p()
  conf = _lib.Config(batch_size=1, image_height=8, image_width=8, classes=3, anchors_per_grid=9,
                     top_n_detection=64, prob_thresh=0.005, nms_thresh=0.4, exp_thresh=1.0,
                     batch_norm_epsilon=1e-5, math_mode=0, max_dets=0)
  _lib.check(lib.sqdet_create(C.byref(conf), gpu_device, C.byref(hd)))
  assert call(good[:1], n=1, e=hd) == ERR_STATE
  assert b'finalize' in lib.sqdet_last_error()
  assert lib.sqdet_tile_results_dev(hd, None, None, None) == ERR_STATE
  lib.sqdet_destroy(hd)

  # the facade raises ValueError for the same kinds of input
  bad = [([frames[0]], good),                                   # tile of a missing frame
         (frames, [(0, 0, 0, TW, TH)]),                         # frame 1 without a tile
         (frames, [(0, 0, 0, TW, TH), (1, 0, 0, TW, H + 1)]),   # outside
         (frames, [(0, 0, 0, TW, TH), (1, 0, 0, 0, TH)]),       # empty
         (frames, [(0, 0, 0, TW, TH), (1, 0, 0, TW)]),          # not 5 numbers
         (frames, []), (frames, good * 2)]
  for fr, tl in bad:
    with pytest.raises(ValueError):
      model.forward_device_tiles(fr, 'bgr', tl)
  with pytest.raises(ValueError):
    model.forward_device_tiles(frames, 'yuyv', good)
  with pytest.raises(ValueError):
    model.forward_device_tiles(frames, 'bgr', good, order='x')
  with pytest.raises(ValueError):
    model.forward_device_tiles([frames[0].cpu(), frames[1]], 'bgr', good)
  assert snapshot(model) == before
  # still right afterwards
  check_case(model, frames, 'bgr', good, 'eval')


def test_demo_video_tiles(gpu_device, tmp_path):
  """`demo.py --mode video --tiles` on a short synthetic video writes full-frame images."""
  import cv2
  video = str(tmp_path / 'in.avi')
  w, h = 1280, 720
  writer = cv2.VideoWriter(video, cv2.VideoWriter_fourcc(*'MJPG'), 10, (w, h))
  assert writer.isOpened()
  rng = np.random.default_rng(17)
  for _ in range(3):
    writer.write(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
  writer.release()
  out = tmp_path / 'out'
  demo.main(['--mode', 'video', '--tiles', '--checkpoint', 'synthetic', '--input_path', video,
             '--out_dir', str(out), '--gpu', str(gpu_device)])
  names = sorted(os.listdir(out))
  assert names == ['000001.jpg', '000002.jpg', '000003.jpg']
  for nm in names:
    assert cv2.imread(str(out / nm)).shape == (h, w, 3)
