"""Whole-frame tile detection at the sizes it ships at, and sqdet_merge_tiles at the edges of its
selection and of its limits.

- SqueezeDet at 1242x375 on two 1080p frames, each the 2 x 4 tile_grid plus an overview tile: the
  merged records bitwise oracle.tiles.merge_tiles on the engine's own rows, each tile row against
  the oracle pipeline (cv2-pinned pre-processing, torch-CPU forward in fp32 and fp64,
  interpret_output, eval.py's rescale), and the merged records against merge_tiles on the oracle's
  rows up to near ties.
- SqueezeDet at 1408x448 and 1600x480, where the per-tile top-N no longer keeps its keys in
  registers, and at 1600x480 the per-image filter neither: merged records bitwise.
- sqdet_merge_tiles of one whole-frame tile per frame bitwise sqdet_topk_nms of the same rows on
  either side of both caching limits; calls whose frames take different branches; a threshold
  overflow on one frame; and the limits of 128 tiles and 1024 candidates."""
import numpy as np
import pytest
import torch

import oracle
from gpu_util import (TOL, adversarial_rows, assert_boxes_close, assert_classes_match,
                      assert_merge_matches_oracle, assert_padding, fetch_results, make_net,
                      merge_gpu, merge_gpu_rc, topk_nms_gpu)
from oracle import pixfmt, preproc
from oracle import tiles as oracle_tiles
from oracle.torch_port import TorchForward
from squeezedet_b200 import _lib
from squeezedet_b200 import config as cfg
from squeezedet_b200.utils.util import tile_grid

ERR_UNSUPPORTED = -3
FRAME_W, FRAME_H, OVERLAP = 1920, 1080, 128
SHIPPED = (1242, 375)
WINDOW_SIZES = [(1408, 448), (1600, 480)]
# The top-N selections give each of their 1024 threads a run of ceil(A / 1024) anchors and keep
# the run's keys in registers up to 20 (the per-tile top-N of the merge) or 24 (the per-image
# filter) of them.  These anchor counts sit on either side of both limits.
FT, MERGE_KEYS, FILTER_KEYS = 1024, 20, 24
SELECT_A = (16848, 20480, 20481, 24576, 24577)


def anchors(width, height):
  grid = oracle.layer_table('squeezeDet', height, width)[-1][2]
  return grid[0] * grid[1] * cfg.kitti_squeezeDet_config().ANCHOR_PER_GRID


def window(A):
  """Which of the two selections keep their keys in registers at A anchors."""
  per = -(-A // FT)
  return 'both' if per <= MERGE_KEYS else 'filter' if per <= FILTER_KEYS else 'neither'


def frame_tiles(f, width, height):
  """Frame f's tile_grid at the engine size, then one overview tile of the whole frame."""
  return ([(f,) + g for g in tile_grid(FRAME_W, FRAME_H, width, height, OVERLAP)]
          + [(f, 0, 0, FRAME_W, FRAME_H)])


def test_cases_reach_every_selection_window():
  """The engine sizes below run the shipped size with both selections cached and 17 or more keys
  per thread, then the merge uncached with the filter cached, then neither; the direct merges sit
  on each side of both limits."""
  A = anchors(*SHIPPED)
  assert A == 16848 and window(A) == 'both' and -(-A // FT) >= 17
  assert [window(anchors(*s)) for s in WINDOW_SIZES] == ['filter', 'neither']
  assert [window(a) for a in SELECT_A] == ['both', 'both', 'filter', 'filter', 'neither']
  assert -(-SELECT_A[1] // FT) == MERGE_KEYS and -(-SELECT_A[3] // FT) == FILTER_KEYS
  assert len(frame_tiles(0, *SHIPPED)) == 9            # the 2 x 4 grid plus the overview
  assert all(len(frame_tiles(0, *s)) == 7 for s in WINDOW_SIZES)


# ---- the engine at full size ----------------------------------------------------------------------
def host_frames(fmt, rng):
  shape = (FRAME_H, FRAME_W, 3) if fmt == 'bgr' else (3 * FRAME_H // 2, FRAME_W)
  return [rng.integers(0, 256, shape, dtype=np.uint8) for _ in range(2)]


def host_bgr(fmt, frame):
  return frame if fmt == 'bgr' else pixfmt.to_bgr('nv12', (frame[:FRAME_H], frame[FRAME_H:]))


def run_and_check_merge(model, host, fmt, tiles, order):
  """forward_device_tiles, then the merged records bitwise merge_tiles on the engine's own rows
  [0, t), padding included, counts of rows [n, B) 0, and every frame keeps a detection.  Returns
  the per-tile rows and the merged records of frames [0, n)."""
  t, n = len(tiles), len(host)
  frames = [torch.from_numpy(h).to(model.gpu_id) for h in host]
  model.forward_device_tiles(frames, fmt, tiles, order=order)
  torch.cuda.synchronize(model.gpu_id)
  rows = fetch_results(model, model.gpu_id)
  dets, counts = model.tile_results(model.mc.BATCH_SIZE)
  want = assert_merge_matches_oracle(dets, counts, {k: v[:t] for k, v in rows.items()}, tiles, n,
                                     model.mc)
  assert not counts[n:].any()
  assert all(len(w[3]) for w in want)
  return rows, dets[:n], counts[:n]


def oracle_rows(mc, weights, host, fmt, tiles, order, dtype):
  """The oracle pipeline on each tile: BGR crop -> preprocess -> TorchForward -> interpret_output
  -> boxes divided by (IMAGE_WIDTH / w, IMAGE_HEIGHT / h) as eval.py:83-84 does.  Returns (preds,
  boxes, probs, classes) of all tiles."""
  bgr = [host_bgr(fmt, h) for h in host]
  fed = np.stack([preproc.preprocess(bgr[f][y:y + h, x:x + w], mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT,
                                     mc.BGR_MEANS, order) for f, x, y, w, h in tiles])
  fwd = TorchForward('squeezeDet', weights, dtype=dtype)
  preds = np.concatenate([fwd(fed[i:i + 2]) for i in range(0, len(tiles), 2)])
  boxes, probs, cls = oracle.interpret_output(preds, mc.ANCHOR_BOX, mc.CLASSES, mc.ANCHOR_PER_GRID,
                                              mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.EXP_THRESH,
                                              dtype)
  for k, (_, _, _, w, h) in enumerate(tiles):
    # Python float scales: numpy divides the float32 rows in float32
    boxes[k, :, 0::2] /= mc.IMAGE_WIDTH / float(w)
    boxes[k, :, 1::2] /= mc.IMAGE_HEIGHT / float(h)
  return preds, boxes, probs, cls


def union(rows_of_tiles, tiles, f, shift=False):
  """Frame f's union of per-tile rows in call order; boxes shifted by the tile origin in their own
  dtype when `shift`."""
  parts = []
  for k, tile in enumerate(tiles):
    if tile[0] != f:
      continue
    r = np.array(rows_of_tiles[k])
    if shift:
      r[:, 0] += r.dtype.type(tile[1])
      r[:, 1] += r.dtype.type(tile[2])
    parts.append(r)
  return np.concatenate(parts)


def assert_merge_near_oracle(dets, counts, rows, ref32, ref64, tiles, mc):
  """Each frame's kept union indices equal those of merge_tiles on the oracle's fp32 rows, except
  for (1) near ties among the union's top TOP_N_DETECTION + 2 scores, the rule of
  test_gpu_configs, (2) anchors whose class differs from the oracle's (assert_classes_match
  allows those only at a near tie of the class scores), (3) anchors with a same-class candidate
  at an IoU that the GPU's boxes, the oracle's fp32 boxes and its fp64 boxes put on different
  sides of NMS_THRESH."""
  _, wb, wp, wc = ref32
  wb64 = ref64[1]
  want = oracle_tiles.merge_tiles(wb, wp, wc, tiles, len(dets), mc.CLASSES, mc.TOP_N_DETECTION,
                                  mc.PROB_THRESH, mc.NMS_THRESH)
  thr32, thr64 = np.float32(mc.NMS_THRESH), float(np.float32(mc.NMS_THRESH))
  for f, (_, _, _, osrc) in enumerate(want):
    src = dets[f]['anchor'][:int(counts[f])].tolist()
    up = union(wp, tiles, f)
    cls_o, cls_g = union(wc, tiles, f), union(rows['det_class'], tiles, f)
    boxes = [union(rows['det_boxes'], tiles, f, True), union(wb, tiles, f, True),
             union(wb64, tiles, f, True)]
    top = np.argsort(-up.astype(np.float64), kind='stable')[:mc.TOP_N_DETECTION + 2]
    s = up[top].astype(np.float64)
    gap = np.abs(s[:, None] - s[None, :]) <= 10 * TOL * s[:, None]
    np.fill_diagonal(gap, False)
    near = {int(top[a]) for a in np.nonzero(gap.any(axis=1))[0]}
    class_tie = {int(j) for j in top if cls_g[j] != cls_o[j]}
    for j in set(src) ^ set(osrc):
      if j in near or j in class_tie:
        continue
      same = [int(i) for i in top if i != j and cls_o[i] == cls_o[j]]
      sides = [oracle.batch_iou(b[same], b[j]) > thr for b, thr in
               zip(boxes, (thr32, thr32, thr64))]
      flipped = any((a != b).any() for a, b in zip(sides, sides[1:]))
      assert flipped, ('kept sets differ outside a near tie', f, j, sorted(near))
    if not near and not class_tie:
      assert src == osrc, f


@pytest.mark.gpu
@pytest.mark.parametrize('fmt,order', [('bgr', 'demo'), ('nv12', 'eval')])
def test_shipped_size_against_oracle_pipeline(fmt, order, gpu_device):
  """SqueezeDet 1242x375, two 1080p frames of 9 tiles each (NV12's tiles interleaved by frame)."""
  rng = np.random.default_rng({'bgr': 41, 'nv12': 42}[fmt])
  host = host_frames(fmt, rng)
  a, b = frame_tiles(0, *SHIPPED), frame_tiles(1, *SHIPPED)
  tiles = a + b if fmt == 'bgr' else [tl for pair in zip(a, b) for tl in pair]
  t = len(tiles)
  model, weights = make_net('squeezeDet', *SHIPPED, t, gpu_device, seed=0)
  mc = model.mc
  assert mc.ANCHORS == 16848 and t == 18 and 0 < mc.TOP_N_DETECTION < mc.ANCHORS
  rows, dets, counts = run_and_check_merge(model, host, fmt, tiles, order)
  ref32 = oracle_rows(mc, weights, host, fmt, tiles, order, np.float32)
  ref64 = oracle_rows(mc, weights, host, fmt, tiles, order, np.float64)
  np.testing.assert_allclose(rows['det_probs'][:t], ref32[2], rtol=TOL, atol=1e-7)
  assert_boxes_close(rows['det_boxes'][:t], ref32[1], ref64[1])
  assert_classes_match(rows['det_class'][:t], ref32[3], ref64[0], mc.ANCHOR_PER_GRID, mc.CLASSES,
                       TOL)
  assert_merge_near_oracle(dets, counts, rows, ref32, ref64, tiles, mc)


@pytest.mark.gpu
@pytest.mark.parametrize('width,height,fmt,order', [(1408, 448, 'bgr', 'demo'),
                                                    (1600, 480, 'nv12', 'eval')])
def test_selection_windows_at_engine_level(width, height, fmt, order, gpu_device):
  """Two 1080p frames of 7 tiles each at an engine size whose per-tile top-N re-reads its keys."""
  tiles = frame_tiles(0, width, height) + frame_tiles(1, width, height)
  model, _ = make_net('squeezeDet', width, height, len(tiles), gpu_device, seed=0)
  assert model.mc.ANCHORS == anchors(width, height)
  host = host_frames(fmt, np.random.default_rng(width))
  run_and_check_merge(model, host, fmt, tiles, order)


# ---- sqdet_merge_tiles on its own -----------------------------------------------------------------
def filter_mc(classes, top_n, thresh, nms):
  return type('mc', (), dict(CLASSES=classes, TOP_N_DETECTION=top_n, PROB_THRESH=thresh,
                             NMS_THRESH=nms))


@pytest.mark.gpu
@pytest.mark.parametrize('top_n', [64, 1024])
@pytest.mark.parametrize('A', SELECT_A)
def test_merge_of_whole_frame_tiles_is_the_filter(A, top_n, gpu_device):
  """One tile at (0, 0) per frame: the merge's selection and the filter's own copy of it give the
  same records, bit for bit, with the cut inside a run of tied scores."""
  rng = np.random.default_rng(A + top_n)
  boxes, probs, cls = adversarial_rows(2, A, 3, rng)
  # the merge adds +0.0 to each centre, which turns a -0.0 into +0.0
  assert not np.signbit(boxes[..., :2]).any()
  tiles = [(0, 0, 0), (1, 0, 0)]
  dm, cm = merge_gpu(boxes, probs, cls, tiles, 2, 3, top_n, 0.005, 0.4, top_n, gpu_device)
  df, cf = topk_nms_gpu(boxes, probs, cls, 3, top_n, 0.005, 0.4, max_dets=top_n, device=gpu_device)
  assert (cm > 0).all()
  assert cm.tolist() == cf.tolist()
  assert dm.tobytes() == df.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize('top_n', [100, 150])
def test_merge_tiles_frames_take_both_branches(top_n, gpu_device):
  """Frames whose union is longer than top_n take the top-N branch (stage 1 keeps whole tiles:
  top_n >= A), the others the PROB_THRESH branch, in one call."""
  A, classes = 100, 3
  frames = [0, 1, 0, 2, 2, 0, 3]
  union_len = [frames.count(f) * A for f in range(4)]
  assert [u > top_n for u in union_len] == [True, False, True, False]
  rng = np.random.default_rng(top_n)
  boxes, probs, cls = adversarial_rows(len(frames), A, classes, rng)
  tiles = [(f, 10 * (k % 2), 3 * k) for k, f in enumerate(frames)]
  dets, counts = merge_gpu(boxes, probs, cls, tiles, 4, classes, top_n, 0.2, 0.4, 1024, gpu_device)
  assert (counts > 0).all()
  assert_merge_matches_oracle(dets, counts, {'det_boxes': boxes, 'det_probs': probs,
                                             'det_class': cls}, tiles, 4,
                              filter_mc(classes, top_n, 0.2, 0.4))


@pytest.mark.gpu
@pytest.mark.parametrize('top_n', [0, 2000])
def test_merge_tiles_overflow_on_one_frame(top_n, gpu_device):
  """Frame 0 holds more threshold candidates than the 1024-entry table: count -1 and padding for
  it alone, the other frames' records as the oracle's.  top_n 2000 is no frame's top-N branch."""
  A, classes, thresh = 500, 3, -1.0
  frames = [0, 1, 0, 2, 0, 2]
  rng = np.random.default_rng(55 + top_n)
  boxes, probs, cls = adversarial_rows(len(frames), A, classes, rng)
  cand = [sum(int((probs[k] > thresh).sum()) for k, fk in enumerate(frames) if fk == f)
          for f in range(3)]
  assert cand[0] > 1024 >= max(cand[1:])
  assert top_n == 0 or top_n >= 3 * A
  tiles = [(f, 10 * (k % 2), 3 * k) for k, f in enumerate(frames)]
  dets, counts = merge_gpu(boxes, probs, cls, tiles, 3, classes, top_n, thresh, 0.4, 1024,
                           gpu_device)
  assert counts[0] == -1
  assert_padding(dets[0], 0, 0)
  # frames 1 and 2 alone, renumbered 0 and 1, keep their tiles' call order and union indices
  keep = [k for k, f in enumerate(frames) if f > 0]
  assert_merge_matches_oracle(dets[1:], counts[1:], {'det_boxes': boxes[keep],
                                                     'det_probs': probs[keep],
                                                     'det_class': cls[keep]},
                              [(frames[k] - 1,) + tiles[k][1:] for k in keep], 2,
                              filter_mc(classes, top_n, thresh, 0.4))


@pytest.mark.gpu
def test_merge_tiles_limits(gpu_device):
  """129 tiles, and a top-N branch of more than 1024 entries or more than max_dets, are refused
  before any device work; top_n 1025 is accepted when no frame's union is longer than it."""
  rng = np.random.default_rng(56)
  lib = _lib.load()
  refused = [
      (129, 1, 100, 64, 64, b'at most 128 tiles'),
      (129, 129, 100, 64, 64, b'at most 128 tiles'),
      (2, 1, 600, 1025, 1025, b'TOP_N_DETECTION above capacity'),
      (2, 1, 600, 64, 63, b'TOP_N_DETECTION above capacity'),
  ]
  for t, n, A, top_n, max_dets, msg in refused:
    boxes, probs, cls = adversarial_rows(t, A, 3, rng)
    tiles = [(k % n, 10 * (k % 2), 3 * k) for k in range(t)]
    rc, dets, counts = merge_gpu_rc(boxes, probs, cls, tiles, n, 3, top_n, 0.005, 0.4, max_dets,
                                    gpu_device)
    assert rc == ERR_UNSUPPORTED, (t, n, top_n, max_dets)
    assert msg in lib.sqdet_last_error(), lib.sqdet_last_error()
    assert (dets.view(np.uint8) == 0x77).all() and (counts == 12345).all()
  boxes, probs, cls = adversarial_rows(2, 500, 3, rng)
  tiles = [(0, 0, 0), (0, 10, 6)]
  dets, counts = merge_gpu(boxes, probs, cls, tiles, 1, 3, 1025, 0.2, 0.4, 1024, gpu_device)
  assert counts[0] > 0
  assert_merge_matches_oracle(dets, counts, {'det_boxes': boxes, 'det_probs': probs,
                                             'det_class': cls}, tiles, 1,
                              filter_mc(3, 1025, 0.2, 0.4))
