"""oracle.tiles.merge_tiles: filter_prediction over each frame's union of tile rows.  One tile
per frame at the origin is filter_prediction per image; multi-tile unions equal the reference's
own filter_prediction on the concatenated, shifted rows (tie-free scores)."""
import numpy as np
import pytest

from oracle import postproc, ref_import, tiles as oracle_tiles

CLASSES, NMS = 3, 0.4


def tile_rows(t, A, rng, tile_w=160, tile_h=60):
  """t tile rows of distinct scores and boxes inside a tile_w x tile_h tile (so NMS bites)."""
  cx = rng.uniform(0.5, tile_w, (t, A))
  cy = rng.uniform(0.5, tile_h, (t, A))
  w = rng.uniform(4, 80, (t, A))
  h = rng.uniform(4, 40, (t, A))
  boxes = np.stack([cx, cy, w, h], -1).astype(np.float32)
  probs = rng.permutation(t * A).reshape(t, A).astype(np.float32) / np.float32(t * A)
  cls = rng.integers(0, CLASSES, (t, A)).astype(np.int64)
  return boxes, probs, cls


@pytest.mark.parametrize('top_n,thresh', [(16, 0.005), (0, 0.6), (400, 0.5)])
def test_one_tile_per_frame_at_origin_is_filter_prediction(top_n, thresh):
  rng = np.random.default_rng(1)
  boxes, probs, cls = tile_rows(4, 100, rng)
  tiles = [(f, 0, 0, 160, 60) for f in range(4)]
  got = oracle_tiles.merge_tiles(boxes, probs, cls, tiles, 4, CLASSES, top_n, thresh, NMS)
  for f in range(4):
    want = postproc.filter_prediction(boxes[f], probs[f], cls[f], CLASSES, top_n, thresh, NMS)
    assert np.array_equal(np.array(got[f][0]), np.array(want[0]))
    assert got[f][1:] == want[1:]


def test_union_index_and_offsets():
  rng = np.random.default_rng(2)
  boxes, probs, cls = tile_rows(3, 50, rng)
  tiles = [(1, 7, 9), (0, 0, 0), (1, 100, 3)]                    # frame 1's tiles: rows 0, 2
  got = oracle_tiles.merge_tiles(boxes, probs, cls, tiles, 2, CLASSES, 10, 0.005, NMS)
  for b, src in zip(got[1][0], got[1][3]):
    p, a = divmod(src, 50)
    k = (0, 2)[p]
    want = boxes[k, a].copy()
    want[0] += np.float32(tiles[k][1])
    want[1] += np.float32(tiles[k][2])
    assert np.array_equal(b, want)


@pytest.mark.skipif(not ref_import.available(), reason='reference tree not present')
@pytest.mark.parametrize('top_n,thresh', [(32, 0.005), (0, 0.7)])
def test_multi_tile_union_matches_reference(top_n, thresh):
  ns = ref_import.load()
  rng = np.random.default_rng(3)
  A = 120
  boxes, probs, cls = tile_rows(5, A, rng)
  tiles = [(0, 0, 0), (1, 0, 0), (0, 130, 0), (1, 40, 50), (0, 0, 45)]
  got = oracle_tiles.merge_tiles(boxes, probs, cls, tiles, 2, CLASSES, top_n, thresh, NMS)
  for f in range(2):
    rows = [k for k, t in enumerate(tiles) if t[0] == f]
    ub = np.concatenate([boxes[k] + np.float32([tiles[k][1], tiles[k][2], 0, 0]) for k in rows])
    up = np.concatenate([probs[k] for k in rows])
    uc = np.concatenate([cls[k] for k in rows])
    fb, fp, fc = ref_import.ref_filter_prediction(ns, ub, up, uc, CLASSES, top_n, thresh, NMS)
    assert len(fb) == len(got[f][0]) > 0
    assert np.array_equal(np.array(fb), np.array(got[f][0]))
    assert [float(p) for p in fp] == [float(p) for p in got[f][1]]
    assert list(fc) == got[f][2]
