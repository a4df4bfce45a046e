"""filter_prediction over whole frames detected as tiles (oracle — test infrastructure only).

Restates what sqdet_forward_tiles / sqdet_merge_tiles compute, on top of the pinned
``oracle.postproc.filter_prediction`` (reference ``src/nn_skeleton.py:696-734``).
"""
from __future__ import annotations

import numpy as np

from .postproc import filter_prediction


def merge_tiles(det_boxes, det_probs, det_class, tiles, n, classes, top_n, prob_thresh,
                nms_thresh):
  """Row k of det_boxes / det_probs / det_class is tile k = tiles[k] = (frame, x, y[, w, h]), its
  boxes in tile pixels.  Frame f's union concatenates its tiles' rows in call order, each box
  shifted by the tile's float32 (x, y); `final_src` is the union index p * A + anchor of the
  frame's p-th tile.  Returns one filter_prediction tuple per frame [0, n)."""
  out = []
  for f in range(n):
    rows = [k for k, tile in enumerate(tiles) if int(tile[0]) == f]
    boxes = []
    for k in rows:
      b = np.array(det_boxes[k], dtype=np.float32)
      b[:, 0] += np.float32(tiles[k][1])
      b[:, 1] += np.float32(tiles[k][2])
      boxes.append(b)
    out.append(filter_prediction(np.concatenate(boxes),
                                 np.concatenate([np.asarray(det_probs[k]) for k in rows]),
                                 np.concatenate([np.asarray(det_class[k]) for k in rows]),
                                 classes, top_n, prob_thresh, nms_thresh))
  return out
