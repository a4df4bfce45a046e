"""The reference's detection error analysis (analyze_detections, src/dataset/kitti.py:182-296,
which eval.py:128-130 runs after the APs), restated: label files and the detection files eval.py
writes in, det_error_file.txt's text and the counts out.  Test infrastructure only.

  text, counts = analyze(label_dir, det_dir, image_ids, class_names)

The rules, with the reference's lines:
  * ground truth (_load_kitti_annotation, :53-98): the label lines whose type, lowercased, is a
    class name, in file order; EXCLUDE_HARD_EXAMPLES is False in every shipped config, so no
    difficulty filter.  Only those boxes must pass x1 >= 0, x1 <= x2, y1 >= 0, y1 <= y2.
  * every box in center form by bbox_transform_inv (utils/util.py:181-196): w = x2 - x1 + 1.0,
    cx = x1 + 0.5 * w, in double.
  * detections (:190-214): each file's lines, read back as doubles, sorted by score descending
    with Python's stable sort (file order on ties: class id, then record order).
  * matching (:226-268): an image with G objects counts its first G detections and nothing
    else; G = 0 contributes nothing.  A counted detection's IoUs against all objects (batch_iou,
    utils/util.py:32-54) give max_iou and gt_idx = the first index reaching it.  max_iou > 0.1
    and the same class: correct when max_iou >= 0.5 and gt_idx is not yet detected, repeated
    when it is, loc when max_iou < 0.5; max_iou > 0.1 and another class: cls; else bg.
  * lines (:183-192, :269-272): the loc / cls / bg detections in sorted order, then each object
    no correct detection took, as 'missed' with score -1.0.
  * counts as COUNT_FIELDS; detected == correct.

load_reference() imports the reference's own kitti.py, unmodified, where the checkout exists;
run_reference() runs its analyze_detections.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys
import types

import numpy as np

from . import ref_import

COUNT_FIELDS = ('num_dets', 'num_objs', 'correct', 'loc', 'cls', 'bg', 'repeated', 'detected')
LINE = '{:s} {:s} {:.1f} {:.1f} {:.1f} {:.1f} {:s} {:.3f}\n'


def center(x1, y1, x2, y2):
  w = x2 - x1 + 1.0
  h = y2 - y1 + 1.0
  return [x1 + 0.5 * w, y1 + 0.5 * h, w, h]


def iou_row(gt, det):
  """IoU of each gt row [cx, cy, w, h] with det, numpy's operations in batch_iou's order."""
  lr = np.maximum(np.minimum(gt[:, 0] + 0.5 * gt[:, 2], det[0] + 0.5 * det[2]) -
                  np.maximum(gt[:, 0] - 0.5 * gt[:, 2], det[0] - 0.5 * det[2]), 0)
  tb = np.maximum(np.minimum(gt[:, 1] + 0.5 * gt[:, 3], det[1] + 0.5 * det[3]) -
                  np.maximum(gt[:, 1] - 0.5 * gt[:, 3], det[1] - 0.5 * det[3]), 0)
  inter = lr * tb
  return inter / (gt[:, 2] * gt[:, 3] + det[2] * det[3] - inter)


def read_ground_truth(path, class_to_idx):
  """[[cx, cy, w, h, class id]] of one label file."""
  out = []
  with open(path) as f:
    for line in f.readlines():
      t = line.strip().split(' ')
      cls = class_to_idx.get(t[0].lower().strip())
      if cls is None:
        continue
      x1, y1, x2, y2 = (float(v) for v in t[4:8])
      if not (x1 >= 0.0 and x1 <= x2 and y1 >= 0.0 and y1 <= y2):
        raise ValueError('%s: the reference asserts x1 >= 0, x1 <= x2, y1 >= 0, y1 <= y2' % path)
      out.append(center(x1, y1, x2, y2) + [cls])
  return out


def read_detections(path, class_to_idx):
  """[[cx, cy, w, h, class id, score]] of one detection file, sorted as the reference sorts."""
  out = []
  with open(path) as f:
    for line in f.readlines():
      t = line.strip().split(' ')
      out.append(center(*(float(v) for v in t[4:8])) + [class_to_idx[t[0].lower().strip()],
                                                        float(t[-1])])
  out.sort(key=lambda d: d[5], reverse=True)
  return out


def analyze(label_dir, det_dir, image_ids, class_names):
  """-> (det_error_file.txt's text, {COUNT_FIELDS: int})."""
  class_to_idx = {c: k for k, c in enumerate(class_names)}
  counts = dict.fromkeys(COUNT_FIELDS, 0)
  text = []

  def line(idx, kind, box, score):
    cx, cy, w, h = box[:4]
    text.append(LINE.format(idx, kind, cx - w / 2., cy - h / 2., cx + w / 2., cy + h / 2.,
                            class_names[int(box[4])], score))

  for idx in image_ids:
    gts = read_ground_truth(os.path.join(label_dir, idx + '.txt'), class_to_idx)
    dets = read_detections(os.path.join(det_dir, idx + '.txt'), class_to_idx)
    counts['num_objs'] += len(gts)
    if not gts:
      continue
    gt = np.array(gts)
    detected = [False] * len(gts)
    for det in dets[:len(gts)]:
      counts['num_dets'] += 1
      ious = iou_row(gt, np.array(det[:4]))
      best, g = np.max(ious), int(np.argmax(ious))
      if best <= 0.1:
        counts['bg'] += 1
        line(idx, 'bg', det, det[5])
      elif gt[g, 4] != det[4]:
        counts['cls'] += 1
        line(idx, 'cls', det, det[5])
      elif best < 0.5:
        counts['loc'] += 1
        line(idx, 'loc', det, det[5])
      elif detected[g]:
        counts['repeated'] += 1
      else:
        counts['correct'] += 1
        detected[g] = True
    for g, hit in enumerate(detected):
      if not hit:
        line(idx, 'missed', gt[g], -1.0)
    counts['detected'] += sum(detected)
  return ''.join(text), counts


# ---- the reference's own analyze_detections ----------------------------------------------------
_kitti_class = None


def load_reference():
  """The reference's kitti class from its unmodified src/dataset/kitti.py.  tensorflow is a stub
  whose variable_scope is a null context (bbox_transform_inv enters one), and `dataset` is a stub
  package over the reference's dataset directory, so that its Python 2 __init__ never runs."""
  global _kitti_class
  if _kitti_class is not None:
    return _kitti_class
  if not ref_import.available():
    raise RuntimeError('reference tree not present at ' + ref_import.REFERENCE_SRC)
  names = ('tensorflow', 'dataset', 'dataset.imdb', 'dataset.kitti', 'utils', 'utils.util')
  saved_mods = {k: sys.modules.get(k) for k in names}
  saved_path = list(sys.path)
  try:
    tf = types.ModuleType('tensorflow')
    tf.variable_scope = lambda *a, **k: contextlib.nullcontext()
    sys.modules['tensorflow'] = tf
    pkg = types.ModuleType('dataset')
    pkg.__path__ = [os.path.join(ref_import.REFERENCE_SRC, 'dataset')]
    sys.modules['dataset'] = pkg
    for m in names[2:]:
      sys.modules.pop(m, None)
    sys.path[:0] = [ref_import.REFERENCE_SRC]
    import importlib
    _kitti_class = importlib.import_module('dataset.kitti').kitti
    return _kitti_class
  finally:
    sys.path[:] = saved_path
    for k, v in saved_mods.items():
      if v is None:
        sys.modules.pop(k, None)
      else:
        sys.modules[k] = v


def run_reference(label_dir, det_dir, image_ids, class_names, error_file):
  """The reference's analyze_detections on the files: writes error_file -> (its `out` dict, the
  text it printed).  The object is built without __init__, with the attributes the analysis
  reads; its ground truth comes from its own _load_kitti_annotation."""
  cls = load_reference()
  imdb = object.__new__(cls)
  imdb._image_idx = list(image_ids)
  imdb._classes = list(class_names)
  imdb._class_to_idx = dict(zip(class_names, range(len(class_names))))
  imdb._label_path = label_dir
  imdb.mc = ref_import._EasyDict(EXCLUDE_HARD_EXAMPLES=False)
  imdb._rois = imdb._load_kitti_annotation()
  buf = io.StringIO()
  with contextlib.redirect_stdout(buf):
    out = imdb.analyze_detections(det_dir, error_file)
  return out, buf.getvalue()
