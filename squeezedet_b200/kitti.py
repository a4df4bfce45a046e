"""KITTI 2-D object scoring on the GPU (sqdet_kitti_eval): the files the KITTI devkit's
evaluate_object writes (stats_<cls>_ap.txt, _detection.txt, _orientation.txt and
plot/<cls>_detection.txt, _orientation.txt), byte for byte, from the engine's filtered records
and the label files, with no detection file read back.

  labels = read_labels('KITTI/training/label_2', image_ids)
  scores = evaluate_device(dets, counts, mc.CLASS_NAMES, labels)    # dets [n, max_dets] records
  write_stats(result_dir, scores)

The records are scored as the devkit scores the detection files eval.py writes from them
(utils/viz.write_kitti_detections: corners with 2 decimals, the score with 3, alpha 0.0).  Class
names match car, pedestrian and cyclist case-insensitively; other classes are never scored.  The
devkit's gnuplot scripts and renders are not written.  No engine is needed."""
from __future__ import annotations

import math
import os

import numpy as np

from . import _lib

CLASSES = ('car', 'pedestrian', 'cyclist')
TYPE_CODES = {'car': 0, 'pedestrian': 1, 'cyclist': 2, 'van': 3, 'person_sitting': 4,
              'dontcare': 5}          # SQDET_KITTI_*; any other type is SQDET_KITTI_OTHER
TYPE_OTHER = 6
MAX_DETS = 1024
N_SAMPLE_PTS = 41

OBJ_DTYPE = np.dtype([('x1', '<f8'), ('y1', '<f8'), ('x2', '<f8'), ('y2', '<f8'),
                      ('truncation', '<f8'), ('aos_term', '<f8'), ('type', '<i4'),
                      ('occlusion', '<i4')])
assert OBJ_DTYPE.itemsize == 56
RESULT_DTYPE = np.dtype([('similarity', '<f8', (9, N_SAMPLE_PTS)), ('tp', '<i4', (9, N_SAMPLE_PTS)),
                         ('fp', '<i4', (9, N_SAMPLE_PTS)), ('fn', '<i4', (9, N_SAMPLE_PTS)),
                         ('n_thresholds', '<i4', (9,)), ('n_gt', '<i4', (9,)),
                         ('evaluated', '<i4', (3,)), ('status', '<i4'), ('reserved', '<i4')])
assert RESULT_DTYPE.itemsize == 7472        # sizeof(sqdet_kitti_result), tail padding included
REASONS = {1: 'its count is outside [0, max_dets] (the filter\'s -1 overflow marker included)',
           2: 'a record\'s class id is outside class_names',
           3: 'a record has a non-finite box or prob',
           4: 'a record\'s prob is outside [0, 1]',
           5: 'its label offsets are not an increasing range within the objects',
           6: 'more than 41 thresholds'}


def _fold(name):
  """strcasecmp's case folding: ASCII letters only."""
  return name.encode().lower().decode()


class Labels:
  """The label files of n images, packed: objs [n_objects] OBJ_DTYPE in file order and
  offsets [n + 1] int64 (image i's objects are objs[offsets[i]:offsets[i + 1]])."""

  def __init__(self, objs, offsets):
    self.objs, self.offsets = objs, offsets

  def __len__(self):
    return len(self.offsets) - 1


def read_labels(label_dir, image_ids):
  """label_dir/<id>.txt for each id -> Labels.  A line holds 15 fields: type, truncation,
  occlusion (an integer), alpha, x1, y1, x2, y2 and 7 fields that scoring does not use; blank
  lines are skipped.  A line with another field count raises ValueError naming the file and line,
  and a missing file FileNotFoundError.  Each object carries (1 + cos(alpha)) / 2, its
  orientation similarity against the detections' alpha of 0.0, from the host's libm."""
  rows, offsets = [], [0]
  for idx in image_ids:
    path = os.path.join(label_dir, idx + '.txt')
    with open(path) as f:
      for ln, line in enumerate(f, 1):
        t = line.split()
        if not t:
          continue
        if len(t) != 15:
          raise ValueError('%s:%d: a label line has 15 fields, got %d' % (path, ln, len(t)))
        try:
          trunc, occ, alpha = float(t[1]), int(t[2]), float(t[3])
          box = [float(v) for v in t[4:8]]
        except ValueError as e:
          raise ValueError('%s:%d: %s' % (path, ln, e)) from None
        rows.append((*box, trunc, (1.0 + math.cos(alpha)) / 2.0,
                     TYPE_CODES.get(_fold(t[0]), TYPE_OTHER), occ))
    offsets.append(len(rows))
  return Labels(np.array(rows, OBJ_DTYPE), np.array(offsets, np.int64))


def _nan():
  return float('-nan')     # what 0.0 / 0.0 gives on x86: the default NaN, sign bit set


def _max_element(x, i):
  """*std::max_element(x.begin() + i, x.end()): the first of the largest under operator<."""
  best = x[i]
  for y in x[i + 1:]:
    if best < y:
      best = y
  return best


def _curves(res, cd):
  """eval_class's precision and AOS from the counts of (class, difficulty) cd."""
  nt = int(res['n_thresholds'][cd])
  precision = [0.0] * N_SAMPLE_PTS
  aos = [0.0] * N_SAMPLE_PTS
  for i in range(nt):
    tp, fp = int(res['tp'][cd, i]), int(res['fp'][cd, i])
    den = float(tp + fp)
    precision[i] = tp / den if den else _nan()
    aos[i] = float(res['similarity'][cd, i]) / den if den else _nan()
  for i in range(nt):
    precision[i] = _max_element(precision, i)
    aos[i] = _max_element(aos, i)
  return precision, aos


def average_precision(precision):
  """The 11-point AP: precision[0], [4], ..., [40] summed in order, over 11."""
  ap = 0.0
  for i in range(0, N_SAMPLE_PTS, 4):
    ap += precision[i]
  return ap / 11.0


def _records(dets, counts, device):
  """dets and counts as contiguous CUDA tensors: dets [n, max_dets] DET_DTYPE (numpy) or a CUDA
  tensor of those bytes with n rows; counts [n] int32."""
  import torch
  if isinstance(dets, np.ndarray):
    if dets.dtype != _lib.DET_DTYPE or dets.ndim != 2:
      raise ValueError('dets must be a [n, max_dets] array of DET_DTYPE records')
    n, max_dets = dets.shape
    d = torch.from_numpy(np.ascontiguousarray(dets).view(np.uint8).reshape(n, -1)).to(device)
  else:
    d = dets.contiguous()
    n = d.shape[0]
    per = d.numel() * d.element_size() // max(n, 1)
    if n < 1 or per % _lib.DET_DTYPE.itemsize or per * n != d.numel() * d.element_size():
      raise ValueError('dets must hold [n, max_dets] records of %d bytes' % _lib.DET_DTYPE.itemsize)
    max_dets = per // _lib.DET_DTYPE.itemsize
  c = torch.as_tensor(np.asarray(counts, np.int32) if not torch.is_tensor(counts) else counts)
  c = c.to(device=device, dtype=torch.int32).contiguous()
  if c.shape != (n,):
    raise ValueError('counts must have one entry per image: %d, got %s' % (n, tuple(c.shape)))
  return d, c, n, max_dets


def evaluate_device(dets, counts, class_names, labels, stream=None, device=None):
  """Scores n images -> {class name: (precision, aos, ap)} for each of car, pedestrian and
  cyclist that has a record anywhere, with precision and aos three 41-point curves (easy,
  moderate, hard) and ap their three 11-point APs, every value the double evaluate_object
  computes.

  dets: [n, max_dets] records (numpy DET_DTYPE, uploaded, or a CUDA tensor of those bytes) and
  counts [n]; class_names: the name of each class id; labels: read_labels of the same n images.
  Runs on `stream` (a torch.cuda.Stream, a raw cudaStream_t, or None for torch's current stream)
  and waits for it at the end, for the few KB of counts.  ValueError names the first image with a
  record that cannot be scored (a count outside [0, max_dets], a class id outside class_names, a
  non-finite box or prob, a prob outside [0, 1]); the engine writes none.

  An image holds at most 1024 scored records.  A numpy dets with a larger capacity is cut to its
  largest count, and ValueError names an image with more than 1024.  With no images at all
  nothing is scored and no class is returned, as evaluate_object writes no stats for an empty
  set."""
  import torch
  from .jpeg import _torch_stream
  n = len(labels)
  if device is None:
    device = dets.device if torch.is_tensor(dets) else torch.device('cuda', torch.cuda.current_device())
  device = torch.device(device)
  if device.type != 'cuda':
    raise ValueError('the scorer runs on a CUDA device, got %s' % (device,))
  codes = [CLASSES.index(_fold(c)) if _fold(c) in CLASSES else -1 for c in class_names]
  if not 1 <= len(codes) <= 64:
    raise ValueError('class_names must name 1 to 64 classes')
  if any(codes.count(k) > 1 for k in range(3)):
    raise ValueError('two class names name the same KITTI class: %r' % (list(class_names),))
  if n == 0:
    return {}
  if isinstance(dets, np.ndarray) and dets.ndim == 2 and dets.shape[1] > MAX_DETS:
    cnt = np.asarray(counts).reshape(-1)
    over = np.nonzero(cnt > MAX_DETS)[0]
    if len(over):
      raise ValueError('image %d: %d records, and the scorer takes at most %d per image'
                       % (over[0], cnt[over[0]], MAX_DETS))
    dets = dets[:, :max(1, int(cnt.max()) if len(cnt) else 1)]
  lib = _lib.load()
  s = _torch_stream(stream, device)
  with torch.cuda.device(device), torch.cuda.stream(s):
    d, c, nd, max_dets = _records(dets, counts, device)
    if nd != n:
      raise ValueError('%d images of records but %d of labels' % (nd, n))
    if not 1 <= max_dets <= MAX_DETS:
      raise ValueError('max_dets must be in [1, %d], got %d' % (MAX_DETS, max_dets))
    n_obj = len(labels.objs)
    objs = torch.from_numpy(labels.objs.view(np.uint8).reshape(-1)).to(device) if n_obj else None
    offsets = torch.from_numpy(labels.offsets).to(device)
    nbytes = lib.sqdet_kitti_eval_scratch_bytes(n, max_dets, n_obj)
    if nbytes < 0:
      raise _lib.SqdetError(-1, lib.sqdet_last_error().decode('utf-8', 'replace'))
    scratch = torch.empty((nbytes,), dtype=torch.uint8, device=device)
    out = torch.empty((RESULT_DTYPE.itemsize,), dtype=torch.uint8, device=device)
    cmap = np.array(codes, np.int32)
    _lib.check(lib.sqdet_kitti_eval(n, max_dets, d.data_ptr(), c.data_ptr(), len(codes),
                                    cmap.ctypes.data, objs.data_ptr() if n_obj else None,
                                    offsets.data_ptr(), n_obj, scratch.data_ptr(), nbytes,
                                    out.data_ptr(), s.cuda_stream))
    res = out.cpu().numpy().view(RESULT_DTYPE)[0]
  status = int(res['status'])
  if status != -1:
    raise ValueError('image %d: %s' % (status // 8, REASONS.get(status % 8, 'unusable records')))
  scores = {}
  for k, name in enumerate(CLASSES):
    if not res['evaluated'][k]:
      continue
    curves = [_curves(res, 3 * k + dd) for dd in range(3)]
    prec = [p for p, _ in curves]
    scores[name] = (prec, [a for _, a in curves], [average_precision(p) for p in prec])
  return scores


def _f(x):
  """printf("%f") as glibc prints it: NaN with its sign."""
  if math.isnan(x):
    return '-nan' if math.copysign(1.0, x) < 0 else 'nan'
  return '%f' % x


def _g(x):
  """std::ostream << x at its default precision (%g) as glibc prints it."""
  if math.isnan(x):
    return '-nan' if math.copysign(1.0, x) < 0 else 'nan'
  return '%g' % x


def write_stats(result_dir, scores):
  """The files evaluate_object writes into result_dir for `scores` (evaluate_device), one line
  or column per difficulty: stats_<cls>_ap.txt ('AP=' and the AP), stats_<cls>_detection.txt
  (precision[0::4]), stats_<cls>_orientation.txt (the 41 AOS values), plot/<cls>_detection.txt and
  plot/<cls>_orientation.txt (recall and the three curves, 41 rows)."""
  plot = os.path.join(result_dir, 'plot')
  os.makedirs(plot, exist_ok=True)
  for name, (prec, aos, ap) in scores.items():
    files = {
        'stats_%s_ap.txt' % name: ''.join('AP=%s\n' % _g(a) for a in ap),
        'stats_%s_detection.txt' % name: ''.join(
            ''.join(_f(p[i]) + ' ' for i in range(0, N_SAMPLE_PTS, 4)) + '\n' for p in prec),
        'stats_%s_orientation.txt' % name: ''.join(
            ''.join(_f(x) + ' ' for x in a) + '\n' for a in aos)}
    for kind, vals in (('detection', prec), ('orientation', aos)):
      files[os.path.join('plot', '%s_%s.txt' % (name, kind))] = ''.join(
          '%s %s %s %s\n' % (_f(i / (N_SAMPLE_PTS - 1.0)), _f(vals[0][i]), _f(vals[1][i]),
                             _f(vals[2][i])) for i in range(N_SAMPLE_PTS))
    for rel, text in files.items():
      with open(os.path.join(result_dir, rel), 'w') as f:
        f.write(text)
