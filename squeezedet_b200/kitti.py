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
devkit's gnuplot scripts and renders are not written.  No engine is needed.

The detection error analysis the reference runs after the APs (analyze_detections, sqdet_kitti_
analyze) comes from the same records and labels:

  stats, lines = analyze_device(dets, counts, mc.CLASS_NAMES, labels)
  print(analysis_text(stats))
  write_error_file(det_error_file, image_ids, mc.CLASS_NAMES, lines)"""
from __future__ import annotations

import math
import os

import numpy as np

from . import _lib
from .frames import torch_stream

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


ERROR_TYPES = ('loc', 'cls', 'bg', 'missed')          # SQDET_KITTI_ERR_*
LINE_DTYPE = np.dtype([('image', '<i4'), ('type', '<i4'), ('cls', '<i4'), ('reserved', '<i4'),
                       ('x1', '<f8'), ('y1', '<f8'), ('x2', '<f8'), ('y2', '<f8'),
                       ('score', '<f8')])
assert LINE_DTYPE.itemsize == 56            # sizeof(sqdet_kitti_error_line)
COUNT_FIELDS = ('num_dets', 'num_objs', 'correct', 'loc', 'cls', 'bg', 'repeated', 'detected')
ANALYSIS_DTYPE = np.dtype([(f, '<i8') for f in COUNT_FIELDS] +
                          [('n_lines', '<i8'), ('status', '<i4'), ('reserved', '<i4')])
assert ANALYSIS_DTYPE.itemsize == 80        # sizeof(sqdet_kitti_analysis)
ANALYSIS_REASONS = dict(REASONS)
del ANALYSIS_REASONS[6]
ANALYSIS_REASONS[7] = 'a record has w < 0 or h < 0'
ANALYSIS_REASONS[8] = ('a label box of an analyzed class is not finite or fails the reference\'s '
                       'assertions x1 >= 0, x1 <= x2, y1 >= 0, y1 <= y2')


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


def _cuda_device(dets, device):
  import torch
  if device is None:
    device = dets.device if torch.is_tensor(dets) else torch.device('cuda', torch.cuda.current_device())
  device = torch.device(device)
  if device.type != 'cuda':
    raise ValueError('the scorer runs on a CUDA device, got %s' % (device,))
  return device


def _cut_capacity(dets, counts):
  """A numpy dets wider than 1024 cut to its largest count; ValueError names an image with more
  than 1024 records."""
  if isinstance(dets, np.ndarray) and dets.ndim == 2 and dets.shape[1] > MAX_DETS:
    cnt = np.asarray(counts).reshape(-1)
    over = np.nonzero(cnt > MAX_DETS)[0]
    if len(over):
      raise ValueError('image %d: %d records, and the scorer takes at most %d per image'
                       % (over[0], cnt[over[0]], MAX_DETS))
    dets = dets[:, :max(1, int(cnt.max()) if len(cnt) else 1)]
  return dets


def _upload(dets, counts, labels, device):
  """Records, counts and labels on `device`, on the current stream: (dets, counts, max_dets,
  n_objects, objs or None, offsets)."""
  import torch
  d, c, nd, max_dets = _records(dets, counts, device)
  if nd != len(labels):
    raise ValueError('%d images of records but %d of labels' % (nd, len(labels)))
  if not 1 <= max_dets <= MAX_DETS:
    raise ValueError('max_dets must be in [1, %d], got %d' % (MAX_DETS, max_dets))
  n_obj = len(labels.objs)
  objs = torch.from_numpy(labels.objs.view(np.uint8).reshape(-1)).to(device) if n_obj else None
  offsets = torch.from_numpy(labels.offsets).to(device)
  return d, c, max_dets, n_obj, objs, offsets


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
  n = len(labels)
  device = _cuda_device(dets, device)
  codes = [CLASSES.index(_fold(c)) if _fold(c) in CLASSES else -1 for c in class_names]
  if not 1 <= len(codes) <= 64:
    raise ValueError('class_names must name 1 to 64 classes')
  if any(codes.count(k) > 1 for k in range(3)):
    raise ValueError('two class names name the same KITTI class: %r' % (list(class_names),))
  if n == 0:
    return {}
  dets = _cut_capacity(dets, counts)
  lib = _lib.load()
  s = torch_stream(stream, device)
  with torch.cuda.device(device), torch.cuda.stream(s):
    d, c, max_dets, n_obj, objs, offsets = _upload(dets, counts, labels, device)
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


def analysis_stats(counts):
  """The reference's `out` dict of analyze_detections from the counts (COUNT_FIELDS): the counts
  as floats and the shares of detections and objects.  Where the reference divides by 0 and
  raises ZeroDivisionError (no counted detection, or no object), the share is float('nan')."""
  f = {k: float(counts[k]) for k in COUNT_FIELDS}

  def share(a, b):
    return a / b if b else float('nan')
  return {'num of detections': f['num_dets'], 'num of objects': f['num_objs'],
          '% correct detections': share(f['correct'], f['num_dets']),
          '% localization error': share(f['loc'], f['num_dets']),
          '% classification error': share(f['cls'], f['num_dets']),
          '% background error': share(f['bg'], f['num_dets']),
          '% repeated error': share(f['repeated'], f['num_dets']),
          '% recall': share(f['detected'], f['num_objs'])}


def analyze_device(dets, counts, class_names, labels, stream=None, device=None):
  """The reference's detection error analysis (analyze_detections, src/dataset/kitti.py:182-296)
  of n images -> (stats, lines): stats the reference's `out` dict (analysis_stats), lines a
  LINE_DTYPE array of det_error_file.txt's lines in file order (write_error_file).

  The arguments are evaluate_device's.  class_names must be distinct names among the lowercase
  'car', 'pedestrian' and 'cyclist', as in every shipped config: the reference looks the lowercased
  detection and label types up among them and fails on any other detection type.  Refused with
  ValueError before any launch.  After the launch, ValueError names the first image with a record
  evaluate_device refuses, a record with w < 0 or h < 0, or a label box of an analyzed class that
  is not finite or fails the reference's assertions (x1 >= 0, x1 <= x2, y1 >= 0, y1 <= y2).

  Runs on `stream` and waits for it at the end, for the counts and then the lines.  With no
  images nothing is launched and every count is 0."""
  import torch
  n = len(labels)
  device = _cuda_device(dets, device)
  names = list(class_names)
  if not 1 <= len(names) <= 3 or any(c not in CLASSES for c in names) or len(set(names)) < len(names):
    raise ValueError('the analysis takes distinct class names among %r, got %r'
                     % (CLASSES, names))
  codes = [CLASSES.index(c) for c in names]
  if n == 0:
    return analysis_stats(dict.fromkeys(COUNT_FIELDS, 0)), np.zeros((0,), LINE_DTYPE)
  dets = _cut_capacity(dets, counts)
  capacity = 2 * int(np.isin(labels.objs['type'], codes).sum())
  lib = _lib.load()
  s = torch_stream(stream, device)
  with torch.cuda.device(device), torch.cuda.stream(s):
    d, c, max_dets, n_obj, objs, offsets = _upload(dets, counts, labels, device)
    nbytes = lib.sqdet_kitti_analyze_scratch_bytes(n, max_dets, n_obj)
    if nbytes < 0:
      raise _lib.SqdetError(-1, lib.sqdet_last_error().decode('utf-8', 'replace'))
    scratch = torch.empty((nbytes,), dtype=torch.uint8, device=device)
    out = torch.empty((ANALYSIS_DTYPE.itemsize,), dtype=torch.uint8, device=device)
    lines = torch.empty((max(capacity, 1) * LINE_DTYPE.itemsize,), dtype=torch.uint8, device=device)
    cmap = np.array(codes, np.int32)
    _lib.check(lib.sqdet_kitti_analyze(n, max_dets, d.data_ptr(), c.data_ptr(), len(codes),
                                       cmap.ctypes.data, objs.data_ptr() if n_obj else None,
                                       offsets.data_ptr(), n_obj, scratch.data_ptr(), nbytes,
                                       out.data_ptr(), lines.data_ptr(), capacity, s.cuda_stream))
    res = out.cpu().numpy().view(ANALYSIS_DTYPE)[0]
    status = int(res['status'])
    if status != -1:
      raise ValueError('image %d: %s' % (status // 16,
                                         ANALYSIS_REASONS.get(status % 16, 'unusable records')))
    n_lines = int(res['n_lines'])
    if n_lines > capacity:         # each image writes at most G detection and G missed lines
      raise RuntimeError('%d error lines for a capacity of %d' % (n_lines, capacity))
    got = lines[:n_lines * LINE_DTYPE.itemsize].cpu().numpy().view(LINE_DTYPE)
  return analysis_stats(res), got


def analysis_text(stats):
  """The block analyze_detections prints, with its wording and '{}' formatting."""
  rows = (('Number of detections', 'num of detections'), ('Number of objects', 'num of objects'),
          ('Percentage of correct detections', '% correct detections'),
          ('Percentage of localization error', '% localization error'),
          ('Percentage of classification error', '% classification error'),
          ('Percentage of background error', '% background error'),
          ('Percentage of repeated detections', '% repeated error'), ('Recall', '% recall'))
  return 'Detection Analysis:\n' + ''.join(
      '    {}: {}\n'.format(label, stats[key]) for label, key in rows)


def error_file_text(image_ids, class_names, lines):
  """det_error_file.txt's text for analyze_device's lines: _save_detection's
  '{:s} {:s} {:.1f} {:.1f} {:.1f} {:.1f} {:s} {:.3f}' per line."""
  fmt = '{:s} {:s} {:.1f} {:.1f} {:.1f} {:.1f} {:s} {:.3f}\n'.format
  return ''.join(fmt(image_ids[i], ERROR_TYPES[t], x1, y1, x2, y2, class_names[c], sc)
                 for i, t, c, x1, y1, x2, y2, sc in zip(
                     *(lines[f].tolist() for f in ('image', 'type', 'cls', 'x1', 'y1', 'x2', 'y2',
                                                   'score'))))


def write_error_file(path, image_ids, class_names, lines):
  """Writes det_error_file.txt (error_file_text) at `path`, creating its directory."""
  os.makedirs(os.path.dirname(path) or '.', exist_ok=True)
  with open(path, 'w') as f:
    f.write(error_file_text(image_ids, class_names, lines))
