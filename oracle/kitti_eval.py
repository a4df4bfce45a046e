"""CPU restatement of the KITTI 2-D object scorer, the reference's
src/dataset/kitti-eval/cpp/evaluate_object.cpp (`evaluate_object kitti_dir image_set result_dir n`,
run by src/dataset/kitti.py:129-136) — test infrastructure, like the rest of oracle/.
tests/test_oracle_kitti_eval.py pins the files it writes byte for byte against the binary that
oracle/build_kitti_eval.sh compiles.

  inputs     result_dir/data/<id>.txt: 16 fields per line, type, alpha (field 3), x1 y1 x2 y2
             (fields 4-7) and the score (field 15) read with %lf (loadDetections, :105-142);
             label_2/<id>.txt: type, truncation %lf, occlusion %d, alpha, x1 y1 x2 y2, 7 ignored
             fields (loadGroundtruth, :144-169).  AOS is computed unless a detection has alpha -10
             (:126-128); eval.py's lines all carry alpha 0.0
  classes    car, pedestrian, cyclist, matched with strcasecmp; a class is evaluated, and gets
             files, only if one detection anywhere has its type (:131-136, :714-778)
  cleanData  (:274-343) per class c and difficulty d: a gt of type c that passes
             height >= MIN_HEIGHT, occlusion <= MAX_OCCLUSION, truncation <= MAX_TRUNCATION is
             counted (0, n_gt += 1); a gt of type c that fails, or a Van for car or a
             Person_sitting for pedestrian, is ignored (1); anything else is skipped (-1).
             DontCare gts are the stuff boxes.  Detections of type c are 0, the others -1
  overlap    boxoverlap (:203-237): w, h of the intersection in double, 0 if either is <= 0,
             else inter / (det_area + gt_area - inter), or inter / det_area against stuff
  recall     computeStatistics without FP (:345-437): gts in file order, skipping -1; each takes
             the unassigned detection of state 0 with overlap > MIN_OVERLAP[c] and the highest
             score, the first on equal scores; none and gt 0: FN; a detection and gt 1: the
             detection is assigned, nothing counted; else TP, its score into v
  thresholds getThresholds (:239-272): v sorted descending, index i skipped while it is not the
             last and (i+2)/n - r < r - (i+1)/n, else v[i] is a threshold and r += 1/40
  PR         computeStatistics with FP per threshold t (:345-498): detections scoring < t are
             left out; each gt takes the unassigned detection of state 0 with the largest
             overlap > MIN_OVERLAP[c] (strict > against a running maximum from 0: the first on
             equal overlaps); FP = unassigned eligible detections, minus those whose stuff
             overlap exceeds MIN_OVERLAP[c]; the similarity is 0.0 plus, in gt order, each TP's
             (1 + cos(gt.alpha - det.alpha)) / 2, and counts when TP + FP > 0
  totals     eval_class (:504-581): TP, FP, FN summed over images; similarity summed in image
             order; precision[i] = tp / (double)(tp + fp), aos[i] = sim / (double)(tp + fp)
             below the threshold count, 0 above; both replaced by *max_element over [i, 41)
  files      saveStats (:171-195) and saveAndPlotPlots (:583-591): stats_<cls>_ap.txt
             `AP=` + ostream << AP (%g), stats_<cls>_detection.txt the 11 precisions [0::4] as
             "%f ", stats_<cls>_orientation.txt the 41 AOS values as "%f ", one line per
             difficulty; plot/<cls>_detection.txt and plot/<cls>_orientation.txt 41 rows of
             "%f %f %f %f\\n".  The .gp scripts and the gnuplot / ps2pdf renders are not written

Every NaN the scorer can print is a 0.0 / 0.0, the x86 default NaN with its sign bit set, which
glibc prints as "-nan".
"""
import bisect
import math
import os

CLASSES = ('car', 'pedestrian', 'cyclist')
MIN_HEIGHT = (40, 25, 25)                 # evaluate_object.cpp:28
MAX_OCCLUSION = (0, 1, 2)                 # :29
MAX_TRUNCATION = (0.15, 0.3, 0.5)         # :30
MIN_OVERLAP = (0.7, 0.5, 0.5)             # :37
NEIGHBOUR = ('van', 'person_sitting', None)   # :291-294
N_SAMPLE_PTS = 41                         # :40
NO_DETECTION = -10000000.0                # :348
MAX_THRESHOLDS = 41


def lower(name):
  """strcasecmp's folding: ASCII letters only."""
  return name.encode().lower().decode()


def read_detections(path):
  """[(type, alpha, x1, y1, x2, y2, score)] of one detection file (loadDetections, :114-138)."""
  out = []
  with open(path) as f:
    for line in f:
      t = line.split()
      if not t:
        continue
      assert len(t) == 16, (path, line)
      out.append((t[0], float(t[3]), float(t[4]), float(t[5]), float(t[6]), float(t[7]),
                  float(t[15])))
  return out


def read_groundtruth(path):
  """[(type, truncation, occlusion, alpha, x1, y1, x2, y2)] of one label file
  (loadGroundtruth, :153-165)."""
  out = []
  with open(path) as f:
    for line in f:
      t = line.split()
      if not t:
        continue
      assert len(t) == 15, (path, line)
      out.append((t[0], float(t[1]), int(t[2]), float(t[3]), float(t[4]), float(t[5]),
                  float(t[6]), float(t[7])))
  return out


def _max(a, b):            # std::max: (a < b) ? b : a
  return b if a < b else a


def _min(a, b):            # std::min: (b < a) ? b : a
  return b if b < a else a


def boxoverlap(a, b, criterion=-1):
  """boxoverlap (:203-237) of boxes (x1, y1, x2, y2): union IoU, or inter / area(a) for 0."""
  x1 = _max(a[0], b[0])
  y1 = _max(a[1], b[1])
  x2 = _min(a[2], b[2])
  y2 = _min(a[3], b[3])
  w = x2 - x1
  h = y2 - y1
  if w <= 0 or h <= 0:
    return 0.0
  inter = w * h
  a_area = (a[2] - a[0]) * (a[3] - a[1])
  b_area = (b[2] - b[0]) * (b[3] - b[1])
  if criterion == -1:
    return inter / (a_area + b_area - inter)
  return inter / a_area


def gt_state(gt, c, d):
  """cleanData's ignored_gt entry (:277-320) of gt for class c, difficulty d: 0, 1 or -1."""
  typ = lower(gt[0])
  if typ == CLASSES[c]:
    valid = 1
  elif NEIGHBOUR[c] is not None and typ == NEIGHBOUR[c]:
    valid = 0
  else:
    valid = -1
  height = gt[7] - gt[5]
  ignore = gt[2] > MAX_OCCLUSION[d] or gt[1] > MAX_TRUNCATION[d] or height < MIN_HEIGHT[d]
  if valid == 1 and not ignore:
    return 0
  if valid == 0 or (ignore and valid == 1):
    return 1
  return -1


def get_thresholds(v, n_gt):
  """getThresholds (:239-272).  At most 41: |v| <= n_gt (each score is a TP of a distinct
  counted gt), and an index i below the last is taken only while r <= (2i + 3) / (2 n); after k
  thresholds r is k/40 to within 1e-15, so a 41st threshold short of the last index would need
  (2i + 3) / (2 n) >= 1 with i <= n - 2, which cannot hold.  So at most 40 come before the last
  index, which is always taken."""
  v = sorted(v, reverse=True)
  n = float(n_gt)
  t = []
  r = 0.0
  for i in range(len(v)):
    l_recall = (i + 1) / n
    r_recall = (i + 2) / n if i < len(v) - 1 else l_recall
    if (r_recall - r) < (r - l_recall) and i < len(v) - 1:
      continue
    t.append(v[i])
    r += 1.0 / (N_SAMPLE_PTS - 1.0)
  assert len(t) <= MAX_THRESHOLDS, len(t)
  return t


class _Image:
  """One image's detections and gts, with what every class needs precomputed."""

  def __init__(self, gts, dets):
    self.gts = gts
    self.stuff = [g for g in gts if lower(g[0]) == 'dontcare']
    self.per_class = []
    for c in range(3):
      idx = [j for j, d in enumerate(dets) if lower(d[0]) == CLASSES[c]]
      boxes = [dets[j][2:6] for j in idx]
      scores = [dets[j][6] for j in idx]
      alphas = [dets[j][1] for j in idx]
      m = MIN_OVERLAP[c]
      # candidates of each gt: (k, overlap) with overlap > MIN_OVERLAP, in detection order
      cand = []
      for g in gts:
        gb = g[4:8]
        cand.append([(k, o) for k, o in ((k, boxoverlap(b, gb)) for k, b in enumerate(boxes))
                     if o > m])
      stuffed = [any(boxoverlap(b, s[4:8], 0) > m for s in self.stuff) for b in boxes]
      free = sorted(scores[k] for k in range(len(idx)) if not stuffed[k])
      self.per_class.append((scores, alphas, cand, stuffed, free))


def _recall(img, c, states):
  """computeStatistics(compute_fp=false) (:345-437): the TP scores of one image."""
  scores, _, cand, _, _ = img.per_class[c]
  assigned = set()
  v = []
  for g, st in enumerate(states):
    if st == -1:
      continue
    best, valid = -1, NO_DETECTION
    for k, _o in cand[g]:
      if k not in assigned and scores[k] > valid:
        best, valid = k, scores[k]
    if valid == NO_DETECTION:
      continue           # an FN when st == 0; not needed here
    assigned.add(best)
    if st == 0:
      v.append(scores[best])
  return v


def _pr(img, c, states, thresh, compute_aos):
  """computeStatistics(compute_fp=true) (:345-498) of one image at one threshold:
  (tp, fp, fn, similarity or -1)."""
  scores, alphas, cand, stuffed, free = img.per_class[c]
  assigned = set()
  tp = fn = 0
  delta = []
  for g, st in enumerate(states):
    if st == -1:
      continue
    best, max_overlap = -1, 0.0
    for k, o in cand[g]:
      if k not in assigned and not scores[k] < thresh and o > max_overlap:
        best, max_overlap = k, o
    if best < 0:
      if st == 0:
        fn += 1
    elif st == 1:
      assigned.add(best)
    else:
      tp += 1
      delta.append(img.gts[g][3] - alphas[best])
      assigned.add(best)
  # eligible = state 0 and not below thresh; FP = eligible, unassigned, not in a stuff box
  fp = len(free) - bisect.bisect_left(free, thresh) - sum(1 for k in assigned if not stuffed[k])
  sim = -1.0
  if compute_aos:
    if tp > 0 or fp > 0:
      sim = 0.0
      for _ in range(fp):
        sim += 0.0
      for dl in delta:
        sim += (1.0 + math.cos(dl)) / 2.0
  return tp, fp, fn, sim


NAN = float('-nan')        # 0.0 / 0.0 on x86: the default NaN, sign bit set


def _div(a, b):
  return a / b if b != 0 else NAN


def _max_element(x, i):
  """*std::max_element(x.begin() + i, x.end()): the first of the largest under operator<."""
  best = x[i]
  for y in x[i + 1:]:
    if best < y:
      best = y
  return best


def eval_class(images, c, d, compute_aos):
  """eval_class (:504-581) -> (precision[41], aos[41] or None)."""
  states = [[gt_state(g, c, d) for g in img.gts] for img in images]
  n_gt = sum(s.count(0) for s in states)
  v = []
  for img, st in zip(images, states):
    v += _recall(img, c, st)
  thresholds = get_thresholds(v, n_gt)
  tp = [0] * len(thresholds)
  fp = [0] * len(thresholds)
  fn = [0] * len(thresholds)
  sim = [0.0] * len(thresholds)
  for img, st in zip(images, states):
    for t, th in enumerate(thresholds):
      a, b, e, s = _pr(img, c, st, th, compute_aos)
      tp[t] += a
      fp[t] += b
      fn[t] += e
      if s != -1:
        sim[t] += s
  precision = [0.0] * N_SAMPLE_PTS
  aos = [0.0] * N_SAMPLE_PTS
  for i in range(len(thresholds)):
    precision[i] = _div(tp[i], float(tp[i] + fp[i]))
    aos[i] = _div(sim[i], float(tp[i] + fp[i]))
  for i in range(len(thresholds)):
    precision[i] = _max_element(precision, i)
    aos[i] = _max_element(aos, i)
  return precision, (aos if compute_aos else None)


def fmt_f(x):
  """printf("%f", x) under glibc."""
  if math.isnan(x):
    return '-nan' if math.copysign(1.0, x) < 0 else 'nan'
  return '%f' % x


def fmt_g(x):
  """std::ostream << x at default precision (%g, 6 digits) under glibc."""
  if math.isnan(x):
    return '-nan' if math.copysign(1.0, x) < 0 else 'nan'
  return '%g' % x


def ap_of(precision):
  """saveStats's AP (:176-185): the 11 samples precision[0::4] summed in order, over 11."""
  ap = 0.0
  for i in range(0, N_SAMPLE_PTS, 4):
    ap += precision[i]
  return ap / 11.0


def evaluate(gts, dets):
  """gts[i], dets[i]: image i's read_groundtruth / read_detections lists ->
  {class name: ([precision] * 3, [aos or None] * 3)} for the classes evaluated."""
  compute_aos = all(d[1] != -10 for ds in dets for d in ds)
  images = [_Image(g, d) for g, d in zip(gts, dets)]
  out = {}
  for c, name in enumerate(CLASSES):
    if not any(lower(d[0]) == name for ds in dets for d in ds):
      continue
    res = [eval_class(images, c, d, compute_aos) for d in range(3)]
    out[name] = ([r[0] for r in res], [r[1] for r in res])
  return out


def stats_files(scores):
  """{relative path: bytes} of the files evaluate_object writes for `scores` (evaluate())."""
  files = {}
  for name, (prec, aos) in scores.items():
    files['stats_%s_ap.txt' % name] = ''.join('AP=%s\n' % fmt_g(ap_of(p)) for p in prec)
    files['stats_%s_detection.txt' % name] = ''.join(
        ''.join(fmt_f(p[i]) + ' ' for i in range(0, N_SAMPLE_PTS, 4)) + '\n' for p in prec)
    curves = [('detection', prec)]
    if aos[0] is not None:
      files['stats_%s_orientation.txt' % name] = ''.join(
          ''.join(fmt_f(x) + ' ' for x in a) + '\n' for a in aos)
      curves.append(('orientation', aos))
    for kind, vals in curves:
      files[os.path.join('plot', '%s_%s.txt' % (name, kind))] = ''.join(
          '%s %s %s %s\n' % (fmt_f(i / (N_SAMPLE_PTS - 1.0)), fmt_f(vals[0][i]), fmt_f(vals[1][i]),
                             fmt_f(vals[2][i])) for i in range(N_SAMPLE_PTS))
  return {k: v.encode() for k, v in files.items()}


def run(label_dir, result_dir, image_ids):
  """evaluate_object on label_dir (kitti_dir/label_2) and result_dir/data -> the files it writes
  into result_dir, as {relative path: bytes} (nothing is written)."""
  gts = [read_groundtruth(os.path.join(label_dir, i + '.txt')) for i in image_ids]
  dets = [read_detections(os.path.join(result_dir, 'data', i + '.txt')) for i in image_ids]
  return stats_files(evaluate(gts, dets))
