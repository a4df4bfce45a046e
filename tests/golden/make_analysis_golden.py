"""Writes tests/golden/analysis_kat.npz: the reference's own analyze_detections (imported
unmodified by oracle/kitti_analysis.load_reference) on every trap of tests/analysis_traps.py and
on a few seeded random sets, so that machines without the reference checkout can check the oracle
and the GPU analysis against its output.

  python tests/golden/make_analysis_golden.py

Per set <k>: the inputs, labels_<k> (the label files' bytes, joined) with label_offsets_<k>,
dets_<k> (DET_DTYPE records, joined) with counts_<k>; and the outputs, error_<k> (the bytes of
det_error_file.txt), stats_<k> (the `out` dict's values in STAT_KEYS order) and printed_<k> (what
it printed).  names lists the sets."""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import analysis_traps as at  # noqa: E402
from oracle import kitti_analysis as ka  # noqa: E402

STAT_KEYS = ('num of detections', 'num of objects', '% correct detections', '% localization error',
             '% classification error', '% background error', '% repeated error', '% recall')
RANDOM = ((11, 12, 8), (12, 25, 40), (13, 6, 300))       # (seed, images, records per image)


def sets():
  out = [(name, labels, records) for name, labels, records in at.traps()]
  for seed, n, dets in RANDOM:
    labels, records = at.random_set(seed, n, dets)
    out.append(('random_%d' % seed, labels, records))
  return out


def main():
  arrays = {}
  names = []
  for name, labels, records in sets():
    with tempfile.TemporaryDirectory() as tmp:
      lab, det, ids = at.write_tree(tmp, labels, records)
      err = os.path.join(tmp, 'det_error_file.txt')
      out, printed = ka.run_reference(lab, det, ids, at.CLASS_NAMES, err)
      with open(err, 'rb') as f:
        error = f.read()
    texts = [t.encode() for t in labels]
    arrays['labels_' + name] = np.frombuffer(b''.join(texts), np.uint8)
    arrays['label_offsets_' + name] = np.cumsum([0] + [len(t) for t in texts]).astype(np.int64)
    arrays['dets_' + name] = np.concatenate(records)
    arrays['counts_' + name] = np.array([len(r) for r in records], np.int32)
    arrays['error_' + name] = np.frombuffer(error, np.uint8)
    arrays['stats_' + name] = np.array([out[k] for k in STAT_KEYS], np.float64)
    arrays['printed_' + name] = np.frombuffer(printed.encode(), np.uint8)
    names.append(name)
  arrays['names'] = np.array(names)
  np.savez_compressed(os.path.join(HERE, 'analysis_kat.npz'), **arrays)


if __name__ == '__main__':
  main()
