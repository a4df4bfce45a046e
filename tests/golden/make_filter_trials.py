#!/usr/bin/env python
"""Generates tests/golden/filter_trials.npz by running the reference's own
ModelSkeleton.filter_prediction (src/nn_skeleton.py:696-734), imported unmodified through
oracle/ref_import.py, on 60 seeded random cases (the inputs are regenerated from the seed by
tests/test_oracle_pinning.py, so only the outputs are stored).

  python tests/golden/make_filter_trials.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_import  # noqa: E402
from test_oracle_pinning import filter_trials  # noqa: E402


def main():
  ns = ref_import.load()
  out = {}
  for t, (boxes, probs, cls, top_n) in enumerate(filter_trials()):
    fb, fp, fc = ref_import.ref_filter_prediction(ns, boxes, probs, cls, 3, top_n, 0.005, 0.4)
    out['t%d_boxes' % t] = np.asarray(fb, np.float32).reshape(-1, 4)
    out['t%d_probs' % t] = np.asarray(fp, np.float32)
    out['t%d_cls' % t] = np.asarray(fc, np.int64)
  np.savez_compressed(os.path.join(HERE, 'filter_trials.npz'), **out)


if __name__ == '__main__':
  main()
