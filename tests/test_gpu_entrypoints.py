"""The reference's two inference entry points executed end to end on the GPU with synthetic
weights (SURVEY config 1 = plumbing): `demo.image_demo` (src/demo.py:161-225) and
`eval.eval_once` (src/eval.py:48-134 + src/dataset/kitti.py:100-159), on generated PNGs, checked
against the oracle pipeline: oracle pre-processing (pinned to cv2) -> torch-CPU forward ->
interpret_output -> [eval: rescale ALL boxes, eval.py:83-84] -> filter_prediction."""
import os

import numpy as np
import pytest

import oracle
from squeezedet_b200 import demo, eval as sq_eval
from squeezedet_b200 import config as cfg
from squeezedet_b200.utils import synth, viz
from squeezedet_b200.utils.util import bbox_transform
from gpu_util import TOL, make_kitti, make_net, make_png, oracle_pipeline

pytestmark = pytest.mark.gpu


def compare(got_boxes, got_probs, got_cls, want, what):
  fb, fp, fc, near_tie = want
  if near_tie:                       # an fp-level reordering of the top-64 is legitimate
    assert abs(len(got_cls) - len(fc)) <= 2, what
    return
  assert list(got_cls) == list(fc), what
  np.testing.assert_allclose(np.asarray(got_probs, np.float64), np.asarray(fp, np.float64),
                             rtol=2 * TOL, atol=1e-7, err_msg=what)
  for g, w in zip(got_boxes, fb):
    np.testing.assert_allclose(np.asarray(g, np.float64), np.asarray(w, np.float64),
                               rtol=2 * TOL, atol=2e-2, err_msg=what)


def test_image_demo_runs_and_matches_oracle(tmp_path, gpu_device):
  frames = {}
  for k, (h, w) in enumerate([(375, 1242), (370, 1224)]):
    frames['%06d.png' % k] = make_png(str(tmp_path / ('%06d.png' % k)), h, w, seed=10 + k)
  flags = demo.parse_flags(['--mode', 'image', '--checkpoint', 'synthetic',
                            '--input_path', str(tmp_path / '0*.png'),
                            '--out_dir', str(tmp_path / 'out'), '--gpu', str(gpu_device)])
  results = demo.image_demo(flags)
  assert len(results) == 2
  mc = cfg.kitti_squeezeDet_config()
  weights = synth.synthetic_weights(oracle.param_specs('squeezeDet'), seed=0)
  for path, boxes, probs, classes in results:
    name = os.path.basename(path)
    assert os.path.exists(tmp_path / 'out' / ('out_' + name))
    fb, fp, fc, near = oracle_pipeline('squeezeDet', mc, weights, frames[name], 'demo', False)
    keep = [i for i in range(len(fp)) if fp[i] > mc.PLOT_PROB_THRESH]       # demo.py:201-205
    want = ([fb[i] for i in keep], [fp[i] for i in keep], [fc[i] for i in keep], near)
    compare(boxes, probs, classes, want, name)


def test_eval_once_reference_order_files_and_scorer(tmp_path, gpu_device):
  data, ids, frames = make_kitti(tmp_path)
  flags = sq_eval.parse_flags(['--data_path', str(data), '--image_set', 'val',
                               '--eval_dir', str(tmp_path / 'eval'),
                               '--checkpoint_path', 'synthetic', '--net', 'squeezeDet',
                               '--gpu', str(gpu_device)])
  all_boxes, aps, names = sq_eval.eval_once(flags)
  mc = cfg.kitti_squeezeDet_config()
  weights = synth.synthetic_weights(oracle.param_specs('squeezeDet'), seed=0)
  det_dir = tmp_path / 'eval' / 'detection_files_0' / 'data'
  for i, idx in enumerate(ids):
    fb, fp, fc, near = oracle_pipeline('squeezeDet', mc, weights, frames[idx], 'eval', True)
    # the reference's all_boxes[c][i].append(bbox_transform(b) + [s])  (eval.py:89-91)
    want = [[] for _ in range(mc.CLASSES)]
    for c, b, s in zip(fc, fb, fp):
      want[c].append(bbox_transform(b) + [s])
    lines = (det_dir / (idx + '.txt')).read_text().splitlines()
    got_n = sum(len(all_boxes[c][i]) for c in range(mc.CLASSES))
    assert len(lines) == got_n
    if near:
      continue
    k = 0
    for c in range(mc.CLASSES):
      assert len(all_boxes[c][i]) == len(want[c]), (idx, c)
      for g, w in zip(all_boxes[c][i], want[c]):
        np.testing.assert_allclose(np.asarray(g, np.float64), np.asarray(w, np.float64),
                                   rtol=2 * TOL, atol=2e-2)
        # and the file holds exactly that record in the KITTI line format (kitti.py:116-127)
        assert lines[k] == viz.kitti_detection_line(mc.CLASS_NAMES[c], g[:4], g[4]).rstrip('\n')
        k += 1
  # the reference's unmodified scorer ran and its AP files were parsed (kitti.py:129-159)
  if not os.path.exists(sq_eval.EVAL_TOOL):
    pytest.skip('scorer binary absent: __graft_entry__.build() compiles it where /root/reference exists')
  assert aps is not None and len(aps) == 3 * mc.CLASSES and names[0] == 'car_easy'
  # evaluate_object writes stats_<class>_ap.txt for exactly the classes that occur in the detection
  # files (its eval_car / eval_pedestrian / eval_cyclist flags, evaluate_object.cpp:695-776)
  res = tmp_path / 'eval' / 'detection_files_0'
  for c, name in enumerate(mc.CLASS_NAMES):
    has = any(len(all_boxes[c][i]) > 0 for i in range(len(ids)))
    assert os.path.exists(res / ('stats_%s_ap.txt' % name)) == has, name
  assert any(os.path.exists(res / ('stats_%s_ap.txt' % n)) for n in mc.CLASS_NAMES)


def test_rescale_before_filter_changes_nothing_but_coordinates(gpu_device):
  """sqdet_set_box_scale: det_boxes come back divided by the scales (float32 division, as numpy
  does in eval.py:83-84) and the records equal the oracle filter run on those rescaled boxes."""
  m, _ = make_net('squeezeDet', 416, 128, 2, gpu_device, seed=5)
  mc = m.mc
  imgs = synth.synthetic_images(2, 128, 416, seed=6)
  b0, p0, c0 = m.detect(imgs)
  scales = np.array([[1248 / 1242.0, 384 / 375.0], [0.75, 1.5]], np.float32)
  m.set_box_scale(scales)
  b1, p1, c1, dets, counts = m.detect(imgs, want_dets=True)
  want = b0.copy()
  for j in range(2):
    want[j, :, 0::2] /= float(scales[j, 0])
    want[j, :, 1::2] /= float(scales[j, 1])
  assert np.array_equal(b1, want) and np.array_equal(p1, p0) and np.array_equal(c1, c0)
  for j in range(2):
    fb, fp, fc, src = oracle.filter_prediction(b1[j], p1[j], c1[j], mc.CLASSES,
                                               mc.TOP_N_DETECTION, mc.PROB_THRESH, mc.NMS_THRESH)
    n = int(counts[j])
    assert dets[j]['anchor'][:n].tolist() == src and dets[j]['cls'][:n].tolist() == fc
  m.set_box_scale(None)
  b2, _, _ = m.detect(imgs)
  assert np.array_equal(b2, b0)


def test_frames_rescale_and_box_scale_table_stay_apart(gpu_device):
  """`rescale` of a frames submission applies to that submission only, and the table of
  sqdet_set_box_scale to the paths fed already-resized images only."""
  m, _ = make_net('squeezeDet', 416, 128, 2, gpu_device, seed=5)
  mc = m.mc
  imgs = synth.synthetic_images(2, 128, 416, seed=6)
  rng = np.random.default_rng(7)
  # not 128 x 416, so the frames' box scales are not 1
  frames = [rng.integers(0, 256, hw + (3,), dtype=np.uint8) for hw in ((150, 500), (100, 380))]
  b0, p0, c0 = m.detect(imgs)
  launches = m.launches_per_forward()
  want_d, want_c = m.detect_frames(frames, order='eval', rescale=True)
  b1, p1, c1 = m.detect(imgs)
  assert b1.tobytes() == b0.tobytes() and p1.tobytes() == p0.tobytes()
  assert c1.tobytes() == c0.tobytes()
  assert m.launches_per_forward() == launches
  scales = np.array([[1248 / 1242.0, 384 / 375.0], [0.75, 1.5]], np.float32)
  m.set_box_scale(scales)
  assert m.launches_per_forward() == launches + 1
  m.detect_frames(frames, order='eval', rescale=False)
  b2, p2, c2 = m.detect(imgs)
  want = b0.copy()
  for j in range(2):
    want[j, :, 0::2] /= float(scales[j, 0])
    want[j, :, 1::2] /= float(scales[j, 1])
  assert np.array_equal(b2, want) and np.array_equal(p2, p0) and np.array_equal(c2, c0)
  d, c = m.detect_frames(frames, order='eval', rescale=True)
  assert np.array_equal(c, want_c) and want_c.sum() > 0
  for j in range(2):
    assert d[j][:c[j]].tobytes() == want_d[j][:c[j]].tobytes()
