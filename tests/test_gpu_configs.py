"""Parity at the BASELINE.json configurations themselves (1242x375, the batch each config
names): SqueezeDet b=20, SqueezeDet+ b=20, ResNet50+ConvDet b=8, VGG16+ConvDet b=8, both math
modes, through the reference-facing Python surface.  Oracle = the torch-CPU backend of the
restatement (oracle/torch_port.py), fp32 and fp64."""
import numpy as np
import pytest

import oracle
from oracle.torch_port import TorchForward
from squeezedet_b200 import _lib
from squeezedet_b200.utils import synth
from gpu_util import TOL, assert_boxes_close, assert_classes_match, make_mc, make_net

pytestmark = pytest.mark.gpu

CONFIGS = [('squeezeDet', 20), ('squeezeDet+', 20), ('resnet50', 8), ('vgg16', 8)]
_cache = {}


def oracle_at_config(net, batch):
  """(mc, weights, images, preds32, preds64, dets32, boxes64): computed once per net, shared by
  the two math modes."""
  key = (net, batch)
  if key in _cache:
    return _cache[key]
  mc = make_mc(net, 1242, 375, batch)
  weights = synth.synthetic_weights(oracle.param_specs(net), seed=0)
  images = synth.synthetic_images(batch, 375, 1242, seed=1234)
  out = {}
  for dt in (np.float32, np.float64):
    fwd = TorchForward(net, weights, dtype=dt)
    chunk = 2
    preds = np.concatenate([fwd(images[i:i + chunk]) for i in range(0, batch, chunk)], axis=0)
    out[dt] = (preds, oracle.interpret_output(preds, mc.ANCHOR_BOX, mc.CLASSES,
                                              mc.ANCHOR_PER_GRID, mc.IMAGE_WIDTH,
                                              mc.IMAGE_HEIGHT, mc.EXP_THRESH, dt))
    del fwd
  _cache.clear()          # keep one net's tensors alive at a time
  _cache[key] = (mc, weights, images, out[np.float32], out[np.float64])
  return _cache[key]


@pytest.mark.parametrize('math_mode', [_lib.MATH_FP32_SIMT, _lib.MATH_TF32X3_TC])
@pytest.mark.parametrize('net,batch', CONFIGS)
def test_baseline_config_detections(net, batch, math_mode, gpu_device):
  mc, weights, images, (p32, (wb, wp, wc)), (p64, (wb64, _, _)) = oracle_at_config(net, batch)
  grid = {'squeezeDet+': (22, 76)}.get(net, (24, 78))
  assert (mc.GRID_H, mc.GRID_W) == grid and mc.ANCHORS == grid[0] * grid[1] * 9
  model, model_weights = make_net(net, 1242, 375, batch, gpu_device, math_mode, seed=0)
  assert [n for n, _ in synth.model_param_specs(model)] == [n for n, _ in oracle.param_specs(net)]
  assert all(model_weights[n].tobytes() == weights[n].tobytes() for n in weights)
  boxes, probs, cls, dets, counts = model.detect(images, want_dets=True)
  assert boxes.shape == (batch, mc.ANCHORS, 4) and cls.dtype == np.int64
  # scores / boxes within 1e-4 relative of the fp32 reference semantics
  np.testing.assert_allclose(probs, wp, rtol=TOL, atol=1e-7)
  assert_boxes_close(boxes, wb, wb64)
  # class ids: exact, except where the fp64 oracle's own top-2 margin is a near tie
  assert_classes_match(cls, wc, p64, mc.ANCHOR_PER_GRID, mc.CLASSES, TOL)
  for i in range(batch):
    # (1) the GPU filter is bit-exact on the GPU's own det tensors
    fb, fp, fc, src = oracle.filter_prediction(boxes[i], probs[i], cls[i], mc.CLASSES,
                                               mc.TOP_N_DETECTION, mc.PROB_THRESH, mc.NMS_THRESH)
    n = int(counts[i])
    assert n == len(src)
    assert dets[i]['anchor'][:n].tolist() == src
    assert dets[i]['cls'][:n].tolist() == fc
    assert np.array_equal(dets[i]['prob'][:n], np.asarray(fp, np.float32))
    # (2) kept-box indices vs the oracle's own pipeline, margin-aware on the top-66 scores
    ob, op, oc, osrc = oracle.filter_prediction(wb[i], wp[i], wc[i], mc.CLASSES,
                                                mc.TOP_N_DETECTION, mc.PROB_THRESH, mc.NMS_THRESH)
    order = np.argsort(-wp[i].astype(np.float64), kind='stable')[:66]
    top = wp[i][order].astype(np.float64)
    gap = np.abs(top[:, None] - top[None, :]) <= 10 * TOL * top[:, None]
    np.fill_diagonal(gap, False)
    near_tie = {int(order[a]) for a in np.nonzero(gap.any(axis=1))[0]}
    diff = set(src) ^ set(osrc)
    assert diff <= near_tie, (net, i, sorted(diff), sorted(near_tie))
    if not near_tie:
      assert src == osrc
  # the device-resident path the benchmark times (sqdet_forward + CUDA graph) gives the same
  # records as the host-buffer call
  d2, c2 = model.detect_records(images)
  assert np.array_equal(c2, counts) and np.array_equal(d2, dets)
