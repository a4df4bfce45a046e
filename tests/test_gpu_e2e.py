"""End-to-end GPU parity through the reference-facing Python surface
(Net(mc, gpu_id) / Session.run / filter_prediction), oracle = numpy restatement."""
import numpy as np
import pytest

import oracle
from squeezedet_b200 import _lib, Session
from squeezedet_b200.nets import SqueezeDet
from squeezedet_b200.utils import synth
from gpu_util import (MODES, TOL, assert_boxes_close, assert_classes_match, make_mc, make_net,
                      rel_err)

pytestmark = pytest.mark.gpu


def oracle_run(net, mc, weights, images, dtype=np.float32, keep=None):
  preds = oracle.forward(net, weights, images, dtype=dtype, keep=keep)
  return preds, oracle.interpret_output(preds, mc.ANCHOR_BOX, mc.CLASSES, mc.ANCHOR_PER_GRID,
                                        mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.EXP_THRESH, dtype)


@pytest.mark.parametrize('math_mode', MODES)
@pytest.mark.parametrize('net,width,height', [
    ('squeezeDet', 208, 112), ('squeezeDet+', 215, 119), ('vgg16', 96, 64),
    ('resnet50', 131, 99)])
def test_layerwise_parity_small_image(net, width, height, math_mode, gpu_device):
  model, weights = make_net(net, width, height, 2, gpu_device, math_mode, seed=3)
  mc = model.mc
  assert [n for n, _ in synth.model_param_specs(model)] == [n for n, _ in oracle.param_specs(net)]
  images = synth.synthetic_images(2, height, width, seed=9)
  keep64, keep32 = {}, {}
  p64, (b64, s64, c64) = oracle_run(net, mc, weights, images, np.float64, keep64)
  p32, (b32, s32, c32) = oracle_run(net, mc, weights, images, np.float32, keep32)
  boxes, probs, cls = model.detect(images)
  checked = 0
  for name, want in keep64.items():
    if name in model._tensors:
      try:
        got = model.read_tensor(name)
      except _lib.SqdetError as exc:
        assert exc.code == -5, exc          # fused away (conv1, run in one kernel with pool1)
        continue
      assert got.shape == want.shape, name
      # (1) the bar: within 1e-4 (relative to the tensor's scale) of the fp32 reference
      assert rel_err(got, keep32[name]) < TOL, (name, rel_err(got, keep32[name]))
      # (2) quality: as close to the fp64 truth as the fp32 reference itself is (x4 slack)
      e_gpu, e_ref = rel_err(got, want), rel_err(keep32[name], want)
      assert e_gpu < max(4 * e_ref, 2e-5), (name, e_gpu, e_ref)
      checked += 1
  assert checked >= 10
  np.testing.assert_allclose(probs, s32, rtol=TOL, atol=1e-7)
  assert_boxes_close(boxes, b32, b64)
  assert_classes_match(cls, c32, p64, mc.ANCHOR_PER_GRID, mc.CLASSES, TOL)


@pytest.mark.parametrize('math_mode', MODES)
def test_full_size_squeezedet_detections(math_mode, gpu_device):
  """SqueezeDet at the BASELINE config size (1242x375), b=2: det tensors within 1e-4 of
  the fp32 oracle; filtered records identical to running the oracle's filter_prediction on
  the oracle's det tensors wherever the oracle's top-65 score gaps exceed the tolerance."""
  net = 'squeezeDet'
  model, weights = make_net(net, 1242, 375, 2, gpu_device, math_mode, seed=0)
  mc = model.mc
  assert (mc.GRID_H, mc.GRID_W, mc.ANCHORS) == (24, 78, 16848)
  images = synth.synthetic_images(2, 375, 1242, seed=1234)
  _, (wb, wp, wc) = oracle_run(net, mc, weights, images, np.float32)
  p64, (wb64, _, _) = oracle_run(net, mc, weights, images, np.float64)
  boxes, probs, cls, dets, counts = model.detect(images, want_dets=True)
  assert boxes.dtype == np.float32 and probs.dtype == np.float32 and cls.dtype == np.int64
  np.testing.assert_allclose(probs, wp, rtol=TOL, atol=1e-7)
  assert_boxes_close(boxes, wb, wb64)
  assert_classes_match(cls, wc, p64, mc.ANCHOR_PER_GRID, mc.CLASSES, TOL)
  for i in range(2):
    # (1) bit-exact: GPU filter on the GPU's own det tensors == oracle filter on them
    fb, fp, fc, src = oracle.filter_prediction(boxes[i], probs[i], cls[i], mc.CLASSES,
                                               mc.TOP_N_DETECTION, mc.PROB_THRESH, mc.NMS_THRESH)
    n = int(counts[i])
    assert n == len(src)
    assert dets[i]['anchor'][:n].tolist() == src
    assert dets[i]['cls'][:n].tolist() == fc
    assert np.array_equal(dets[i]['prob'][:n], np.asarray(fp, np.float32))
    # (2) margin-aware vs the oracle's own pipeline: kept-box indices must agree except for
    # anchors whose oracle score sits within 10*TOL of another top-66 score (a near tie whose
    # order fp noise may legitimately flip)
    ob, op, oc, osrc = oracle.filter_prediction(wb[i], wp[i], wc[i], mc.CLASSES,
                                                mc.TOP_N_DETECTION, mc.PROB_THRESH, mc.NMS_THRESH)
    order = np.argsort(-wp[i].astype(np.float64), kind='stable')[:66]
    top = wp[i][order].astype(np.float64)
    near_tie = set()
    for a in range(len(top)):
      for b in range(len(top)):
        if a != b and abs(top[a] - top[b]) <= 10 * TOL * top[a]:
          near_tie.add(int(order[a]))
    diff = set(src) ^ set(osrc)
    assert diff <= near_tie, (sorted(diff), sorted(near_tie))
    if not near_tie:
      assert src == osrc


@pytest.mark.parametrize('math_mode', MODES)
def test_session_run_contract_and_filter_prediction(math_mode, gpu_device):
  """The reference call shape: sess.run([det_boxes, det_probs, det_class], feed_dict) then
  model.filter_prediction per image (demo.py:193-199)."""
  model, _ = make_net('squeezeDet', 416, 128, 1, gpu_device, math_mode, seed=5)
  mc = model.mc
  img = synth.synthetic_images(1, 128, 416, seed=6)[0]
  with Session() as sess:
    det_boxes, det_probs, det_class = sess.run(
        [model.det_boxes, model.det_probs, model.det_class],
        feed_dict={model.image_input: [img]})
  A = mc.ANCHORS
  assert det_boxes.shape == (1, A, 4) and det_probs.shape == (1, A) and det_class.shape == (1, A)
  final_boxes, final_probs, final_class = model.filter_prediction(
      det_boxes[0], det_probs[0], det_class[0])
  ob, op, oc, _ = oracle.filter_prediction(det_boxes[0], det_probs[0], det_class[0], mc.CLASSES,
                                           mc.TOP_N_DETECTION, mc.PROB_THRESH, mc.NMS_THRESH)
  assert final_class == oc
  assert all(np.array_equal(a, b) for a, b in zip(final_boxes, ob))
  assert [float(x) for x in final_probs] == [float(x) for x in op]
  assert isinstance(final_boxes, list) and isinstance(final_class[0], int)
  # one-pass variant gives the same triple
  fb2, fp2, fc2 = model.detect_filtered([img])[0]
  assert fc2 == final_class and all(np.array_equal(a, b) for a, b in zip(fb2, final_boxes))
  # static feed shape, like the TF placeholder
  with pytest.raises(ValueError):
    model.detect(np.zeros((2, 128, 416, 3), np.float32))
  # counters follow the reference formulas (nn_skeleton.py:549-561)
  assert sum(v for _, v in model.model_size_counter) == 2082120
  assert len(model.model_params) == 64


@pytest.mark.parametrize('math_mode', MODES)
def test_forward_profiled_matches_detect(math_mode, gpu_device):
  """sqdet_forward_profiled: one time per op_table() row, and the same det tensors and filtered
  records as sqdet_detect on the same images.  Every result buffer is overwritten with 0xff bytes
  first, so a skipped interpret or filter launch shows.  VGG16 fuses no pool into its producer, so
  every op issues work and every time is positive."""
  model, _ = make_net('vgg16', 96, 64, 2, gpu_device, math_mode, seed=5)
  images = synth.synthetic_images(2, 64, 96, seed=6)
  want = dict(zip(('det_boxes', 'det_probs', 'det_class', 'dets', 'counts'),
                  model.detect(images, want_dets=True)))
  assert want['counts'].sum() > 0
  lib, res = model._lib, model.results_device()
  for key, arr in want.items():
    fill = np.full(arr.nbytes, 0xff, np.uint8)
    _lib.check(lib.sqdet_memcpy_h2d(res[key], fill.ctypes.data, fill.nbytes, None))
  _lib.check(lib.sqdet_stream_sync(gpu_device, None))
  x = _lib.DeviceBuffer.from_numpy(images, gpu_device)
  rows = model.forward_profiled(x.ptr)
  table = model.op_table()
  assert len(rows) == lib.sqdet_num_ops(model._engine) == len(table)
  assert [row[0] for row, _ in rows] == [row[0] for row in table]
  assert all(ms > 0 for _, ms in rows), rows
  for key, arr in want.items():
    got = np.empty_like(arr)
    _lib.check(lib.sqdet_memcpy_d2h(got.ctypes.data, res[key], got.nbytes, None))
    _lib.check(lib.sqdet_stream_sync(gpu_device, None))
    assert got.tobytes() == arr.tobytes(), key


def test_batch_invariance_and_determinism(gpu_device):
  m1, _ = make_net('squeezeDet', 320, 96, 1, gpu_device, seed=8)
  m3, _ = make_net('squeezeDet', 320, 96, 3, gpu_device, seed=8)
  imgs = synth.synthetic_images(3, 96, 320, seed=4)
  b3, p3, c3 = m3.detect(imgs)
  b3b, p3b, c3b = m3.detect(imgs)
  assert np.array_equal(p3, p3b) and np.array_equal(b3, b3b) and np.array_equal(c3, c3b)
  for i in range(3):
    b1, p1, c1 = m1.detect(imgs[i:i + 1])
    assert np.array_equal(p1[0], p3[i]) and np.array_equal(b1[0], b3[i])


def test_set_param_errors(gpu_device):
  mc = make_mc('squeezeDet', 160, 96, 1)
  m = SqueezeDet(mc, gpu_device)
  with pytest.raises(_lib.SqdetError):
    m.set_param('conv1/kernels', np.zeros((3, 3, 3, 63), np.float32))
  with pytest.raises(_lib.SqdetError):
    m.set_param('nope/kernels', np.zeros((1,), np.float32))


def test_pipelined_submit_and_uint8_input(gpu_device):
  """sqdet_submit/sqdet_wait (depth-2 pipeline) and the uint8 path: same records as the
  synchronous fp32 feed of `im - BGR_MEANS` (demo.py:187-190)."""
  m, _ = make_net('squeezeDet', 320, 96, 2, gpu_device, seed=8)
  mc = m.mc
  rng = np.random.default_rng(3)
  batches = [rng.integers(0, 256, (2, 96, 320, 3), dtype=np.uint8) for _ in range(4)]
  feeds = [(b.astype(np.float32) - np.asarray(mc.BGR_MEANS)).astype(np.float32) for b in batches]
  want = [m.detect_records(f) for f in feeds]
  # uint8 path, synchronous convenience
  for b, (wd, wc) in zip(batches, want):
    d, c = m.detect_u8(b)
    assert np.array_equal(c, wc) and np.array_equal(d, wd)
  # pipelined, two in flight, mixing input types
  outs = [(np.empty((2, m.max_dets), _lib.DET_DTYPE), np.empty((2,), np.int32)) for _ in batches]
  keep_alive = []
  for i in range(len(batches)):
    src = np.ascontiguousarray(batches[i]) if i % 2 == 0 else np.ascontiguousarray(feeds[i])
    keep_alive.append(src)
    m.submit(src.ctypes.data, outs[i][0].ctypes.data, outs[i][1].ctypes.data,
             _lib.IMG_U8 if i % 2 == 0 else _lib.IMG_F32)
    if i >= 1:
      m.wait()
  m.wait()
  for (d, c), (wd, wc) in zip(outs, want):
    assert np.array_equal(c, wc) and np.array_equal(d, wd)
  with pytest.raises(_lib.SqdetError):
    m.wait()                                   # nothing in flight
