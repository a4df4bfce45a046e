"""sqdet_forward_frames_u8 / ModelSkeleton.forward_device_frames: uint8 BGR frames of any size and
row pitch, already in device memory, resized and mean-subtracted by one batched launch into tensor
0, then the forward.  Every check is bitwise: the resized images against sqdet_preprocess_u8 on a
tight copy of each frame, the results against the host frames path (detect_frames) on the same
bytes."""
import ctypes as C

import numpy as np
import pytest
import torch

from gpu_util import build, fetch_results, make_net, preprocess_gpu
from oracle import preproc
from squeezedet_b200 import _lib
from squeezedet_b200._lib import DeviceBuffer, PinnedArray
from squeezedet_b200.utils import synth

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_STATE = -1, -4
RESULT_ROWS = ('det_boxes', 'det_probs', 'det_class', 'dets')
# (extra bytes per row, bytes before the first row): tight, padded rows, odd start and odd pitch
LAYOUTS = [(0, 0), (13, 0), (5, 3)]


def small_engine(batch, device):
  """A SqueezeDet-like engine (conv+pool, fire) at 47 x 133."""
  return build([('conv', 'conv1', 64, 3, 2, 'SAME'), ('pool', 'pool1', 3, 2, 'SAME'),
                ('fire', 'fire2', 16, 64, 64)], batch, 47, 133, _lib.MATH_TF32X3_TC, device)[1]


def random_frames(shapes, seed):
  rng = np.random.default_rng(seed)
  return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]


def device_view(arr, layout, device):
  """A CUDA uint8 view [h, w, 3] of arr whose rows are 3w + pad bytes apart, starting `offset`
  bytes into its storage; the bytes between rows hold 0xA5."""
  pad, offset = layout
  h, w = arr.shape[:2]
  pitch = 3 * w + pad
  store = torch.full((offset + h * pitch + 8,), 0xA5, dtype=torch.uint8, device=device)
  view = torch.as_strided(store, (h, w, 3), (pitch, 3, 1), offset)
  view.copy_(torch.from_numpy(arr).to(device))
  return view


def device_views(arrs, device, layouts=None):
  layouts = layouts or [LAYOUTS[i % len(LAYOUTS)] for i in range(len(arrs))]
  return [device_view(a, lay, device) for a, lay in zip(arrs, layouts)]


def host_reference(model, arrs, order, rescale):
  """Every result buffer after the host frames path on the same bytes."""
  model.detect_frames(arrs, order=order, rescale=rescale)
  return fetch_results(model, model.gpu_id)


def run_device(model, views, order, rescale, stream=None):
  model.forward_device_frames(views, order=order, rescale=rescale,
                              stream=stream.cuda_stream if stream is not None else None)
  torch.cuda.synchronize(model.gpu_id)
  return fetch_results(model, model.gpu_id)


def assert_results(got, want, n, *what):
  """Rows [0, n) bitwise, counts of rows [n, B) zeroed (the sqdet_forward_n rules)."""
  for key in RESULT_ROWS:
    assert got[key][:n].tobytes() == want[key][:n].tobytes(), (key, n) + what
  assert np.array_equal(got['counts'][:n], want['counts'][:n]), ('counts', n) + what
  assert not got['counts'][n:].any(), ('counts past n', n) + what


def resized(model, arrs, order):
  """sqdet_preprocess_u8 of a tight copy of each frame, stacked."""
  mc = model.mc
  return np.stack([preprocess_gpu(a, mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BGR_MEANS, order,
                                  model.gpu_id) for a in arrs])


# ---- 1. the resized images ----------------------------------------------------------------------
PRE_SHAPES = [(94, 300), (20, 50), (47, 133), (1, 1), (1, 200), (60, 1),
              (370, 1224), (720, 1280), (37, 41), (5, 7)]


@pytest.mark.parametrize('order', ['demo', 'eval'])
def test_preprocessing_bitwise(order, gpu_device):
  """Every frame shape under every layout: rows [0, n) of tensor 0 are sqdet_preprocess_u8 of a
  tight copy bit for bit, and within 2 float32 ulp of 255 of oracle.preproc."""
  n = len(PRE_SHAPES)
  model = small_engine(n, gpu_device)
  mc = model.mc
  arrs = random_frames(PRE_SHAPES, seed=1)
  want = resized(model, arrs, order)
  ulp = float(np.spacing(np.float32(255.0)))
  for i, (h, w) in enumerate(PRE_SHAPES):
    ref = preproc.preprocess(arrs[i], mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT,
                             np.asarray(mc.BGR_MEANS, np.float64).reshape(3), order)
    assert np.abs(want[i] - ref).max() <= 2 * ulp, (h, w)
  for shift in range(len(LAYOUTS)):
    layouts = [LAYOUTS[(i + shift) % len(LAYOUTS)] for i in range(n)]
    model.forward_device_frames(device_views(arrs, gpu_device, layouts), order=order)
    torch.cuda.synchronize(gpu_device)
    got = model.read_tensor('image_input')
    for i in range(n):
      assert got[i].tobytes() == want[i].tobytes(), (PRE_SHAPES[i], layouts[i])


# ---- 2. the results -------------------------------------------------------------------------------
RES_SHAPES = [(50, 140), (47, 133), (94, 266), (30, 100), (45, 131), (64, 64), (47, 132), (80, 120)]


@pytest.mark.parametrize('rescale', [False, True], ids=['plain', 'rescale'])
@pytest.mark.parametrize('order', ['demo', 'eval'])
def test_results_bitwise(order, rescale, gpu_device):
  B = len(RES_SHAPES)
  model = small_engine(B, gpu_device)
  stream = torch.cuda.Stream(device=gpu_device)
  arrs = random_frames(RES_SHAPES, seed=2)
  views = device_views(arrs, gpu_device)
  for n in (1, 7, B):
    want = host_reference(model, arrs[:n], order, rescale)
    got = run_device(model, views[:n], order, rescale, stream)
    assert_results(got, want, n, order, rescale)


def test_full_size_crop_views(gpu_device):
  """SqueezeDet 1242x375, b = 20: 1080p frames passed as video_demo's crop
  frame[500:-205, 239:-439], a 375 x 1242 view starting 717 bytes into each row."""
  B = 20
  model, _ = make_net('squeezeDet', 1242, 375, B, gpu_device)
  rng = np.random.default_rng(3)
  full = [rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8) for _ in range(B)]
  crops = [f[500:-205, 239:-439] for f in full]
  views = [torch.from_numpy(f).to(gpu_device)[500:-205, 239:-439] for f in full]
  assert views[0].shape == (375, 1242, 3) and views[0].storage_offset() == 500 * 5760 + 717
  stream = torch.cuda.Stream(device=gpu_device)
  for order, rescale in (('eval', True), ('demo', False)):
    want = host_reference(model, [np.ascontiguousarray(c) for c in crops], order, rescale)
    got = run_device(model, views, order, rescale, stream)
    assert_results(got, want, B, order, rescale)
    assert got['counts'].sum() > 0


# ---- 3. replays -------------------------------------------------------------------------------------
def test_replays_see_only_their_own_frames(gpu_device):
  """Consecutive calls on one stream, changing pointers, sizes, pitches, n, order and rescale;
  the repeated (n, rescale) pairs replay the cached forward graph."""
  B = 6
  model = small_engine(B, gpu_device)
  stream = torch.cuda.Stream(device=gpu_device)
  calls = [  # (shapes, layout, order, rescale)
      ([(60, 150)] * 6, (0, 0), 'eval', True),
      ([(40, 120), (90, 200), (47, 133), (20, 30), (47, 140), (100, 100)], (7, 1), 'eval', True),
      ([(33, 77), (47, 133), (200, 400)], (2, 2), 'demo', True),
      ([(50, 50), (47, 133), (10, 300)], (0, 0), 'demo', False),
      ([(60, 150)] * 6, (11, 3), 'eval', True),
      ([(47, 133)], (1, 1), 'eval', False),
  ]
  plans = []
  for k, (shapes, layout, order, rescale) in enumerate(calls):
    arrs = random_frames(shapes, seed=10 + k)
    plans.append((arrs, device_views(arrs, gpu_device, [layout] * len(arrs)), order, rescale,
                  host_reference(model, arrs, order, rescale)))
  for k, (arrs, views, order, rescale, want) in enumerate(plans):
    got = run_device(model, views, order, rescale, stream)
    assert_results(got, want, len(arrs), 'call', k)


# ---- 4. the two scale tables ------------------------------------------------------------------------
def test_box_scale_table_stays_apart(gpu_device):
  B = 3
  model = small_engine(B, gpu_device)
  mc = model.mc
  stream = torch.cuda.Stream(device=gpu_device)
  imgs = synth.synthetic_images(B, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, seed=4)
  x = torch.from_numpy(imgs).to(gpu_device)
  model.forward_device(x.data_ptr(), stream.cuda_stream)
  stream.synchronize()
  b0 = fetch_results(model, gpu_device)['det_boxes']
  arrs = random_frames([(60, 200), (30, 90), (47, 133)], seed=5)
  views = device_views(arrs, gpu_device)
  wants = {r: host_reference(model, arrs, 'eval', r) for r in (False, True)}
  scales = np.array([[1.25, 0.5], [0.75, 1.5], [2.0, 3.0]], np.float32)
  model.set_box_scale(scales)
  for r in (False, True, False):
    assert_results(run_device(model, views, 'eval', r, stream), wants[r], B, 'rescale', r)
  model.forward_device(x.data_ptr(), stream.cuda_stream)
  stream.synchronize()
  want = b0.copy()
  for j in range(B):
    want[j, :, 0::2] /= float(scales[j, 0])
    want[j, :, 1::2] /= float(scales[j, 1])
  assert np.array_equal(fetch_results(model, gpu_device)['det_boxes'], want)


# ---- 5. stream order --------------------------------------------------------------------------------
def test_frames_written_on_the_callers_stream(gpu_device):
  """The frames are written by torch kernels queued on the caller's stream behind a long-running
  kernel, and the call follows on that stream with no synchronisation in between."""
  B = 4
  model = small_engine(B, gpu_device)
  arrs = random_frames([(80, 200), (47, 133), (25, 70), (120, 300)], seed=6)
  want = host_reference(model, arrs, 'demo', True)
  srcs = [torch.from_numpy(a).to(gpu_device) for a in arrs]
  views = device_views([np.zeros_like(a) for a in arrs], gpu_device)
  torch.cuda.synchronize(gpu_device)
  stream = torch.cuda.Stream(device=gpu_device)
  with torch.cuda.stream(stream):
    torch.cuda._sleep(20_000_000)
    for v, s in zip(views, srcs):
      v.copy_(s)
  model.forward_device_frames(views, order='demo', rescale=True, stream=stream.cuda_stream)
  stream.synchronize()
  assert_results(fetch_results(model, gpu_device), want, B)


# ---- 6. refusals --------------------------------------------------------------------------------
def call(lib, eng, ptrs, hs, ws, pitches, n=None, order=0, rescale=0, stream=None):
  k = len(hs) if hs is not None else 1
  arr = lambda t, v: None if v is None else (t * k)(*v)  # noqa: E731
  return lib.sqdet_forward_frames_u8(eng, k if n is None else n, arr(C.c_void_p, ptrs),
                                     arr(C.c_int32, hs), arr(C.c_int32, ws),
                                     arr(C.c_int64, pitches), order, rescale, stream)


def test_refusals_before_device_work(gpu_device):
  """Each invalid argument is refused with no device work: tensor 0 keeps its images, a pending
  frames submission completes with its own records, and a valid call afterwards is right."""
  B = 2
  model = small_engine(B, gpu_device)
  mc = model.mc
  lib = model._lib
  eng = model._engine
  arrs = random_frames([(60, 150), (30, 90)], seed=7)
  want_sub = host_reference(model, arrs, 'eval', True)
  want_dev = host_reference(model, arrs, 'demo', False)
  feed = synth.synthetic_images(B, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, seed=8)
  model.detect(feed)
  good = DeviceBuffer.from_numpy(arrs[0], gpu_device)
  small = DeviceBuffer(1 << 16, gpu_device)
  pinned = PinnedArray((60, 150, 3), np.uint8)
  pageable = np.zeros((60, 150, 3), np.uint8)
  p, h, w = [good.ptr], [60], [150]
  cases = [
      ('null engine', dict(eng=None), ERR_INVALID_ARG),
      ('null frames', dict(ptrs=None), ERR_INVALID_ARG),
      ('null heights', dict(hs=None), ERR_INVALID_ARG),
      ('null widths', dict(ws=None), ERR_INVALID_ARG),
      ('n = 0', dict(n=0), ERR_INVALID_ARG),
      ('n > B', dict(n=B + 1), ERR_INVALID_ARG),
      ('order', dict(order=2), ERR_INVALID_ARG),
      ('null frame', dict(ptrs=[None]), ERR_INVALID_ARG),
      ('zero height', dict(hs=[0]), ERR_INVALID_ARG),
      ('zero width', dict(ws=[0]), ERR_INVALID_ARG),
      ('negative height', dict(hs=[-5]), ERR_INVALID_ARG),
      ('short pitch', dict(pitches=[3 * 150 - 1]), ERR_INVALID_ARG),
      ('pinned host', dict(ptrs=[pinned.ptr]), ERR_INVALID_ARG),
      ('pageable host', dict(ptrs=[pageable.ctypes.data]), ERR_INVALID_ARG),
      # 64 KiB allocated, 64 MiB claimed
      ('overlong frame', dict(ptrs=[small.ptr], hs=[1 << 14], ws=[1 << 10]), ERR_INVALID_ARG),
      ('overlong pitch', dict(ptrs=[small.ptr], hs=[2], ws=[4], pitches=[1 << 26]), ERR_INVALID_ARG),
      ('pitch overflow', dict(ptrs=[small.ptr], hs=[1 << 30], ws=[4], pitches=[1 << 62]),
       ERR_INVALID_ARG),
  ]
  dets = np.empty((B, model.max_dets), _lib.DET_DTYPE)
  counts = np.empty((B,), np.int32)
  model.submit_frames(arrs, dets.ctypes.data, counts.ctypes.data, order='eval', rescale=True)
  for name, kw, code in cases:
    args = dict(eng=eng, ptrs=p, hs=h, ws=w, pitches=None)
    args.update(kw)
    assert call(lib, args['eng'], args['ptrs'], args['hs'], args['ws'], args['pitches'],
                n=kw.get('n'), order=kw.get('order', 0)) == code, name
    assert lib.sqdet_last_error(), name
  model.wait()
  assert np.array_equal(counts, want_sub['counts'])
  for j in range(B):
    assert dets[j].tobytes() == want_sub['dets'][j].tobytes()
  assert model.read_tensor('image_input').tobytes() == feed.tobytes()
  # an engine not yet finalized
  hd = C.c_void_p()
  conf = _lib.Config(batch_size=1, image_height=8, image_width=8, classes=3, anchors_per_grid=9,
                     top_n_detection=64, prob_thresh=0.005, nms_thresh=0.4, exp_thresh=1.0,
                     batch_norm_epsilon=1e-5, math_mode=0, max_dets=0)
  _lib.check(lib.sqdet_create(C.byref(conf), gpu_device, C.byref(hd)))
  assert call(lib, hd, p, h, w, None) == ERR_STATE
  assert b'finalize' in lib.sqdet_last_error()
  lib.sqdet_destroy(hd)
  # still working: a valid call, then another pipelined submission
  got = run_device(model, device_views(arrs, gpu_device), 'demo', False,
                   torch.cuda.Stream(device=gpu_device))
  assert_results(got, want_dev, B)
  d2, c2 = model.detect_frames(arrs, order='eval', rescale=True)
  assert np.array_equal(c2, want_sub['counts']) and d2.tobytes() == want_sub['dets'].tobytes()
  pinned.free()
  small.free()
  good.free()


# ---- 7. tensor 0 ----------------------------------------------------------------------------------
def test_tensor0(gpu_device):
  """A frames submission leaves tensor 0 as it was; the device frames call writes the resized
  images into rows [0, n) and leaves rows [n, B) alone."""
  B = 4
  model = small_engine(B, gpu_device)
  mc = model.mc
  feed = synth.synthetic_images(B, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, seed=9)
  model.detect(feed)
  arrs = random_frames([(70, 160), (20, 40), (47, 133)], seed=10)
  model.detect_frames(arrs, order='eval')
  assert model.read_tensor('image_input').tobytes() == feed.tobytes()
  model.forward_device_frames(device_views(arrs, gpu_device), order='eval')
  torch.cuda.synchronize(gpu_device)
  got = model.read_tensor('image_input')
  assert got[:3].tobytes() == resized(model, arrs, 'eval').tobytes()
  assert got[3].tobytes() == feed[3].tobytes()


# ---- 8. the facade ---------------------------------------------------------------------------------
def test_facade_checks(gpu_device):
  B = 2
  model = small_engine(B, gpu_device)
  arr = random_frames([(120, 300)], seed=11)[0]
  x = torch.from_numpy(arr).to(gpu_device)
  crop = x[10:-20, 7:-13]                      # a strided view at an odd byte offset
  want = host_reference(model, [np.ascontiguousarray(arr[10:-20, 7:-13])], 'demo', False)
  model.forward_device_frames([crop])
  torch.cuda.synchronize(gpu_device)
  assert_results(fetch_results(model, gpu_device), want, 1)
  wide = torch.zeros((40, 50, 6), dtype=torch.uint8, device=gpu_device)
  bad = {
      'float32': [x.float()],
      'host tensor': [torch.from_numpy(arr)],
      'stride(2) != 1': [wide[:, :, ::2]],
      'four channels': [torch.zeros((40, 50, 4), dtype=torch.uint8, device=gpu_device)],
      'more than B frames': [x] * (B + 1),
      'no frame': [],
  }
  for name, frames in bad.items():
    with pytest.raises(ValueError):
      model.forward_device_frames(frames)
      pytest.fail(name)
