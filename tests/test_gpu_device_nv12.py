"""sqdet_forward_frames_nv12 / ModelSkeleton.forward_device_frames_nv12: NV12 frames (a hardware
video decoder's output) already in device memory, converted, cropped, resized and mean-subtracted by
one batched launch into tensor 0, then the forward.  Every check is bitwise against
forward_device_frames on the BGR crops that oracle.nv12.nv12_to_bgr (pinned to
cv2.cvtColor(COLOR_YUV2BGR_NV12)) makes of the same bytes."""
import ctypes as C

import numpy as np
import pytest
import torch

from gpu_util import build, fetch_results
from oracle import nv12 as oracle_nv12, preproc
from squeezedet_b200 import _lib
from squeezedet_b200._lib import DeviceBuffer, PinnedArray
from squeezedet_b200.utils import synth

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_STATE = -1, -4
RESULT_ROWS = ('det_boxes', 'det_probs', 'det_class', 'dets')
FRAMES_PER_LAUNCH = 56                       # kNv12FramesPerLaunch
# How a frame sits in device memory: one tight [3H/2, W] tensor; the same with 9 padding bytes per
# row; separate luma and chroma allocations with different pitches; separate planes at odd start
# bytes with odd pitches.
LAYOUTS = ('stacked', 'padded', 'separate', 'odd')
VIDEO_DEMO_CROP = (239, 500, 1242, 375)      # frame[500:-205, 239:-439] of a 1080p frame


def small_engine(batch, device):
  """A SqueezeDet-like engine (conv+pool, fire) at 47 x 133."""
  return build([('conv', 'conv1', 64, 3, 2, 'SAME'), ('pool', 'pool1', 3, 2, 'SAME'),
                ('fire', 'fire2', 16, 64, 64)], batch, 47, 133, _lib.MATH_TF32X3_TC, device)[1]


def random_nv12(h, w, rng):
  return (rng.integers(0, 256, (h, w), dtype=np.uint8),
          rng.integers(0, 256, (h // 2, w), dtype=np.uint8))


def filled(rows, w, pitch, offset, device):
  """A CUDA uint8 view [rows, w] with rows `pitch` bytes apart, `offset` bytes into a buffer of
  0xA5 bytes that ends right after its last row."""
  store = torch.full((offset + (rows - 1) * pitch + w,), 0xA5, dtype=torch.uint8, device=device)
  return torch.as_strided(store, (rows, w), (pitch, 1), offset)


def device_nv12(luma, chroma, layout, device):
  """The frame in device memory as forward_device_frames_nv12 takes it."""
  h, w = luma.shape
  planes = np.concatenate([luma, chroma])
  if layout in ('stacked', 'padded'):
    view = filled(h + h // 2, w, w + (9 if layout == 'padded' else 0), 0, device)
    view.copy_(torch.from_numpy(planes).to(device))
    return view
  lp, cp, lo, co = (w + 16, w + 4, 0, 0) if layout == 'separate' else (w + 7, w + 3, 5, 1)
  y = filled(h, w, lp, lo, device)
  uv = filled(h // 2, w, cp, co, device)
  y.copy_(torch.from_numpy(luma).to(device))
  uv.copy_(torch.from_numpy(chroma).to(device))
  return (y, uv)


def bgr_crop(luma, chroma, crop):
  bgr = oracle_nv12.nv12_to_bgr(luma, chroma)
  if crop is None:
    return bgr
  x, y, w, h = crop
  return np.ascontiguousarray(bgr[y:y + h, x:x + w])


def bgr_reference(model, frames, crops, order, rescale):
  """(tensor 0 rows, every result buffer) of forward_device_frames on the BGR crops."""
  dev = model.gpu_id
  views = [torch.from_numpy(bgr_crop(lu, ch, c)).to(dev) for (lu, ch), c in zip(frames, crops)]
  model.forward_device_frames(views, order=order, rescale=rescale)
  torch.cuda.synchronize(dev)
  return model.read_tensor('image_input')[:len(frames)].copy(), fetch_results(model, dev)


def run_nv12(model, frames, crops, order, rescale, layouts=None, stream=None):
  dev = model.gpu_id
  layouts = layouts or [LAYOUTS[i % len(LAYOUTS)] for i in range(len(frames))]
  dframes = [device_nv12(lu, ch, lay, dev) for (lu, ch), lay in zip(frames, layouts)]
  model.forward_device_frames_nv12(dframes, crops=crops, order=order, rescale=rescale,
                                   stream=stream.cuda_stream if stream is not None else None)
  torch.cuda.synchronize(dev)
  return model.read_tensor('image_input')[:len(frames)].copy(), fetch_results(model, dev)


def assert_results(got, want, n, *what):
  """Rows [0, n) bitwise, counts of rows [n, B) zeroed (the sqdet_forward_n rules)."""
  for key in RESULT_ROWS:
    assert got[key][:n].tobytes() == want[key][:n].tobytes(), (key, n) + what
  assert np.array_equal(got['counts'][:n], want['counts'][:n]), ('counts', n) + what
  assert not got['counts'][n:].any(), ('counts past n', n) + what


# ---- 1. tensor 0 -------------------------------------------------------------------------------
# (frame h, w, crop): no crop, video_demo's crop, the four origin parities, smaller and larger
# than the 47 x 133 engine, a 1 x 1 crop, a 2 x 2 frame
T0_CASES = [(60, 150, None), (1080, 1920, VIDEO_DEMO_CROP),
            (40, 100, (2, 4, 51, 23)), (40, 100, (3, 4, 51, 23)), (40, 100, (2, 5, 51, 23)),
            (40, 100, (3, 5, 51, 23)), (20, 30, None), (100, 300, (7, 9, 1, 1)), (2, 2, None),
            (94, 266, (1, 1, 133, 47))]


@pytest.mark.parametrize('order', ['demo', 'eval'])
def test_tensor0_bitwise(order, gpu_device):
  """Every case under every layout: rows [0, n) of tensor 0 are those of forward_device_frames on
  the BGR crops bit for bit, and within 2 float32 ulp of 255 of oracle.preproc on them."""
  n = len(T0_CASES)
  model = small_engine(n, gpu_device)
  mc = model.mc
  rng = np.random.default_rng(1)
  frames = [random_nv12(h, w, rng) for h, w, _ in T0_CASES]
  crops = [c for _, _, c in T0_CASES]
  want, _ = bgr_reference(model, frames, crops, order, False)
  ulp = float(np.spacing(np.float32(255.0)))
  means = np.asarray(mc.BGR_MEANS, np.float64).reshape(3)
  for i, ((lu, ch), c) in enumerate(zip(frames, crops)):
    ref = preproc.preprocess(bgr_crop(lu, ch, c), mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, means, order)
    assert np.abs(want[i] - ref).max() <= 2 * ulp, T0_CASES[i]
  for shift in range(len(LAYOUTS)):
    layouts = [LAYOUTS[(i + shift) % len(LAYOUTS)] for i in range(n)]
    got, _ = run_nv12(model, frames, crops, order, False, layouts)
    for i in range(n):
      assert got[i].tobytes() == want[i].tobytes(), (T0_CASES[i], layouts[i])


# ---- 2. the results ------------------------------------------------------------------------------
RES_CASES = [(50, 140, None), (48, 134, None), (94, 266, (3, 1, 261, 91)), (30, 100, None),
             (200, 300, (21, 33, 130, 46)), (64, 64, (1, 0, 63, 64)), (1080, 1920, VIDEO_DEMO_CROP),
             (80, 120, (0, 7, 120, 60))]


@pytest.mark.parametrize('rescale', [False, True], ids=['plain', 'rescale'])
@pytest.mark.parametrize('order', ['demo', 'eval'])
def test_results_bitwise(order, rescale, gpu_device):
  B = len(RES_CASES)
  model = small_engine(B, gpu_device)
  stream = torch.cuda.Stream(device=gpu_device)
  rng = np.random.default_rng(2)
  frames = [random_nv12(h, w, rng) for h, w, _ in RES_CASES]
  crops = [c for _, _, c in RES_CASES]
  for n in (1, 5, B):
    want_t0, want = bgr_reference(model, frames[:n], crops[:n], order, rescale)
    got_t0, got = run_nv12(model, frames[:n], crops[:n], order, rescale, stream=stream)
    assert got_t0.tobytes() == want_t0.tobytes(), (n, order, rescale)
    assert_results(got, want, n, order, rescale)


# ---- 3. more frames than one launch holds -----------------------------------------------------------
def test_more_frames_than_one_launch(gpu_device):
  B = FRAMES_PER_LAUNCH + 4
  model = small_engine(B, gpu_device)
  rng = np.random.default_rng(3)
  shapes = [(2 * int(rng.integers(10, 60)), 2 * int(rng.integers(20, 90))) for _ in range(B)]
  frames = [random_nv12(h, w, rng) for h, w in shapes]
  crops = [None if i % 3 == 0 else (i % 2, i % 5, w // 2, h // 2) for i, (h, w) in enumerate(shapes)]
  for n, order, rescale in ((B, 'eval', True), (FRAMES_PER_LAUNCH + 1, 'demo', False)):
    want_t0, want = bgr_reference(model, frames[:n], crops[:n], order, rescale)
    got_t0, got = run_nv12(model, frames[:n], crops[:n], order, rescale)
    assert got_t0.tobytes() == want_t0.tobytes(), n
    assert_results(got, want, n, order, rescale)


# ---- 4. stream order --------------------------------------------------------------------------------
def test_frames_written_on_the_callers_stream(gpu_device):
  """The planes are written by torch kernels queued on the caller's stream behind a long-running
  kernel, and the call follows on that stream with no synchronisation in between."""
  B = 4
  model = small_engine(B, gpu_device)
  rng = np.random.default_rng(4)
  shapes = [(80, 200), (48, 134), (26, 70), (120, 300)]
  frames = [random_nv12(h, w, rng) for h, w in shapes]
  crops = [None, (1, 3, 101, 41), None, (5, 2, 250, 99)]
  _, want = bgr_reference(model, frames, crops, 'demo', True)
  srcs = [(torch.from_numpy(lu).to(gpu_device), torch.from_numpy(ch).to(gpu_device))
          for lu, ch in frames]
  dframes = [device_nv12(np.zeros_like(lu), np.zeros_like(ch), LAYOUTS[i % 4], gpu_device)
             for i, (lu, ch) in enumerate(frames)]
  torch.cuda.synchronize(gpu_device)
  stream = torch.cuda.Stream(device=gpu_device)
  with torch.cuda.stream(stream):
    torch.cuda._sleep(20_000_000)
    for d, (lu, ch) in zip(dframes, srcs):
      if isinstance(d, tuple):
        d[0].copy_(lu)
        d[1].copy_(ch)
      else:
        h = lu.shape[0]
        d[:h].copy_(lu)
        d[h:].copy_(ch)
  model.forward_device_frames_nv12(dframes, crops=crops, order='demo', rescale=True,
                                   stream=stream.cuda_stream)
  stream.synchronize()
  assert_results(fetch_results(model, gpu_device), want, B)


# ---- 5. refusals --------------------------------------------------------------------------------
def call(lib, eng, luma, lpitch, chroma, cpitch, hs, ws, crops, n=None, order=0, rescale=0):
  k = len(hs) if hs is not None else 1
  arr = lambda t, v, m=1: None if v is None else (t * (m * k))(*v)  # noqa: E731
  return lib.sqdet_forward_frames_nv12(eng, k if n is None else n, arr(C.c_void_p, luma),
                                       arr(C.c_int64, lpitch), arr(C.c_void_p, chroma),
                                       arr(C.c_int64, cpitch), arr(C.c_int32, hs),
                                       arr(C.c_int32, ws), arr(C.c_int32, crops, 4), order,
                                       rescale, None)


def test_refusals_before_device_work(gpu_device):
  """Each invalid argument is refused with no device work: tensor 0 and every result buffer stay
  bitwise as they were, and a valid call afterwards is right."""
  B = 2
  model = small_engine(B, gpu_device)
  mc = model.mc
  lib, eng = model._lib, model._engine
  rng = np.random.default_rng(5)
  frames = [random_nv12(60, 150, rng), random_nv12(30, 90, rng)]
  _, want = bgr_reference(model, frames, [None, (1, 1, 40, 20)], 'eval', True)
  feed = synth.synthetic_images(B, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, seed=6)
  model.detect(feed)
  before = fetch_results(model, gpu_device)
  H, W = 60, 150
  luma = DeviceBuffer.from_numpy(frames[0][0], gpu_device)
  chroma = DeviceBuffer.from_numpy(frames[0][1], gpu_device)
  short = DeviceBuffer(2048, gpu_device)        # the chroma plane is 30 * 150 = 4500 bytes
  pinned = PinnedArray((H, W), np.uint8)
  pageable = np.zeros((H, W), np.uint8)
  cases = [
      ('null engine', dict(eng=None), ERR_INVALID_ARG),
      ('null luma array', dict(luma=None), ERR_INVALID_ARG),
      ('null chroma array', dict(chroma=None), ERR_INVALID_ARG),
      ('null heights', dict(hs=None), ERR_INVALID_ARG),
      ('null widths', dict(ws=None), ERR_INVALID_ARG),
      ('n = 0', dict(n=0), ERR_INVALID_ARG),
      ('n > B', dict(n=B + 1), ERR_INVALID_ARG),
      ('order', dict(order=2), ERR_INVALID_ARG),
      ('null luma plane', dict(luma=[None]), ERR_INVALID_ARG),
      ('null chroma plane', dict(chroma=[None]), ERR_INVALID_ARG),
      ('zero height', dict(hs=[0]), ERR_INVALID_ARG),
      ('negative width', dict(ws=[-150]), ERR_INVALID_ARG),
      ('odd height', dict(hs=[59]), ERR_INVALID_ARG),
      ('odd width', dict(ws=[149]), ERR_INVALID_ARG),
      ('short luma pitch', dict(lpitch=[W - 1]), ERR_INVALID_ARG),
      ('short chroma pitch', dict(cpitch=[W - 1]), ERR_INVALID_ARG),
      ('empty crop', dict(crops=[0, 0, 0, 10]), ERR_INVALID_ARG),
      ('crop past the right edge', dict(crops=[1, 0, W, H]), ERR_INVALID_ARG),
      ('crop past the bottom', dict(crops=[0, 1, W, H]), ERR_INVALID_ARG),
      ('negative crop origin', dict(crops=[-1, 0, 10, 10]), ERR_INVALID_ARG),
      ('pinned host luma', dict(luma=[pinned.ptr]), ERR_INVALID_ARG),
      ('pageable host chroma', dict(chroma=[pageable.ctypes.data]), ERR_INVALID_ARG),
      ('short chroma plane', dict(chroma=[short.ptr]), ERR_INVALID_ARG),
      ('luma pitch past the buffer', dict(lpitch=[W + 1]), ERR_INVALID_ARG),
      ('pitch overflow', dict(lpitch=[1 << 62]), ERR_INVALID_ARG),
      ('chroma pitch overflow', dict(cpitch=[1 << 62]), ERR_INVALID_ARG),
  ]
  for name, kw, code in cases:
    args = dict(eng=eng, luma=[luma.ptr], lpitch=None, chroma=[chroma.ptr], cpitch=None, hs=[H],
                ws=[W], crops=None)
    args.update({k: v for k, v in kw.items() if k not in ('n', 'order')})
    assert call(lib, args['eng'], args['luma'], args['lpitch'], args['chroma'], args['cpitch'],
                args['hs'], args['ws'], args['crops'], n=kw.get('n'),
                order=kw.get('order', 0)) == code, name
    assert lib.sqdet_last_error(), name
  torch.cuda.synchronize(gpu_device)
  assert model.read_tensor('image_input').tobytes() == feed.tobytes()
  after = fetch_results(model, gpu_device)
  for key in before:
    assert after[key].tobytes() == before[key].tobytes(), key
  # an engine not yet finalized
  hd = C.c_void_p()
  conf = _lib.Config(batch_size=1, image_height=8, image_width=8, classes=3, anchors_per_grid=9,
                     top_n_detection=64, prob_thresh=0.005, nms_thresh=0.4, exp_thresh=1.0,
                     batch_norm_epsilon=1e-5, math_mode=0, max_dets=0)
  _lib.check(lib.sqdet_create(C.byref(conf), gpu_device, C.byref(hd)))
  assert call(lib, hd, [luma.ptr], None, [chroma.ptr], None, [H], [W], None) == ERR_STATE
  assert b'finalize' in lib.sqdet_last_error()
  lib.sqdet_destroy(hd)
  # still working
  _, got = run_nv12(model, frames, [None, (1, 1, 40, 20)], 'eval', True)
  assert_results(got, want, B)
  pinned.free()
  for b in (luma, chroma, short):
    b.free()


# ---- 6. a first layer without a fused pool -------------------------------------------------------
def test_first_conv_without_pool(gpu_device):
  """A lone first conv reads tensor 0 as an ordinary fp32 input: the same bits there and in the
  results."""
  B = 3
  model = build([('conv', 'conv1', 16, 3, 2, 'SAME')], B, 19, 45, _lib.MATH_FP32_SIMT,
                gpu_device)[1]
  rng = np.random.default_rng(7)
  frames = [random_nv12(h, w, rng) for h, w in ((40, 90), (1080, 1920), (18, 44))]
  crops = [(3, 1, 45, 19), VIDEO_DEMO_CROP, None]
  for order, rescale in (('demo', False), ('eval', True)):
    want_t0, want = bgr_reference(model, frames, crops, order, rescale)
    got_t0, got = run_nv12(model, frames, crops, order, rescale)
    assert got_t0.tobytes() == want_t0.tobytes(), order
    assert_results(got, want, B, order, rescale)


# ---- 7. the facade ---------------------------------------------------------------------------------
def test_facade_checks(gpu_device):
  B = 2
  model = small_engine(B, gpu_device)
  rng = np.random.default_rng(8)
  lu, ch = random_nv12(120, 300, rng)
  x = torch.from_numpy(np.concatenate([lu, ch])).to(gpu_device)
  _, want = bgr_reference(model, [(lu, ch)], [(7, 11, 200, 90)], 'demo', False)
  model.forward_device_frames_nv12([x], crops=[(7, 11, 200, 90)])
  torch.cuda.synchronize(gpu_device)
  assert_results(fetch_results(model, gpu_device), want, 1)
  bad = {
      'float32': dict(frames=[x.float()]),
      'host tensor': dict(frames=[x.cpu()]),
      'rows not a multiple of 3': dict(frames=[x[:-1]]),
      'odd width': dict(frames=[x[:, :-1]]),
      'column stride 2': dict(frames=[x[:, ::2]]),
      'three-dimensional': dict(frames=[x[:, :, None]]),
      'chroma of another width': dict(frames=[(x[:120], x[120:, :298])]),
      'chroma of another height': dict(frames=[(x[:120], x[121:])]),
      'crop outside': dict(frames=[x], crops=[(200, 0, 101, 10)]),
      'empty crop': dict(frames=[x], crops=[(0, 0, 0, 10)]),
      'crops of another count': dict(frames=[x], crops=[None, None]),
      'more than B frames': dict(frames=[x] * (B + 1)),
      'no frame': dict(frames=[]),
  }
  for name, kw in bad.items():
    with pytest.raises(ValueError):
      model.forward_device_frames_nv12(**kw)
      pytest.fail(name)
