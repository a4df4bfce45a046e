"""sqdet_forward_frames / ModelSkeleton.forward_device_frames_fmt: RGB, BGRA, RGBA, planar RGB, NV12
and I420 frames already in device memory, converted, cropped, resized and mean-subtracted by one
batched launch into tensor 0, then the forward; and sqdet_forward_frames_nv12 /
forward_device_frames_nv12, which are that call for NV12.  Every check is bitwise against
forward_device_frames on the BGR crops that oracle.pixfmt.to_bgr (pinned to cv2.cvtColor) makes of
the same bytes, uploaded tight."""
import ctypes as C

import numpy as np
import pytest
import torch

from gpu_util import build, fetch_results
from oracle import pixfmt, preproc
from squeezedet_b200 import _lib
from squeezedet_b200._lib import DeviceBuffer, PinnedArray
from squeezedet_b200.utils import synth

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_STATE = -1, -4
FMT = {name: code for code, name in enumerate(pixfmt.FORMATS)}    # SQDET_FMT_*
FORMATS = ('rgb', 'bgra', 'rgba', 'rgb_planar', 'nv12', 'i420')    # every one but BGR, the reference
YUV = ('nv12', 'i420')
RESULT_ROWS = ('det_boxes', 'det_probs', 'det_class', 'dets')
# How a frame sits in device memory: the one-tensor form (packed [h, w, C], planar [3, h, w],
# stacked YUV [3h/2, w]) with tight rows; the same with 9 padding bytes per row (I420, whose
# stacked form is tight, as planes at those pitches); each plane in its own allocation at an odd
# start byte with an odd pitch; each plane in its own allocation at a padded even pitch.
LAYOUTS = ('tight', 'padded', 'odd', 'separate')
VIDEO_DEMO_CROP = (239, 500, 1242, 375)      # frame[500:-205, 239:-439] of a 1080p frame
# frames per conversion launch, as sqdet_b200.h documents them
FRAMES_PER_LAUNCH = {'bgr': 64, 'rgb': 64, 'bgra': 64, 'rgba': 64, 'rgb_planar': 45, 'nv12': 56,
                     'i420': 45}


def small_engine(batch, device):
  """A SqueezeDet-like engine (conv+pool, fire) at 47 x 133."""
  return build([('conv', 'conv1', 64, 3, 2, 'SAME'), ('pool', 'pool1', 3, 2, 'SAME'),
                ('fire', 'fire2', 16, 64, 64)], batch, 47, 133, _lib.MATH_TF32X3_TC, device)[1]


def random_planes(fmt, h, w, rng):
  """The host planes of an h x w frame in `fmt`, as oracle.pixfmt.to_bgr takes them."""
  u8 = lambda *s: rng.integers(0, 256, s, dtype=np.uint8)  # noqa: E731
  if fmt in ('bgr', 'rgb'):
    return (u8(h, w, 3),)
  if fmt in ('bgra', 'rgba'):
    return (u8(h, w, 4),)
  if fmt == 'rgb_planar':
    return (u8(h, w), u8(h, w), u8(h, w))
  if fmt == 'nv12':
    return (u8(h, w), u8(h // 2, w))
  return (u8(h, w), u8(h // 2, w // 2), u8(h // 2, w // 2))


def place(a, pitch, offset, device):
  """A CUDA view of host array a ([rows, cols] or [rows, cols, C]) with rows `pitch` bytes apart,
  `offset` bytes into a buffer of 0xA5 bytes that ends right after its last row."""
  rows, rb = a.shape[0], a[0].size
  store = torch.full((offset + (rows - 1) * pitch + rb,), 0xA5, dtype=torch.uint8, device=device)
  strides = (pitch, 1) if a.ndim == 2 else (pitch, a.shape[2], 1)
  view = torch.as_strided(store, a.shape, strides, offset)
  view.copy_(torch.from_numpy(np.ascontiguousarray(a)).to(device))
  return view


def device_frame(fmt, planes, layout, device):
  """The frame in device memory as forward_device_frames_fmt takes it."""
  rb = [p[0].size for p in planes]
  if fmt in ('bgr', 'rgb', 'bgra', 'rgba'):
    (a,) = planes
    pitch, off = {'tight': (rb[0], 0), 'padded': (rb[0] + 9, 0), 'separate': (rb[0] + 16, 0),
                  'odd': (rb[0] + 1 + rb[0] % 2, 5)}[layout]
    return place(a, pitch, off, device)
  if layout == 'odd':
    return tuple(place(p, r + 1 + r % 2, o, device) for p, r, o in zip(planes, rb, (5, 1, 3)))
  if layout == 'separate':
    return tuple(place(p, r + pad, 0, device) for p, r, pad in zip(planes, rb, (16, 4, 8)))
  if fmt == 'i420':
    if layout == 'tight':
      y, u, v = planes
      h, w = y.shape
      flat = np.concatenate([y.ravel(), u.ravel(), v.ravel()]).reshape(3 * h // 2, w)
      return torch.from_numpy(flat).to(device)
    return tuple(place(p, r + 9, 0, device) for p, r in zip(planes, rb))
  if fmt == 'nv12':
    return place(np.concatenate(planes), rb[0] + (9 if layout == 'padded' else 0), 0, device)
  # rgb_planar: one [3, h, w] tensor, rows (and so planes) at the layout's pitch
  h, w = planes[0].shape
  pitch = w + (9 if layout == 'padded' else 0)
  store = torch.full((3 * h * pitch,), 0xA5, dtype=torch.uint8, device=device)
  view = torch.as_strided(store, (3, h, w), (h * pitch, pitch, 1))
  view.copy_(torch.from_numpy(np.stack(planes)).to(device))
  return view


def bgr_crop(fmt, planes, crop):
  """The BGR crop as a fresh [h, w, 3] array, so that its strides are (3w, 3, 1) even where a
  dimension is 1 (forward_device_frames checks them)."""
  bgr = pixfmt.to_bgr(fmt, planes)
  if crop is not None:
    x, y, w, h = crop
    bgr = bgr[y:y + h, x:x + w]
  out = np.empty(bgr.shape, np.uint8)
  out[...] = bgr
  return out


def bgr_reference(model, fmt, frames, crops, order, rescale):
  """(tensor 0 rows, every result buffer) of forward_device_frames on the BGR crops."""
  dev = model.gpu_id
  views = [torch.from_numpy(bgr_crop(fmt, p, c)).to(dev) for p, c in zip(frames, crops)]
  model.forward_device_frames(views, order=order, rescale=rescale)
  torch.cuda.synchronize(dev)
  return model.read_tensor('image_input')[:len(frames)].copy(), fetch_results(model, dev)


def run_fmt(model, fmt, frames, crops, order, rescale, layouts=None, stream=None):
  dev = model.gpu_id
  layouts = layouts or [LAYOUTS[i % len(LAYOUTS)] for i in range(len(frames))]
  dframes = [device_frame(fmt, p, lay, dev) for p, lay in zip(frames, layouts)]
  model.forward_device_frames_fmt(dframes, fmt, crops=crops, order=order, rescale=rescale,
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
# than the 47 x 133 engine, a 1 x 1 crop, a 2 x 2 frame; odd sizes for the formats that take them
T0_CASES = [(60, 150, None), (1080, 1920, VIDEO_DEMO_CROP),
            (40, 100, (2, 4, 51, 23)), (40, 100, (3, 4, 51, 23)), (40, 100, (2, 5, 51, 23)),
            (40, 100, (3, 5, 51, 23)), (20, 30, None), (100, 300, (7, 9, 1, 1)), (2, 2, None),
            (94, 266, (1, 1, 133, 47))]
T0_ODD_CASES = [(47, 133, None), (31, 77, (3, 2, 40, 21)), (1, 1, None), (5, 3, (1, 1, 1, 1))]


@pytest.mark.parametrize('order', ['demo', 'eval'])
@pytest.mark.parametrize('fmt', FORMATS)
def test_tensor0_bitwise(fmt, order, gpu_device):
  """Every case under every layout: rows [0, n) of tensor 0 are those of forward_device_frames on
  the BGR crops bit for bit, and within 2 float32 ulp of 255 of oracle.preproc on them."""
  cases = T0_CASES + ([] if fmt in YUV else T0_ODD_CASES)
  n = len(cases)
  model = small_engine(n, gpu_device)
  mc = model.mc
  rng = np.random.default_rng(1)
  frames = [random_planes(fmt, h, w, rng) for h, w, _ in cases]
  crops = [c for _, _, c in cases]
  want, _ = bgr_reference(model, fmt, frames, crops, order, False)
  ulp = float(np.spacing(np.float32(255.0)))
  means = np.asarray(mc.BGR_MEANS, np.float64).reshape(3)
  for i, (p, c) in enumerate(zip(frames, crops)):
    ref = preproc.preprocess(bgr_crop(fmt, p, c), mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, means, order)
    assert np.abs(want[i] - ref).max() <= 2 * ulp, cases[i]
  for shift in range(len(LAYOUTS)):
    layouts = [LAYOUTS[(i + shift) % len(LAYOUTS)] for i in range(n)]
    got, _ = run_fmt(model, fmt, frames, crops, order, False, layouts)
    for i in range(n):
      assert got[i].tobytes() == want[i].tobytes(), (fmt, cases[i], layouts[i])


# ---- 2. the results ------------------------------------------------------------------------------
RES_CASES = [(50, 140, None), (48, 134, None), (94, 266, (3, 1, 261, 91)), (30, 100, None),
             (200, 300, (21, 33, 130, 46)), (64, 64, (1, 0, 63, 64)), (1080, 1920, VIDEO_DEMO_CROP),
             (80, 120, (0, 7, 120, 60))]


@pytest.mark.parametrize('rescale', [False, True], ids=['plain', 'rescale'])
@pytest.mark.parametrize('order', ['demo', 'eval'])
@pytest.mark.parametrize('fmt', FORMATS)
def test_results_bitwise(fmt, order, rescale, gpu_device):
  B = len(RES_CASES)
  model = small_engine(B, gpu_device)
  stream = torch.cuda.Stream(device=gpu_device)
  rng = np.random.default_rng(2)
  frames = [random_planes(fmt, h, w, rng) for h, w, _ in RES_CASES]
  crops = [c for _, _, c in RES_CASES]
  for n in (1, 5, 7, B):
    want_t0, want = bgr_reference(model, fmt, frames[:n], crops[:n], order, rescale)
    got_t0, got = run_fmt(model, fmt, frames[:n], crops[:n], order, rescale, stream=stream)
    assert got_t0.tobytes() == want_t0.tobytes(), (fmt, n, order, rescale)
    assert_results(got, want, n, fmt, order, rescale)


# ---- 3. BGR and NV12 through the new call ----------------------------------------------------------
def call(lib, eng, fmt, planes, pitches, hs, ws, crops, n=None, order=0, rescale=0):
  """sqdet_forward_frames with per-frame lists: planes/pitches of 3 entries per frame."""
  k = len(hs) if hs is not None else 1
  arr = lambda t, v, m=1: None if v is None else (t * (m * k))(*v)  # noqa: E731
  return lib.sqdet_forward_frames(eng, k if n is None else n, fmt, arr(C.c_void_p, planes, 3),
                                  arr(C.c_int64, pitches, 3), arr(C.c_int32, hs),
                                  arr(C.c_int32, ws), arr(C.c_int32, crops, 4), order, rescale,
                                  None)


def test_bgr_and_nv12_formats_equal_their_calls(gpu_device):
  """SQDET_FMT_BGR is sqdet_forward_frames_u8 (with a crop, on the crop view), SQDET_FMT_NV12 is
  sqdet_forward_frames_nv12: tensor 0 and the results bit for bit."""
  model = small_engine(3, gpu_device)
  lib, eng = model._lib, model._engine
  rng = np.random.default_rng(9)
  shapes = [(60, 150), (1080, 1920), (40, 100)]
  crops = [None, VIDEO_DEMO_CROP, (3, 5, 51, 23)]
  flat = lambda c, h, w: list(c) if c is not None else [0, 0, w, h]  # noqa: E731

  def snapshot():
    torch.cuda.synchronize(gpu_device)
    return model.read_tensor('image_input').copy(), fetch_results(model, gpu_device)

  for order, rescale in ((0, 0), (1, 1)):
    bgr = [torch.from_numpy(random_planes('bgr', h, w, rng)[0]).to(gpu_device) for h, w in shapes]
    views = [f if c is None else f[c[1]:c[1] + c[3], c[0]:c[0] + c[2]] for f, c in zip(bgr, crops)]
    _lib.check(lib.sqdet_forward_frames_u8(
        eng, 3, (C.c_void_p * 3)(*[v.data_ptr() for v in views]),
        (C.c_int32 * 3)(*[v.shape[0] for v in views]), (C.c_int32 * 3)(*[v.shape[1] for v in views]),
        (C.c_int64 * 3)(*[v.stride(0) for v in views]), order, rescale, None))
    want_t0, want = snapshot()
    planes = sum([[f.data_ptr(), None, None] for f in bgr], [])
    _lib.check(call(lib, eng, FMT['bgr'], planes, None, [h for h, _ in shapes],
                    [w for _, w in shapes], sum([flat(c, h, w) for c, (h, w) in zip(crops, shapes)], []),
                    order=order, rescale=rescale))
    got_t0, got = snapshot()
    assert got_t0.tobytes() == want_t0.tobytes(), ('bgr', order)
    assert_results(got, want, 3, 'bgr', order)

    nv = [random_planes('nv12', h, w, rng) for h, w in shapes]
    dn = [(place(y, w + 3, 1, gpu_device), place(uv, w + 5, 0, gpu_device))
          for (y, uv), (_, w) in zip(nv, shapes)]
    _lib.check(lib.sqdet_forward_frames_nv12(
        eng, 3, (C.c_void_p * 3)(*[y.data_ptr() for y, _ in dn]),
        (C.c_int64 * 3)(*[y.stride(0) for y, _ in dn]),
        (C.c_void_p * 3)(*[uv.data_ptr() for _, uv in dn]),
        (C.c_int64 * 3)(*[uv.stride(0) for _, uv in dn]), (C.c_int32 * 3)(*[h for h, _ in shapes]),
        (C.c_int32 * 3)(*[w for _, w in shapes]),
        (C.c_int32 * 12)(*sum([flat(c, h, w) for c, (h, w) in zip(crops, shapes)], [])), order,
        rescale, None))
    want_t0, want = snapshot()
    got_t0, got = run_fmt(model, 'nv12', nv, crops, ('demo', 'eval')[order], bool(rescale),
                          layouts=['separate', 'odd', 'padded'])
    assert got_t0.tobytes() == want_t0[:3].tobytes(), ('nv12', order)
    assert_results(got, want, 3, 'nv12', order)


# ---- 4. more frames than one launch holds -----------------------------------------------------------
@pytest.mark.parametrize('fmt', ['rgba', 'rgb_planar', 'nv12', 'i420'])
def test_more_frames_than_one_launch(fmt, gpu_device):
  """68 frames, and one more than the format's launch holds: two launches of 64 packed, 56 NV12
  or 45 three-plane descriptors."""
  B = max(FRAMES_PER_LAUNCH.values()) + 4
  model = small_engine(B, gpu_device)
  rng = np.random.default_rng(3)
  shapes = [(2 * int(rng.integers(10, 60)), 2 * int(rng.integers(20, 90))) for _ in range(B)]
  frames = [random_planes(fmt, h, w, rng) for h, w in shapes]
  crops = [None if i % 3 == 0 else (i % 2, i % 5, w // 2, h // 2) for i, (h, w) in enumerate(shapes)]
  for n, order, rescale in ((B, 'eval', True), (FRAMES_PER_LAUNCH[fmt] + 1, 'demo', False)):
    want_t0, want = bgr_reference(model, fmt, frames[:n], crops[:n], order, rescale)
    got_t0, got = run_fmt(model, fmt, frames[:n], crops[:n], order, rescale)
    assert got_t0.tobytes() == want_t0.tobytes(), (fmt, n)
    assert_results(got, want, n, fmt, order, rescale)


# ---- 5. stream order --------------------------------------------------------------------------------
@pytest.mark.parametrize('fmt', FORMATS)
def test_frames_written_on_the_callers_stream(fmt, gpu_device):
  """The planes are written by torch kernels queued on the caller's stream behind a long-running
  kernel, and the call follows on that stream with no synchronisation in between."""
  B = 4
  model = small_engine(B, gpu_device)
  rng = np.random.default_rng(4)
  shapes = [(80, 200), (48, 134), (26, 70), (120, 300)]
  frames = [random_planes(fmt, h, w, rng) for h, w in shapes]
  crops = [None, (1, 3, 101, 41), None, (5, 2, 250, 99)]
  _, want = bgr_reference(model, fmt, frames, crops, 'demo', True)
  dframes = [device_frame(fmt, [np.zeros_like(p) for p in planes], LAYOUTS[i % 4], gpu_device)
             for i, planes in enumerate(frames)]
  srcs = [device_frame(fmt, planes, LAYOUTS[i % 4], gpu_device) for i, planes in enumerate(frames)]
  torch.cuda.synchronize(gpu_device)
  stream = torch.cuda.Stream(device=gpu_device)
  with torch.cuda.stream(stream):
    torch.cuda._sleep(20_000_000)
    for d, s in zip(dframes, srcs):
      for dp, sp in (zip(d, s) if isinstance(d, tuple) else [(d, s)]):
        dp.copy_(sp)
  model.forward_device_frames_fmt(dframes, fmt, crops=crops, order='demo', rescale=True,
                                  stream=stream.cuda_stream)
  stream.synchronize()
  assert_results(fetch_results(model, gpu_device), want, B, fmt)


# ---- 6. a first layer without a fused pool -------------------------------------------------------
@pytest.mark.parametrize('fmt', FORMATS)
def test_first_conv_without_pool(fmt, gpu_device):
  """A lone first conv reads tensor 0 as an ordinary fp32 input: the same bits there and in the
  results."""
  B = 3
  model = build([('conv', 'conv1', 16, 3, 2, 'SAME')], B, 19, 45, _lib.MATH_FP32_SIMT,
                gpu_device)[1]
  rng = np.random.default_rng(7)
  frames = [random_planes(fmt, h, w, rng) for h, w in ((40, 90), (1080, 1920), (18, 44))]
  crops = [(3, 1, 45, 19), VIDEO_DEMO_CROP, None]
  for order, rescale in (('demo', False), ('eval', True)):
    want_t0, want = bgr_reference(model, fmt, frames, crops, order, rescale)
    got_t0, got = run_fmt(model, fmt, frames, crops, order, rescale)
    assert got_t0.tobytes() == want_t0.tobytes(), (fmt, order)
    assert_results(got, want, B, fmt, order, rescale)


# ---- 7. refusals --------------------------------------------------------------------------------
def test_refusals_before_device_work(gpu_device):
  """Each invalid argument is refused with no device work: tensor 0 and every result buffer stay
  bitwise as they were, and valid calls afterwards are right."""
  B = 2
  model = small_engine(B, gpu_device)
  mc = model.mc
  lib, eng = model._lib, model._engine
  rng = np.random.default_rng(5)
  H, W = 60, 150
  rgba = random_planes('rgba', H, W, rng)
  i420 = random_planes('i420', H, W, rng)
  _, want_rgba = bgr_reference(model, 'rgba', [rgba], [None], 'eval', True)
  _, want_i420 = bgr_reference(model, 'i420', [i420], [(1, 1, 40, 20)], 'demo', False)
  feed = synth.synthetic_images(B, mc.IMAGE_HEIGHT, mc.IMAGE_WIDTH, seed=6)
  model.detect(feed)
  before = fetch_results(model, gpu_device)
  packed = DeviceBuffer.from_numpy(rgba[0], gpu_device)
  yuv = [DeviceBuffer.from_numpy(p, gpu_device) for p in i420]
  short = DeviceBuffer(2048, gpu_device)        # U and V are 30 * 75 = 2250 bytes
  pinned = PinnedArray((H, W), np.uint8)
  pageable = np.zeros((H, W), np.uint8)
  P = [packed.ptr, None, None]
  Y = [b.ptr for b in yuv]
  cases = [
      # (name, format, planes, pitches, heights, widths, crops, n, order)
      ('unknown format', 7, P, None, [H], [W], None, None, 0),
      ('negative format', -1, P, None, [H], [W], None, None, 0),
      ('null engine', 'engine', P, None, [H], [W], None, None, 0),
      ('null planes array', 'rgba', None, None, [H], [W], None, None, 0),
      ('null heights', 'rgba', P, None, None, [W], None, None, 0),
      ('null widths', 'rgba', P, None, [H], None, None, None, 0),
      ('n = 0', 'rgba', P, None, [H], [W], None, 0, 0),
      ('n > B', 'rgba', P, None, [H], [W], None, B + 1, 0),
      ('order', 'rgba', P, None, [H], [W], None, None, 2),
      ('null packed plane', 'rgba', [None, None, None], None, [H], [W], None, None, 0),
      ('null V plane', 'i420', Y[:2] + [None], None, [H], [W], None, None, 0),
      ('null B plane', 'rgb_planar', Y[:1] * 2 + [None], None, [H], [W], None, None, 0),
      ('zero height', 'rgba', P, None, [0], [W], None, None, 0),
      ('negative width', 'rgb', P, None, [H], [-W], None, None, 0),
      ('odd I420 height', 'i420', Y, None, [H - 1], [W], None, None, 0),
      ('odd I420 width', 'i420', Y, None, [H], [W - 1], None, None, 0),
      ('RGBA pitch below 4 * width', 'rgba', P, [4 * W - 1, 0, 0], [H], [W], None, None, 0),
      ('RGB pitch below 3 * width', 'rgb', P, [3 * W - 1, 0, 0], [H], [W], None, None, 0),
      ('U pitch below half the width', 'i420', Y, [W, W // 2 - 1, W // 2], [H], [W], None, None, 0),
      ('G pitch below the width', 'rgb_planar', Y[:1] * 3, [W, W - 1, W], [H], [W], None, None, 0),
      ('empty crop', 'rgba', P, None, [H], [W], [0, 0, 0, 10], None, 0),
      ('crop past the right edge', 'i420', Y, None, [H], [W], [1, 0, W, H], None, 0),
      ('crop past the bottom', 'rgba', P, None, [H], [W], [0, 1, W, H], None, 0),
      ('negative crop origin', 'i420', Y, None, [H], [W], [-1, 0, 10, 10], None, 0),
      ('pinned host plane', 'rgb_planar', [pinned.ptr] + Y[:1] * 2, None, [H], [W], None, None, 0),
      ('pageable host U', 'i420', [Y[0], pageable.ctypes.data, Y[2]], None, [H], [W], None, None, 0),
      ('short V plane', 'i420', Y[:2] + [short.ptr], None, [H], [W], None, None, 0),
      ('pitch past the buffer', 'rgba', P, [4 * W + 1, 0, 0], [H], [W], None, None, 0),
      ('V pitch past the buffer', 'i420', Y, [W, W // 2, W // 2 + 1], [H], [W], None, None, 0),
      ('pitch overflow', 'rgba', P, [1 << 62, 0, 0], [H], [W], None, None, 0),
      ('chroma pitch overflow', 'i420', Y, [W, 1 << 62, W // 2], [H], [W], None, None, 0),
  ]
  for name, fmt, planes, pitches, hs, ws, crops, n, order in cases:
    code = fmt if isinstance(fmt, int) else FMT.get(fmt, FMT['rgba'])
    assert call(lib, None if fmt == 'engine' else eng, code, planes, pitches, hs, ws, crops, n=n,
                order=order) == ERR_INVALID_ARG, name
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
  assert call(lib, hd, FMT['i420'], Y, None, [H], [W], None) == ERR_STATE
  assert b'finalize' in lib.sqdet_last_error()
  lib.sqdet_destroy(hd)
  # still working, with the unused plane entries NULL and the pitches NULL (tight)
  _lib.check(call(lib, eng, FMT['rgba'], P, None, [H], [W], None, order=1, rescale=1))
  assert_results(fetch_results(model, gpu_device), want_rgba, 1)
  _lib.check(call(lib, eng, FMT['i420'], Y, None, [H], [W], [1, 1, 40, 20]))
  assert_results(fetch_results(model, gpu_device), want_i420, 1)
  pinned.free()
  for b in [packed, short] + yuv:
    b.free()


def call_nv12(lib, eng, luma, lpitch, chroma, cpitch, hs, ws, crops, n=None, order=0, rescale=0):
  """sqdet_forward_frames_nv12 with per-frame lists."""
  k = len(hs) if hs is not None else 1
  arr = lambda t, v, m=1: None if v is None else (t * (m * k))(*v)  # noqa: E731
  return lib.sqdet_forward_frames_nv12(eng, k if n is None else n, arr(C.c_void_p, luma),
                                       arr(C.c_int64, lpitch), arr(C.c_void_p, chroma),
                                       arr(C.c_int64, cpitch), arr(C.c_int32, hs),
                                       arr(C.c_int32, ws), arr(C.c_int32, crops, 4), order,
                                       rescale, None)


def test_nv12_entry_refusals(gpu_device):
  """sqdet_forward_frames_nv12 refuses each invalid argument with no device work: tensor 0 and
  every result buffer stay bitwise as they were, and a valid call afterwards is right."""
  B = 2
  model = small_engine(B, gpu_device)
  mc = model.mc
  lib, eng = model._lib, model._engine
  rng = np.random.default_rng(5)
  frames = [random_planes('nv12', 60, 150, rng), random_planes('nv12', 30, 90, rng)]
  crops = [None, (1, 1, 40, 20)]
  _, want = bgr_reference(model, 'nv12', frames, crops, 'eval', True)
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
      ('null engine', dict(eng=None)),
      ('null luma array', dict(luma=None)),
      ('null chroma array', dict(chroma=None)),
      ('null heights', dict(hs=None)),
      ('null widths', dict(ws=None)),
      ('n = 0', dict(n=0)),
      ('n > B', dict(n=B + 1)),
      ('order', dict(order=2)),
      ('null luma plane', dict(luma=[None])),
      ('null chroma plane', dict(chroma=[None])),
      ('zero height', dict(hs=[0])),
      ('negative width', dict(ws=[-150])),
      ('odd height', dict(hs=[59])),
      ('odd width', dict(ws=[149])),
      ('short luma pitch', dict(lpitch=[W - 1])),
      ('short chroma pitch', dict(cpitch=[W - 1])),
      ('empty crop', dict(crops=[0, 0, 0, 10])),
      ('crop past the right edge', dict(crops=[1, 0, W, H])),
      ('crop past the bottom', dict(crops=[0, 1, W, H])),
      ('negative crop origin', dict(crops=[-1, 0, 10, 10])),
      ('pinned host luma', dict(luma=[pinned.ptr])),
      ('pageable host chroma', dict(chroma=[pageable.ctypes.data])),
      ('short chroma plane', dict(chroma=[short.ptr])),
      ('luma pitch past the buffer', dict(lpitch=[W + 1])),
      ('pitch overflow', dict(lpitch=[1 << 62])),
      ('chroma pitch overflow', dict(cpitch=[1 << 62])),
  ]
  for name, kw in cases:
    args = dict(eng=eng, luma=[luma.ptr], lpitch=None, chroma=[chroma.ptr], cpitch=None, hs=[H],
                ws=[W], crops=None)
    args.update({k: v for k, v in kw.items() if k not in ('n', 'order')})
    assert call_nv12(lib, args['eng'], args['luma'], args['lpitch'], args['chroma'],
                     args['cpitch'], args['hs'], args['ws'], args['crops'], n=kw.get('n'),
                     order=kw.get('order', 0)) == ERR_INVALID_ARG, name
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
  assert call_nv12(lib, hd, [luma.ptr], None, [chroma.ptr], None, [H], [W], None) == ERR_STATE
  assert b'finalize' in lib.sqdet_last_error()
  lib.sqdet_destroy(hd)
  # still working
  _, got = run_fmt(model, 'nv12', frames, crops, 'eval', True)
  assert_results(got, want, B)
  pinned.free()
  for b in (luma, chroma, short):
    b.free()


# ---- 8. the facade ---------------------------------------------------------------------------------
def test_planar_batch_rows(gpu_device):
  """The frames of list(batch) of an [n, 3, h, w] batch go in as they are."""
  B = 3
  model = small_engine(B, gpu_device)
  rng = np.random.default_rng(10)
  batch = rng.integers(0, 256, (B, 3, 90, 160), dtype=np.uint8)
  frames = [tuple(b) for b in batch]
  crops = [None, (1, 2, 133, 47), (5, 3, 80, 40)]
  want_t0, want = bgr_reference(model, 'rgb_planar', frames, crops, 'eval', True)
  model.forward_device_frames_fmt(list(torch.from_numpy(batch).to(gpu_device)), 'rgb_planar',
                                  crops=crops, order='eval', rescale=True)
  torch.cuda.synchronize(gpu_device)
  assert model.read_tensor('image_input').tobytes() == want_t0.tobytes()
  assert_results(fetch_results(model, gpu_device), want, B)


def test_facade_checks(gpu_device):
  B = 2
  model = small_engine(B, gpu_device)
  rng = np.random.default_rng(8)
  rgba = torch.from_numpy(random_planes('rgba', 120, 300, rng)[0]).to(gpu_device)
  planar = torch.from_numpy(np.stack(random_planes('rgb_planar', 120, 300, rng))).to(gpu_device)
  y, u, v = (torch.from_numpy(p).to(gpu_device) for p in random_planes('i420', 120, 300, rng))
  i420 = torch.cat([y.reshape(-1), u.reshape(-1), v.reshape(-1)]).reshape(180, 300)
  nv12 = torch.from_numpy(np.concatenate(random_planes('nv12', 120, 300, rng))).to(gpu_device)
  model.forward_device_frames_fmt([rgba, rgba[1:, 2:]], 'rgba', crops=[(7, 11, 200, 90), None])
  model.forward_device_frames_fmt([i420, (y, u, v)], 'i420')
  model.forward_device_frames_fmt([nv12, (nv12[:120], nv12[120:])], 'nv12')
  torch.cuda.synchronize(gpu_device)
  bad = {
      'unknown format': dict(frames=[rgba], fmt='yuy2'),
      'float32': dict(frames=[rgba.float()], fmt='rgba'),
      'host tensor': dict(frames=[rgba.cpu()], fmt='rgba'),
      'three channels as rgba': dict(frames=[rgba[:, :, :3]], fmt='rgba'),
      'four channels as rgb': dict(frames=[rgba], fmt='rgb'),
      'column stride 2': dict(frames=[rgba[:, ::2]], fmt='bgra'),
      'channel stride 2': dict(frames=[rgba[:, :, ::2]], fmt='rgb'),
      'planar of 4 planes': dict(frames=[torch.cat([planar, planar[:1]])], fmt='rgb_planar'),
      'planar HWC': dict(frames=[planar.permute(1, 2, 0)], fmt='rgb_planar'),
      'planar transposed rows': dict(frames=[planar.transpose(1, 2)], fmt='rgb_planar'),
      'planar tuple of 2': dict(frames=[(planar[0], planar[1])], fmt='rgb_planar'),
      'planar planes of other sizes': dict(frames=[(planar[0], planar[1], planar[2, 1:])],
                                           fmt='rgb_planar'),
      'stacked I420 with padded rows': dict(frames=[torch.zeros(180, 310, dtype=torch.uint8,
                                                                device=gpu_device)[:, :300]],
                                            fmt='i420'),
      'I420 rows not a multiple of 3': dict(frames=[i420[:-1]], fmt='i420'),
      'odd I420 width': dict(frames=[(y[:, :-1], u, v)], fmt='i420'),
      'I420 U of another size': dict(frames=[(y, u[:, :-1], v)], fmt='i420'),
      'I420 tuple of 2': dict(frames=[(y, u)], fmt='i420'),
      'NV12 float32': dict(frames=[nv12.float()], fmt='nv12'),
      'NV12 host tensor': dict(frames=[nv12.cpu()], fmt='nv12'),
      'NV12 rows not a multiple of 3': dict(frames=[nv12[:-1]], fmt='nv12'),
      'odd NV12 width': dict(frames=[nv12[:, :-1]], fmt='nv12'),
      'NV12 column stride 2': dict(frames=[nv12[:, ::2]], fmt='nv12'),
      'three-dimensional NV12': dict(frames=[nv12[:, :, None]], fmt='nv12'),
      'NV12 chroma of another width': dict(frames=[(nv12[:120], nv12[120:, :298])], fmt='nv12'),
      'NV12 chroma of another height': dict(frames=[(nv12[:120], nv12[121:])], fmt='nv12'),
      'crop outside': dict(frames=[rgba], fmt='rgba', crops=[(200, 0, 101, 10)]),
      'empty crop': dict(frames=[i420], fmt='i420', crops=[(0, 0, 0, 10)]),
      'crops of another count': dict(frames=[rgba], fmt='rgba', crops=[None, None]),
      'more than B frames': dict(frames=[rgba] * (B + 1), fmt='rgba'),
      'no frame': dict(frames=[], fmt='rgba'),
      'order': dict(frames=[rgba], fmt='rgba', order='train'),
  }
  for name, kw in bad.items():
    with pytest.raises(ValueError):
      model.forward_device_frames_fmt(**kw)
      pytest.fail(name)


def test_nv12_method_is_the_nv12_format(gpu_device):
  """forward_device_frames_nv12 gives tensor 0 and the results of forward_device_frames_fmt with
  'nv12', which are those of the BGR crop."""
  model = small_engine(2, gpu_device)
  rng = np.random.default_rng(8)
  planes = random_planes('nv12', 120, 300, rng)
  x = torch.from_numpy(np.concatenate(planes)).to(gpu_device)
  crops = [(7, 11, 200, 90)]
  want_t0, want = bgr_reference(model, 'nv12', [planes], crops, 'demo', False)
  model.forward_device_frames_nv12([x], crops=crops)
  torch.cuda.synchronize(gpu_device)
  assert model.read_tensor('image_input')[:1].tobytes() == want_t0.tobytes()
  assert_results(fetch_results(model, gpu_device), want, 1)
  got_t0, got = run_fmt(model, 'nv12', [planes], crops, 'demo', False, layouts=['tight'])
  assert got_t0.tobytes() == want_t0.tobytes()
  assert_results(got, want, 1)


# ---- 9. a JPEG decoded on the GPU -------------------------------------------------------------------
def test_decode_jpeg_output_as_rgb_planar(gpu_device):
  """torchvision.io.decode_jpeg(device='cuda')'s [3, h, w] RGB tensor goes straight in; the
  reference is the same decoded bytes through cv2.cvtColor(COLOR_RGB2BGR)."""
  cv2 = pytest.importorskip('cv2')
  tv_io = pytest.importorskip('torchvision.io')
  rng = np.random.default_rng(11)
  im = rng.integers(0, 256, (375, 1242, 3), dtype=np.uint8)
  im[100:220, 300:700] = (40, 200, 90)
  ok, jpeg = cv2.imencode('.jpg', im)
  assert ok
  data = torch.from_numpy(jpeg.reshape(-1).copy())
  try:
    rgb = tv_io.decode_jpeg(data, device=torch.device('cuda', gpu_device))
  except (RuntimeError, NotImplementedError) as exc:
    pytest.skip('this torchvision build cannot decode JPEG on the GPU: %s' % exc)
  torch.cuda.synchronize(gpu_device)
  assert rgb.shape == (3, 375, 1242) and rgb.dtype == torch.uint8
  B = 2
  model = small_engine(B, gpu_device)
  host = rgb.cpu().numpy()
  bgr = cv2.cvtColor(np.ascontiguousarray(host.transpose(1, 2, 0)), cv2.COLOR_RGB2BGR)
  crops = [None, (239, 0, 1003, 375)]
  refs = [bgr, np.ascontiguousarray(bgr[:, 239:])]
  model.forward_device_frames([torch.from_numpy(r).to(gpu_device) for r in refs], order='eval',
                              rescale=True)
  torch.cuda.synchronize(gpu_device)
  want_t0, want = model.read_tensor('image_input').copy(), fetch_results(model, gpu_device)
  model.forward_device_frames_fmt([rgb, rgb], 'rgb_planar', crops=crops, order='eval',
                                  rescale=True)
  torch.cuda.synchronize(gpu_device)
  assert model.read_tensor('image_input').tobytes() == want_t0.tobytes()
  assert_results(fetch_results(model, gpu_device), want, B)
