"""sqdet_draw_dets / ModelSkeleton.draw_detections_device: detections drawn onto frames in device
memory, checked bitwise.  BGR frames against cv2 (utils.viz.draw_box) on a host copy; RGB, BGRA, RGBA
and planar RGB against draw_box on cv2.cvtColor's BGR frame, written back in the frame's channel
order; NV12 and I420 against oracle.draw.  Every byte of every plane, padding included, is compared,
so bytes outside the canvas must be unchanged."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import draw, pixfmt
from squeezedet_b200 import _lib, demo
from squeezedet_b200.utils.util import tile_grid
from squeezedet_b200.utils.viz import draw_box

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip('cv2')

ERR_INVALID_ARG = -1
NAMES = ('car', 'pedestrian', 'cyclist')
BGR = np.array([(255, 191, 0), (255, 0, 191), (0, 191, 255)], np.uint8)
THRESH = 0.4
PACKED = {'bgr': 3, 'rgb': 3, 'bgra': 4, 'rgba': 4}


def plane_shapes(fmt, h, w):
  """(rows, row bytes) of each plane of an h x w frame."""
  if fmt in PACKED:
    return [(h, PACKED[fmt] * w)]
  if fmt == 'rgb_planar':
    return [(h, w)] * 3
  if fmt == 'nv12':
    return [(h, w), (h // 2, w)]
  return [(h, w), (h // 2, w // 2), (h // 2, w // 2)]


class Frame:
  """A random frame on the device, each plane inside a buffer of `pad` extra bytes per row."""

  def __init__(self, fmt, h, w, rng, device, pad):
    self.fmt, self.h, self.w = fmt, h, w
    self.bufs = [torch.from_numpy(rng.integers(0, 256, (r, b + pad), dtype=np.uint8)).to(device)
                 for r, b in plane_shapes(fmt, h, w)]
    self.before = [b.cpu().numpy() for b in self.bufs]

  def ptrs(self):
    return [b.data_ptr() for b in self.bufs] + [None] * (3 - len(self.bufs))

  def pitches(self):
    return [b.stride(0) for b in self.bufs] + [0] * (3 - len(self.bufs))

  def now(self):
    return [b.cpu().numpy() for b in self.bufs]

  def expected(self, crop, dets, count):
    """The planes (padding included) after drawing, as the contract says."""
    x, y, cw, ch = crop
    out = [b.copy() for b in self.before]
    planes = [b[:r, :n] for b, (r, n) in zip(out, plane_shapes(self.fmt, self.h, self.w))]
    if self.fmt in ('nv12', 'i420'):
      u, v = ((planes[1][:, 0::2], planes[1][:, 1::2]) if self.fmt == 'nv12'
              else (planes[1], planes[2]))
      draw.draw_yuv420(planes[0], u, v, crop, dets, count, NAMES, BGR, THRESH, 0.3)
      return out
    if self.fmt == 'rgb_planar':
      bgr = pixfmt.to_bgr('rgb_planar', planes)
    else:
      bgr = pixfmt.to_bgr(self.fmt, [planes[0].reshape(self.h, self.w, PACKED[self.fmt])])
    cv2_draw(bgr[y:y + ch, x:x + cw], dets, count)
    if self.fmt == 'rgb_planar':
      for p, c in zip(planes, (2, 1, 0)):
        p[:] = bgr[..., c]
    else:
      f = planes[0].reshape(self.h, self.w, PACKED[self.fmt])      # a copy when rows are padded
      f[..., list(pixfmt._PACKED[self.fmt][1])] = bgr
      planes[0][:] = f.reshape(planes[0].shape)
    return out


def cv2_draw(canvas, dets, count):
  """demo.draw_detections' selection + viz.draw_box on a BGR canvas (a view works), record by
  record.  Records draw_box cannot take follow the contract: an out-of-range class or a
  non-finite corner is skipped, a prob outside [0, 1] draws its rectangle alone."""
  cdict = {n: tuple(int(v) for v in c) for n, c in zip(NAMES, BGR)}
  for r in dets[:max(count, 0)]:
    prob, cls = np.float32(r['prob']), int(r['cls'])
    corners = draw.box_corners(r['cx'], r['cy'], r['w'], r['h'])
    if not prob > THRESH or not 0 <= cls < len(NAMES) or corners is None:
      continue
    if 0 <= prob <= 1:
      draw_box(canvas, [np.array([r['cx'], r['cy'], r['w'], r['h']], np.float32)],
               [NAMES[cls] + ': (%.2f)' % prob], cdict=cdict)
    else:
      cv2.rectangle(canvas, tuple(corners[:2]), tuple(corners[2:]), cdict[NAMES[cls]], 1)
  return canvas


def records(rng, n, h, w):
  d = np.zeros(n, _lib.DET_DTYPE)
  d['cls'] = rng.integers(0, 3, n)
  d['prob'] = rng.uniform(0, 1, n).astype(np.float32)
  d['cx'] = rng.uniform(-0.3 * w, 1.3 * w, n)
  d['cy'] = rng.uniform(-0.3 * h, 1.3 * h, n)
  d['w'] = rng.uniform(0, 0.7 * w + 4, n)
  d['h'] = rng.uniform(0, 0.7 * h + 4, n)
  return d


def style(classes=3, names=NAMES, font_scale=0.3, bgr=BGR):
  enc = [None if s is None else s.encode('ascii') for s in names]
  keep = ((C.c_char_p * len(enc))(*enc), (C.c_uint8 * bgr.size)(*bgr.reshape(-1).tolist()))
  st = _lib.DrawStyle(classes, keep[0], keep[1], THRESH, font_scale)
  st._keep = keep
  return st


def call(frames, fmt, crops, dets_dev, counts_dev, max_dets, st=None, stream=None,
         pitches=None, n=None):
  n = len(frames) if n is None else n
  ptrs = [p for f in frames for p in f.ptrs()]
  pit = [p for f in frames for p in f.pitches()] if pitches is None else pitches
  flat = None if crops is None else (C.c_int32 * (4 * len(crops)))(*[v for c in crops for v in c])
  return _lib.load().sqdet_draw_dets(
      n, pixfmt.FORMATS.index(fmt), (C.c_void_p * len(ptrs))(*ptrs), (C.c_int64 * len(pit))(*pit),
      (C.c_int32 * len(frames))(*[f.h for f in frames]),
      (C.c_int32 * len(frames))(*[f.w for f in frames]), flat, dets_dev, counts_dev, max_dets,
      C.byref(style() if st is None else st), stream)


def upload(dets, counts, device):
  d = torch.from_numpy(np.ascontiguousarray(dets).view(np.uint8).copy()).to(device)
  c = torch.from_numpy(np.asarray(counts, np.int32)).to(device)
  return d, c


@pytest.mark.parametrize('fmt', pixfmt.FORMATS)
@pytest.mark.parametrize('cropped', [False, True], ids=['whole', 'crops'])
def test_draw_bitwise(fmt, cropped, gpu_device):
  """Five frames of different sizes (odd origins, padded pitches, a 2x2 frame), random records
  past every edge, overlaps of different colours, and counts of max_dets, fewer, 0 and -1."""
  rng = np.random.default_rng(pixfmt.FORMATS.index(fmt) * 2 + cropped)
  sizes = [(60, 90), (38, 124), (2, 2), (120, 64), (16, 20)]
  frames = [Frame(fmt, h, w, rng, gpu_device, pad) for (h, w), pad in zip(sizes, (0, 13, 1, 64, 3))]
  crops = []
  for f in frames:
    if cropped and f.h > 2:
      x, y = int(rng.integers(0, 8)) | 1, int(rng.integers(0, 8)) | 1
      crops.append((x, y, int(rng.integers(1, f.w - x + 1)), int(rng.integers(1, f.h - y + 1))))
    else:
      crops.append((0, 0, f.w, f.h))
  max_dets = 12
  dets = np.concatenate([records(rng, max_dets, c[3], c[2]) for c in crops])
  dets['cls'][3] = 7                             # out of range: skipped
  dets['cx'][5] = np.nan                         # non-finite: skipped
  dets['prob'][6] = 1.5                          # kept: rectangle, no label
  counts = [max_dets, 7, max_dets, 0, -1]
  d, c = upload(dets, counts, gpu_device)
  rc = call(frames, fmt, crops if cropped else None, d.data_ptr(), c.data_ptr(), max_dets)
  assert rc == 0, _lib.load().sqdet_last_error()
  torch.cuda.synchronize(gpu_device)
  for i, f in enumerate(frames):
    recs = dets[i * max_dets:(i + 1) * max_dets]
    for p, (got, want) in enumerate(zip(f.now(), f.expected(crops[i], recs, counts[i]))):
      np.testing.assert_array_equal(got, want, err_msg='frame %d plane %d' % (i, p))


@pytest.mark.parametrize('scale', [0.5, 1.0])
def test_draw_font_scales(scale, gpu_device):
  rng = np.random.default_rng(int(scale * 8))
  f = Frame('bgr', 80, 160, rng, gpu_device, 0)
  dets = records(rng, 10, 80, 160)
  dets['prob'] = np.maximum(dets['prob'], 0.5)
  d, c = upload(dets, [10], gpu_device)
  assert call([f], 'bgr', None, d.data_ptr(), c.data_ptr(), 10, st=style(font_scale=scale)) == 0
  want = f.before[0].reshape(80, 160, 3).copy()
  for r in dets:
    x0, y0, x1, y1 = draw.box_corners(r['cx'], r['cy'], r['w'], r['h'])
    col = tuple(int(v) for v in BGR[r['cls']])
    cv2.rectangle(want, (x0, y0), (x1, y1), col, 1)
    cv2.putText(want, NAMES[r['cls']] + ': (%.2f)' % r['prob'], (x0, y1), cv2.FONT_HERSHEY_SIMPLEX,
                scale, col, 1)
  np.testing.assert_array_equal(f.now()[0].reshape(80, 160, 3), want)


def test_draw_many_frames_one_call(gpu_device):
  """More frames than one launch takes (24), on a non-default stream."""
  rng = np.random.default_rng(21)
  frames = [Frame('nv12', 10, 16, rng, gpu_device, 2) for _ in range(60)]
  dets = np.concatenate([records(rng, 3, 10, 16) for _ in frames])
  d, c = upload(dets, [3] * 60, gpu_device)
  s = torch.cuda.Stream(gpu_device)
  with torch.cuda.stream(s):
    assert call(frames, 'nv12', None, d.data_ptr(), c.data_ptr(), 3, stream=s.cuda_stream) == 0
  s.synchronize()
  for i, f in enumerate(frames):
    for got, want in zip(f.now(), f.expected((0, 0, 16, 10), dets[3 * i:3 * i + 3], 3)):
      np.testing.assert_array_equal(got, want)


def test_refusals_leave_frames_untouched(gpu_device):
  rng = np.random.default_rng(4)
  f = Frame('bgr', 20, 30, rng, gpu_device, 0)
  dets = records(rng, 4, 20, 30)
  dets['prob'] = 0.9
  d, c = upload(dets, [4], gpu_device)
  dp, cp = d.data_ptr(), c.data_ptr()
  host = np.zeros((20, 90), np.uint8)
  host_dets, host_counts = dets.copy(), np.array([4], np.int32)
  bad_calls = [
      lambda: call([f], 'bgr', [(0, 0, 31, 20)], dp, cp, 4),             # crop outside
      lambda: call([f], 'bgr', [(0, 0, 0, 5)], dp, cp, 4),               # empty crop
      lambda: call([f], 'bgr', None, dp, cp, 4, pitches=[89, 0, 0]),     # short pitch
      lambda: call([f], 'bgr', None, dp, cp, 4, pitches=[1 << 36, 0, 0]),  # past the allocation
      lambda: call([f], 'bgr', None, dp, cp, 0),                         # max_dets
      lambda: call([f], 'bgr', None, dp, cp, 4, n=0),
      lambda: call([f] * 129, 'bgr', None, dp, cp, 4),
      lambda: call([f], 'bgr', None, dp, cp, 4, st=style(classes=0)),
      lambda: call([f], 'bgr', None, dp, cp, 4, st=style(classes=65, names=NAMES * 22,
                                                             bgr=np.zeros((66, 3), np.uint8))),
      lambda: call([f], 'bgr', None, dp, cp, 4, st=style(names=('car', 'x' * 32, 'cyclist'))),
      lambda: call([f], 'bgr', None, dp, cp, 4, st=style(names=('car', 'a\tb', 'cyclist'))),
      lambda: call([f], 'bgr', None, dp, cp, 4, st=style(names=('car', None, 'cyclist'))),
      lambda: call([f], 'bgr', None, dp, cp, 4, st=style(font_scale=0.0)),
      lambda: call([f], 'bgr', None, dp, cp, 4, st=style(font_scale=float('nan'))),
      lambda: call([f], 'bgr', None, dp, cp, 4, st=style(font_scale=float('inf'))),
      lambda: call([f], 'bgr', None, host_dets.ctypes.data, cp, 4),        # host records
      lambda: call([f], 'bgr', None, dp, host_counts.ctypes.data, 4),      # host counts
  ]
  for k, bad in enumerate(bad_calls):
    assert bad() == ERR_INVALID_ARG, k
  odd = Frame('nv12', 20, 30, rng, gpu_device, 0)
  odd.h = 19                                                             # odd 4:2:0 height
  assert call([odd], 'nv12', None, dp, cp, 4) == ERR_INVALID_ARG
  lib = _lib.load()
  hp = (C.c_void_p * 3)(host.ctypes.data, None, None)                    # host memory
  assert lib.sqdet_draw_dets(1, 0, hp, None, (C.c_int32 * 1)(20), (C.c_int32 * 1)(30), None, dp,
                             cp, 4, C.byref(style()), None) == ERR_INVALID_ARG
  assert b'not inside one device allocation' in lib.sqdet_last_error()
  torch.cuda.synchronize(gpu_device)
  assert not host.any()
  for fr in (f, odd):
    for got, want in zip(fr.now(), fr.before):
      np.testing.assert_array_equal(got, want)


def full_model(batch, device, thresh):
  mc, model = demo.build_model('squeezeDet', device, 'synthetic', batch=batch)
  mc.PLOT_PROB_THRESH = thresh
  return mc, model


@pytest.mark.parametrize('fmt', ['bgr', 'nv12'])
def test_engine_tiles_match_demo_draw(fmt, gpu_device):
  """forward_device_tiles on two 1080p frames -> draw_detections_device gives the pixels of the
  demo's host draw (demo.draw_detections on the frame's BGR copy; the oracle for NV12)."""
  rng = np.random.default_rng(2)
  H, W = 1080, 1920
  grid0 = tile_grid(W, H, 1242, 375, 128)
  grid = [(f,) + t for f in range(2) for t in grid0]
  mc, model = full_model(len(grid), gpu_device, 0.0)
  shape = (H, W, 3) if fmt == 'bgr' else (3 * H // 2, W)
  host = [rng.integers(0, 256, shape, dtype=np.uint8) for _ in range(2)]
  frames = [torch.from_numpy(h).to(gpu_device) for h in host]
  model.forward_device_tiles(frames, fmt, grid, order='demo')
  dets, counts = model.tile_results(2)
  model.draw_detections_device(frames, fmt, which='tiles')
  torch.cuda.synchronize(gpu_device)
  assert counts.sum() > 0
  for i in range(2):
    boxes, probs, cls = model.records_to_lists(dets[i], int(counts[i]))
    if fmt == 'bgr':
      want, _, _, _ = demo.draw_detections(mc, host[i].copy(), boxes, probs, cls)
    else:
      want = host[i].copy()
      colours = np.array([demo_colour(n) for n in mc.CLASS_NAMES], np.uint8)
      draw.draw_yuv420(want[:H], want[H:, 0::2], want[H:, 1::2], (0, 0, W, H), dets[i],
                       int(counts[i]), list(mc.CLASS_NAMES), colours, mc.PLOT_PROB_THRESH, 0.3)
    np.testing.assert_array_equal(frames[i].cpu().numpy(), want)


def demo_colour(name):
  from squeezedet_b200.utils.viz import CLASS_COLORS
  return CLASS_COLORS.get(name, (0, 255, 0))


def test_engine_frames_rescaled_crops_match_demo_draw(gpu_device):
  """forward_device_frames_fmt(rescale=True) on 1080p crops -> draw on the same crops."""
  rng = np.random.default_rng(3)
  mc, model = full_model(3, gpu_device, 0.0)
  host = [rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8) for _ in range(3)]
  crops = [(239, 500, 1242, 375), (0, 0, 1920, 1080), (101, 33, 700, 301)]
  frames = [torch.from_numpy(h).to(gpu_device) for h in host]
  model.forward_device_frames_fmt(frames, 'bgr', crops=crops, rescale=True)
  res = model.results_device()
  torch.cuda.synchronize(gpu_device)
  n, md = 3, res['max_dets']
  dets = np.empty((mc.BATCH_SIZE, md), _lib.DET_DTYPE)
  counts = np.empty((mc.BATCH_SIZE,), np.int32)
  _lib.check(_lib.load().sqdet_memcpy_d2h(dets.ctypes.data, res['dets'], dets.nbytes, None))
  _lib.check(_lib.load().sqdet_memcpy_d2h(counts.ctypes.data, res['counts'], counts.nbytes, None))
  model.draw_detections_device(frames, 'bgr', which='frames', crops=crops)
  torch.cuda.synchronize(gpu_device)
  assert counts[:n].sum() > 0
  for i, (x, y, w, h) in enumerate(crops):
    want = host[i].copy()
    demo.draw_detections(mc, want[y:y + h, x:x + w], *model.records_to_lists(dets[i], int(counts[i])))
    np.testing.assert_array_equal(frames[i].cpu().numpy(), want)


def test_demo_video_tiles_files_unchanged(gpu_device, tmp_path, monkeypatch):
  """`demo.py --mode video --tiles` draws on the device frame; each file it writes is byte for byte
  the one of drawing the same records on the host frame with demo.draw_detections."""
  import os
  video = str(tmp_path / 'in.avi')
  w, h = 1280, 720
  writer = cv2.VideoWriter(video, cv2.VideoWriter_fourcc(*'MJPG'), 10, (w, h))
  rng = np.random.default_rng(19)
  for _ in range(3):
    writer.write(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
  writer.release()
  wants = []
  build = demo.build_model

  def build_model(*args, **kwargs):
    mc, model = build(*args, **kwargs)
    draw_device = model.draw_detections_device

    def draw_and_record(frames, fmt, **kw):
      dets, counts = model.tile_results(1)
      im, _, _, _ = demo.draw_detections(mc, frames[0].cpu().numpy(),
                                         *model.records_to_lists(dets[0], int(counts[0])))
      wants.append(im)
      return draw_device(frames, fmt, **kw)

    model.draw_detections_device = draw_and_record
    return mc, model

  monkeypatch.setattr(demo, 'build_model', build_model)
  out = tmp_path / 'out'
  demo.main(['--mode', 'video', '--tiles', '--checkpoint', 'synthetic', '--input_path', video,
             '--out_dir', str(out), '--gpu', str(gpu_device)])
  assert len(wants) == 3
  for k, im in enumerate(wants, 1):
    want = str(tmp_path / ('want%d.jpg' % k))
    cv2.imwrite(want, im)
    with open(want, 'rb') as a, open(os.path.join(out, str(k).zfill(6) + '.jpg'), 'rb') as b:
      assert a.read() == b.read(), k


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_draw_runs_on_the_frames_device(gpu_device):
  """Frames and records on cuda:1 draw while cuda:0 is current."""
  rng = np.random.default_rng(31)
  f = Frame('bgr', 30, 40, rng, 1, 0)
  dets = records(rng, 4, 30, 40)
  d, c = upload(dets, [4], 1)
  torch.cuda.set_device(0)
  assert call([f], 'bgr', None, d.data_ptr(), c.data_ptr(), 4) == 0, _lib.load().sqdet_last_error()
  torch.cuda.synchronize(1)
  np.testing.assert_array_equal(f.now()[0], f.expected((0, 0, 40, 30), dets, 4)[0])
