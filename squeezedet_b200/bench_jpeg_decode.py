#!/usr/bin/env python
"""What feeding JPEG files to the engine costs, two ways.

  python -m squeezedet_b200.bench_jpeg_decode --rounds 5 --steps 10 --warmup 3

A SqueezeDet engine at 1242x375 (b = --frames) runs forward_device_frames on --frames JPEG files
per step, quality 95, of smooth synthetic pictures (bilinear upsampled noise plus grain, as
bench_jpeg makes them, seeded on the host).  Three workloads: 1242x375 files, 1920x1080 files and
4000x3000 files, the size of a 12 MP camera's.
Each step starts from the files' bytes on the host and ends one of two ways:
  (a) a thread pool of cv2.imdecode (one file per task, os.cpu_count() threads), the BGR frames
      uploaded, then forward_device_frames;
  (b) decode_jpeg_device on the engine's stream, then forward_device_frames.
The step ends at a device synchronisation; the forms alternate within each round.  Every step's
records of (b) are checked bitwise against (a)'s.

The decode kernels alone are timed in a separate pass under torch.profiler: the device durations of
the decode_jpeg_device calls' kernels, copies and memsets, summed, per frame.

--progressive writes the files with IMWRITE_JPEG_PROGRESSIVE and decodes them with
decode_jpeg_device(progressive=True); the kernel pass then also reports each kernel's share: the
first scans, the DC refinements and the AC refinements separately.

--reduce s (2, 4 or 8) decodes at 1/s of the size: (a) with cv2.imdecode(f,
IMREAD_REDUCED_COLOR_s), (b) with decode_jpeg_device(reduce=s); the forward resizes the smaller
frames.  Each row reports the device bytes of a call: its frames and its decode scratch.

--layout cmyk or rgb writes the same pictures as Pillow's CMYK files (Adobe-inverted, 4:4:4, four
components) or its RGB-coded files (keep_rgb: Adobe transform 0, 4:4:4), quality 95, and decodes
them with decode_jpeg_device(any_layout=True); (a) is cv2.imdecode of the same files.

Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .bench_device_frames import make_model
from .bench_device_u8 import gpu_info

FORMS = ('a_cv2_imdecode_pool', 'b_decode_jpeg_device')
QUALITY = 95
KERNELS = ('destuff_count_kernel', 'scan_chunks_kernel', 'destuff_compact_kernel',
           'intervals_kernel', 'sync_tiles_kernel', 'sync_chain_kernel', 'scan_counts_kernel',
           'decode_write_kernel', 'idct_kernel', 'color_kernel')
PROG_KERNELS = ('prog_seq_kernel', 'prog_dc_refine_kernel', 'idct_kernel', 'color_kernel')


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--frames', type=int, default=8)
  ap.add_argument('--gpu', type=int, default=0)
  ap.add_argument('--progressive', action='store_true')
  ap.add_argument('--reduce', type=int, choices=(1, 2, 4, 8), default=1)
  ap.add_argument('--layout', choices=('cmyk', 'rgb'), default=None)
  return ap.parse_args(argv)


def picture(h, w, rng):
  """A smooth uint8 [h, w, 3] picture: bilinear upsampled noise plus grain."""
  import cv2
  low = rng.uniform(0, 255, (max(h // 24, 2), max(w // 24, 2), 3)).astype(np.float32)
  up = cv2.resize(low, (w, h), interpolation=cv2.INTER_LINEAR)
  return np.clip(up + rng.normal(0, 4, (h, w, 3)), 0, 255).astype(np.uint8)


def encode(img, args):
  """A quality-95 JPEG of BGR img: cv2's (4:2:0), or with --layout Pillow's CMYK or RGB-coded one."""
  import cv2
  if args.layout is None:
    params = [cv2.IMWRITE_JPEG_QUALITY, QUALITY] + ([cv2.IMWRITE_JPEG_PROGRESSIVE, 1] if args.progressive else [])
    return cv2.imencode('.jpg', img, params)[1].tobytes()
  import io
  from PIL import Image
  rgb = np.ascontiguousarray(img[..., ::-1])
  if args.layout == 'cmyk':
    im = Image.fromarray(np.concatenate([255 - rgb, np.zeros(rgb.shape[:2] + (1,), np.uint8)], axis=2), 'CMYK')
    kw = {}
  else:
    im, kw = Image.fromarray(rgb, 'RGB'), {'keep_rgb': True}
  buf = io.BytesIO()
  im.save(buf, 'JPEG', quality=QUALITY, progressive=args.progressive, **kw)
  return buf.getvalue()


def measure_workload(args, name, model, files, torch):
  import ctypes as C
  import cv2
  from . import _lib
  from .jpeg import decode_jpeg_device, jpeg_info
  dev = torch.device('cuda', args.gpu)
  flag = {1: cv2.IMREAD_COLOR, 2: cv2.IMREAD_REDUCED_COLOR_2, 4: cv2.IMREAD_REDUCED_COLOR_4,
          8: cv2.IMREAD_REDUCED_COLOR_8}[args.reduce]
  lib = model._lib
  stream = torch.cuda.ExternalStream(lib.sqdet_engine_stream(model._engine), device=dev)
  pool = ThreadPoolExecutor(os.cpu_count() or 1)

  def records():
    res = model.results_device()
    out = np.empty((len(files), res['max_dets']), _lib.DET_DTYPE)
    _lib.check(lib.sqdet_memcpy_d2h(out.ctypes.data, res['dets'], out.nbytes, None))
    return out

  def form_a():
    imgs = list(pool.map(lambda f: cv2.imdecode(np.frombuffer(f, np.uint8), flag), files))
    with torch.cuda.stream(stream):
      frames = [torch.from_numpy(im).to(dev, non_blocking=False) for im in imgs]
    model.forward_device_frames(frames, stream=stream.cuda_stream)
    stream.synchronize()

  def form_b():
    frames, status = decode_jpeg_device(files, dev, stream=stream, progressive=args.progressive,
                                        reduce=args.reduce, any_layout=args.layout is not None)
    model.forward_device_frames(frames, stream=stream.cuda_stream)
    stream.synchronize()
    return status

  form_a()
  want = records()
  st = form_b()
  assert st.cpu().tolist() == [0] * len(files)
  assert records().tobytes() == want.tobytes(), '%s: the records differ' % name
  forms = {FORMS[0]: form_a, FORMS[1]: form_b}
  for form in FORMS:
    for _ in range(args.warmup):
      forms[form]()
  step = {form: [] for form in FORMS}
  for r in range(args.rounds):
    for form in (FORMS if r % 2 == 0 else FORMS[::-1]):
      for _ in range(args.steps):
        t0 = time.perf_counter()
        forms[form]()
        step[form].append(time.perf_counter() - t0)
      assert records().tobytes() == want.tobytes(), '%s: the records of %s differ' % (name, form)
  pool.shutdown()

  from torch.autograd import DeviceType
  from torch.profiler import ProfilerActivity, profile
  calls = 20
  keep = []
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(calls):
      keep.append(decode_jpeg_device(files, dev, stream=stream, progressive=args.progressive,
                                     reduce=args.reduce, any_layout=args.layout is not None))
    stream.synchronize()
  names = (PROG_KERNELS if args.progressive else KERNELS) + (('color_any_kernel',) if args.layout else ())
  evs = [ev for ev in prof.events() if ev.device_type == DeviceType.CUDA and
         any(k in ev.name for k in names + ('emset', 'emcpy', 'Memcpy', 'Memset'))]
  kern = [ev for ev in evs if any(k in ev.name for k in names)]
  assert len(kern) >= calls * (3 if args.progressive else len(KERNELS)) * 9 // 10, \
      'found %d decode launches' % len(kern)
  us = sum(ev.time_range.elapsed_us() for ev in evs) / calls
  us_k = sum(ev.time_range.elapsed_us() for ev in kern) / calls
  n = len(files)
  row = {'workload': name, 'frames': n, 'file_bytes_mean': float(np.mean([len(f) for f in files]))}
  for form in FORMS:
    row[form] = {'ms_per_frame_step_median': 1e3 * float(np.median(step[form])) / n,
                 'ms_per_frame_step_min': 1e3 * min(step[form]) / n}
  row['decode_device'] = {'us_per_frame_kernels': us_k / n, 'us_per_frame_with_copy_and_memsets': us / n,
                          'calls_timed': calls}
  infos = [jpeg_info(f, args.progressive, args.reduce, args.layout is not None) for f in files]
  bufs = [C.create_string_buffer(f, len(f)) for f in files]
  options = _lib.JpegDecodeOptions(int(args.progressive), args.reduce, int(args.layout is not None))
  scratch = lib.sqdet_jpeg_decode_scratch_bytes_options(
      n, (C.c_void_p * n)(*[C.addressof(b) for b in bufs]), (C.c_int64 * n)(*map(len, files)), C.byref(options))
  row['device_bytes_per_call'] = {'frames': sum(3 * i['height'] * i['width'] for i in infos),
                                  'decode_scratch': int(scratch),
                                  'frame_hw': [infos[0]['height'], infos[0]['width']]}
  if args.progressive:
    # a call's first prog_seq_kernel decodes the first scans, its later ones the AC refinements
    share = {}
    prev = None
    for ev in sorted(kern, key=lambda e: e.time_range.start):
      k = next(k for k in names if k in ev.name)
      if k == 'prog_seq_kernel':
        k = 'ac_refine' if prev in ('prog_seq_kernel', 'prog_dc_refine_kernel', 'ac_refine') else 'first_scans'
      share[k] = share.get(k, 0.0) + ev.time_range.elapsed_us() / calls / n
      prev = k if k != 'first_scans' else 'prog_seq_kernel'
    row['decode_device']['us_per_frame_by_kernel'] = share
  return row


def measure(args):
  import torch
  from . import _lib
  import cv2
  if _lib.device_count() < 1:
    raise SystemExit('bench_jpeg_decode: no CUDA device visible; the engine has no CPU fallback')
  rng = np.random.default_rng(7)
  model = make_model(1242, 375, args.frames, args.gpu)
  rows = []
  for name, (h, w) in (('kitti_1242x375', (375, 1242)), ('1080p', (1080, 1920)),
                       ('camera_4000x3000', (3000, 4000))):
    files = [encode(picture(h, w, rng), args) for _ in range(args.frames)]
    rows.append(measure_workload(args, name, model, files, torch))
  kind = ('progressive ' if args.progressive else '') + \
      {None: '', 'cmyk': "Pillow's CMYK ", 'rgb': "Pillow's RGB-coded "}[args.layout]
  scale = ' at 1/%d (IMREAD_REDUCED_COLOR_%d)' % (args.reduce, args.reduce) if args.reduce > 1 else ''
  return {'workload': 'squeezeDet 1242x375 forward_device_frames on %sJPEG files (quality 95, %s, '
                      'smooth synthetic pictures) decoded%s by a cv2.imdecode thread pool and '
                      'uploaded, or by decode_jpeg_device' % (kind, '4:4:4' if args.layout else '4:2:0', scale),
          'reduce': args.reduce, 'layout': args.layout or 'ycc',
          'gpu': gpu_info(args.gpu), 'cpu_threads': os.cpu_count(),
          'timer': 'host clock per step from the files on the host to a device synchronisation '
                   'after the forward; decode kernels: torch.profiler device durations, summed, per frame',
          'rounds': args.rounds, 'steps': args.steps, 'forms': list(FORMS), 'rows': rows}


def main(argv=None):
  print(json.dumps(measure(parse_args(argv))))


if __name__ == '__main__':
  main()
