#!/usr/bin/env python
"""What writing annotated 1080p frames as PNG files costs, two ways.

  python -m squeezedet_b200.bench_png --rounds 5 --steps 10 --warmup 3

A SqueezeDet engine at 1242x375 runs `frames` 1080p frames (smooth synthetic pictures made on the
device from a seed: upsampled noise plus a little grain) as a utils.util.tile_grid of 8 tiles each,
and draw_detections_device draws the merged records on them, as bench_draw and bench_jpeg do.
Two frame formats: packed BGR and NV12.  Each step then ends one of two ways:
  (a) every frame copied to the host, cv2.cvtColor'd to BGR (NV12), and cv2.imencode('.png');
  (b) encode_png_device on the same stream, then png_bytes copies back only each file's bytes
      (a PNG of these pictures is several MB, so the copy is a real part of the cost).
The forms alternate within each round.  A step's time is split at a device synchronisation after
the draw: `ending` is the encode and copy alone, `step` the whole step (a fresh copy of the frames,
forward, draw, ending).  Every step's files of (b) are checked bitwise against (a)'s.  The
measurement is bench_jpeg's, with the PNG encoder.

The encode kernels alone are timed in a separate pass under torch.profiler: the device durations of
the encode_png_device calls' kernels and memsets, summed, per frame, also per kernel.

Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.
"""
from __future__ import annotations

import argparse
import json

from .bench_jpeg import Encoder, measure

KERNELS = ('filter_kernel', 'mark_kernel', 'seg_scan_kernel', 'count_kernel', 'emit_kernel',
           'tree_kernel', 'frame_kernel', 'pack_kernel', 'idat_kernel')


def parse_args(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--frames', type=int, default=2)
  ap.add_argument('--gpu', type=int, default=0)
  return ap.parse_args(argv)


def png_encoder():
  from .png import encode_png_device, png_bytes
  # two scans and a memset per 16 frames
  return Encoder('png', '.png', [],
                 lambda frames, fmt, stream: encode_png_device(frames, fmt, stream=stream),
                 png_bytes, KERNELS, len(KERNELS) + 2, 'PNG files (cv2 defaults)', {},
                 by_kernel=True)


def main(argv=None):
  print(json.dumps(measure(parse_args(argv), png_encoder())))


if __name__ == '__main__':
  main()
