#!/usr/bin/env python
"""SqueezeDet demo — drop-in for reference ``src/demo.py`` (image mode and video mode), same
flags: --mode --checkpoint --input_path --out_dir --demo_net --gpu.

    python -m squeezedet_b200.demo --input_path './data/*.png' \\
        --checkpoint ./data/model_checkpoints/squeezeDet/model.ckpt-87000

`--checkpoint` takes the reference's own Saver path (TensorFlow V2 `.index/.data` bundle or V1
table, read without TensorFlow: utils/tf_checkpoint.py), an .npz keyed by the reference's
variable names, or the word `synthetic` for seeded random weights (plumbing run, SURVEY
config 1).  Per image: cv2.imread -> float32 -> cv2.resize to
(mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT) -> minus mc.BGR_MEANS (reference demo.py:187-190) -> ONE GPU
pass doing detect + filter_prediction (demo.py:193-199) -> keep prob > PLOT_PROB_THRESH -> draw ->
imwrite out_<name>.

`--mode video --tiles` looks at whole frames instead of the reference's fixed crop: each frame is
uploaded once and covered by overlapping network-sized tiles at native scale
(utils.util.tile_grid, 128 px overlap), whose detections are merged per frame on the GPU
(ModelSkeleton.forward_device_tiles) and drawn on the full frame in device memory
(ModelSkeleton.draw_detections_device, bitwise draw_detections), then encoded to JPEG on the device
(jpeg.encode_jpeg_device, byte for byte cv2.imwrite's file): only the file's bytes come back.
`--host_encode` copies the drawn frame back and writes it with cv2.imwrite instead.
"""
from __future__ import annotations

import argparse
import glob
import os
import time

import numpy as np


def parse_flags(argv=None):
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument('--mode', default='image', help="'image' or 'video'.")
  ap.add_argument('--checkpoint', default='./data/model_checkpoints/squeezeDet/model.ckpt-87000',
                  help='Path to the model parameter file: TF checkpoint, .npz, or "synthetic".')
  ap.add_argument('--input_path', default='./data/sample.png',
                  help='Input image or video to be detected. Can process glob input such as '
                       './data/00000*.png.')
  ap.add_argument('--out_dir', default='./data/out/', help='Directory to dump output image or video.')
  ap.add_argument('--demo_net', default='squeezeDet', help='Neural net architecture.')
  ap.add_argument('--gpu', default='0', help='gpu id.')
  ap.add_argument('--tiles', action='store_true',
                  help='Video mode: detect over whole frames as overlapping tiles, merged per '
                       'frame on the GPU, instead of the reference crop.')
  ap.add_argument('--host_encode', action='store_true',
                  help='With --tiles: copy each drawn frame back and cv2.imwrite it instead of '
                       'encoding it on the GPU (the same bytes).')
  return ap.parse_args(argv)


def build_model(demo_net, gpu, checkpoint, batch=1):
  from . import config as cfg
  from .nets import SqueezeDet, SqueezeDetPlus
  from .utils import checkpoint as ckpt, synth
  assert demo_net in ('squeezeDet', 'squeezeDet+'), \
      'Selected nueral net architecture not supported: {}'.format(demo_net)
  mc = cfg.kitti_squeezeDet_config() if demo_net == 'squeezeDet' else cfg.kitti_squeezeDetPlus_config()
  mc.BATCH_SIZE = batch
  mc.LOAD_PRETRAINED_MODEL = False          # parameters come from the checkpoint only
  model = (SqueezeDet if demo_net == 'squeezeDet' else SqueezeDetPlus)(mc, int(gpu))
  if checkpoint == 'synthetic':
    model.load_weights(synth.synthetic_weights(synth.model_param_specs(model), seed=0))
  else:
    model.load_weights(ckpt.load_weights_file(checkpoint, names=model.param_names()))
  return mc, model


def preprocess(im_bgr_u8, mc):
  """demo.py:187-190: float32 -> resize -> minus BGR means (float64 subtraction, fp32 feed)."""
  import cv2
  im = im_bgr_u8.astype(np.float32, copy=False)
  im = cv2.resize(im, (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT))
  return im, (im - mc.BGR_MEANS).astype(np.float32)


def draw_detections(mc, im, final_boxes, final_probs, final_class):
  """Draws the detections above mc.PLOT_PROB_THRESH on `im`; returns them."""
  from .utils.viz import CLASS_COLORS, draw_box
  keep = [i for i in range(len(final_probs)) if final_probs[i] > mc.PLOT_PROB_THRESH]
  final_boxes = [final_boxes[i] for i in keep]
  final_probs = [final_probs[i] for i in keep]
  final_class = [final_class[i] for i in keep]
  draw_box(im, final_boxes,
           [mc.CLASS_NAMES[idx] + ': (%.2f)' % prob for idx, prob in zip(final_class, final_probs)],
           cdict=CLASS_COLORS)
  return im, final_boxes, final_probs, final_class


def detect_and_draw(model, mc, im, frame_u8):
  """`frame_u8`: the uint8 BGR frame as read; resize + mean subtraction (demo.py:187-190) run on
  the GPU in front of the forward (sqdet_submit_frames, order = resize then subtract)."""
  dets, counts = model.detect_frames([frame_u8], order='demo', rescale=False)
  return draw_detections(mc, im, *model.records_to_lists(dets[0], int(counts[0])))


def image_demo(flags):
  """Detect image(s)."""
  import cv2
  mc, model = build_model(flags.demo_net, flags.gpu, flags.checkpoint)
  os.makedirs(flags.out_dir, exist_ok=True)
  results = []
  for f in sorted(glob.iglob(flags.input_path)):
    frame = cv2.imread(f)
    im = cv2.resize(frame.astype(np.float32, copy=False), (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT))
    im, boxes, probs, classes = detect_and_draw(model, mc, im, frame)   # `im`: drawing canvas
    out_file_name = os.path.join(flags.out_dir, 'out_' + os.path.split(f)[1])
    cv2.imwrite(out_file_name, im)
    print('Image detection output saved to {}'.format(out_file_name))
    results.append((f, boxes, probs, classes))
  return results


def video_demo(flags):
  """Detect videos (reference demo.py:44-158: same per-frame crop and per-stage wall clock)."""
  if flags.tiles:
    return video_demo_tiles(flags)
  import cv2
  mc, model = build_model(flags.demo_net, flags.gpu, flags.checkpoint)
  cap = cv2.VideoCapture(flags.input_path)
  os.makedirs(flags.out_dir, exist_ok=True)
  count = 0
  while cap.isOpened():
    t_start = time.time()
    count += 1
    ret, frame = cap.read()
    if not ret:
      break
    frame = frame[500:-205, 239:-439, :]           # the reference's hard-coded crop (demo.py:91)
    frame = np.ascontiguousarray(frame)
    im = cv2.resize(frame.astype(np.float32, copy=False), (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT))
    t_reshape = time.time()
    im, boxes, probs, classes = detect_and_draw(model, mc, im, frame)
    t_detect = time.time()
    cv2.imwrite(os.path.join(flags.out_dir, str(count).zfill(6) + '.jpg'), im)
    t_draw = time.time()
    print('Total time: {:.4f}, detail: reshape {:.4f} detect+filter {:.4f} draw {:.4f}'.format(
        t_draw - t_start, t_reshape - t_start, t_detect - t_reshape, t_draw - t_detect))
  cap.release()


def video_demo_tiles(flags):
  """Detect videos over whole frames: the frame goes to the GPU once and runs as a tile_grid of
  network-sized tiles, merged per frame (forward_device_tiles); boxes are drawn on the full
  frame on the device (draw_detections_device) and encoded there (encode_jpeg_device), so only
  the JPEG's bytes come back; with --host_encode the frame comes back for cv2.imwrite."""
  import cv2
  import torch
  from . import config as cfg
  from .jpeg import encode_jpeg_device, jpeg_bytes
  from .utils.util import tile_grid
  cap = cv2.VideoCapture(flags.input_path)
  w, h = int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
  net_mc = cfg.kitti_squeezeDet_config()
  grid = [(0,) + tile for tile in tile_grid(w, h, net_mc.IMAGE_WIDTH, net_mc.IMAGE_HEIGHT, 128)]
  mc, model = build_model(flags.demo_net, flags.gpu, flags.checkpoint, batch=len(grid))
  os.makedirs(flags.out_dir, exist_ok=True)
  dev = 'cuda:%d' % int(flags.gpu)
  count = 0
  while cap.isOpened():
    t_start = time.time()
    count += 1
    ret, frame = cap.read()
    if not ret:
      break
    frame_dev = torch.from_numpy(frame).to(dev)
    t_upload = time.time()
    model.forward_device_tiles([frame_dev], 'bgr', grid, order='demo')
    torch.cuda.synchronize(dev)                    # the forward and merge are asynchronous
    t_detect = time.time()
    # boxes and labels drawn on the device frame, bitwise draw_detections on its host copy
    model.draw_detections_device([frame_dev], 'bgr', which='tiles')
    out_file = os.path.join(flags.out_dir, str(count).zfill(6) + '.jpg')
    if flags.host_encode:
      cv2.imwrite(out_file, frame_dev.cpu().numpy())
    else:                                          # cv2.imwrite's bytes, encoded on the device
      (data,) = jpeg_bytes(*encode_jpeg_device([frame_dev], 'bgr'))
      with open(out_file, 'wb') as f:
        f.write(data)
    t_draw = time.time()
    print('Total time: {:.4f}, detail: upload {:.4f} detect+merge {:.4f} draw {:.4f}'.format(
        t_draw - t_start, t_upload - t_start, t_detect - t_upload, t_draw - t_detect))
  cap.release()


def main(argv=None):
  flags = parse_flags(argv)
  if flags.mode == 'image':
    image_demo(flags)
  else:
    video_demo(flags)


if __name__ == '__main__':
  main()
