#!/usr/bin/env python
"""Evaluation loop — drop-in for the detection part of reference ``src/eval.py``
(`eval_once`, lines 48-134), same flags: --dataset --data_path --image_set --eval_dir
--checkpoint_path --run_once --net --gpu, plus --batch_size.

Per image, in the reference's order (eval.py:69-92): the uint8 frame goes to the GPU, where it
is converted to float32, has the BGR means subtracted and is resized (src/dataset/imdb.py:85-97);
forward; ALL det boxes are rescaled to the original image (eval.py:83-84) and only then
filtered (filter_prediction + NMS on original-image coordinates, eval.py:86-87) - one
`sqdet_submit_frames_n(..., order=eval, rescale=1)` call per group of --batch_size images
(default 1, the reference's image-by-image loop, eval.py:150); the last group is short and runs
on the same engine.  Two groups are in flight on the GPU while a thread pool decodes the next one
with cv2.imread.  Corner format + score go into all_boxes[cls][image].  Then the KITTI detection
files are written
(src/dataset/kitti.py:100-127), and the records, uploaded once as one [N, max_dets] array, are
scored on the GPU (squeezedet_b200.kitti, byte for byte the files of the KITTI devkit's
`evaluate_object`, which src/dataset/kitti.py:129-136 runs) into stats_*.txt next to `data/`,
whose APs are parsed as the reference parses them (kitti.py:138-159).  Then, as eval.py:128-130
does, the detections are analyzed on the GPU from the same records (kitti.analyze_device, line
for line the reference's analyze_detections, kitti.py:182-296): the "Detection Analysis" block
is printed and detection_files_0/error_analysis/det_error_file.txt written.  Where the reference
divides by zero there (no counted detection or no object), the share prints as nan.  The
TensorBoard summaries, the images visualize_detections draws for them (imdb.py:254-305) and the
checkpoint-polling loop (eval.py:171-239) are not rebuilt.
"""
from __future__ import annotations

import argparse
import collections
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .utils.util import Timer, bbox_transform
from .utils.viz import parse_kitti_ap_files, write_kitti_detections


def parse_flags(argv=None):
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument('--dataset', default='KITTI', help='Currently support KITTI dataset.')
  ap.add_argument('--data_path', default='', help='Root directory of data')
  ap.add_argument('--image_set', default='test', help='train, trainval, val, or test')
  ap.add_argument('--eval_dir', default='/tmp/bichen/logs/squeezeDet/eval')
  ap.add_argument('--checkpoint_path', default='/tmp/bichen/logs/squeezeDet/train',
                  help='TF checkpoint path, .npz keyed by reference variable names, or "synthetic".')
  ap.add_argument('--run_once', action='store_true', default=True)
  ap.add_argument('--net', default='squeezeDet', help='Neural net architecture.')
  ap.add_argument('--gpu', default='0', help='gpu id.')
  ap.add_argument('--batch_size', type=int, default=1,
                  help='Images per forward; the last group of the image set may be shorter.')
  return ap.parse_args(argv)


NETS = {'vgg16': ('VGG16ConvDet', 'kitti_vgg16_config'),
        'resnet50': ('ResNet50ConvDet', 'kitti_res50_config'),
        'squeezeDet': ('SqueezeDet', 'kitti_squeezeDet_config'),
        'squeezeDet+': ('SqueezeDetPlus', 'kitti_squeezeDetPlus_config')}


def read_image(path, mc):
  """imdb.read_image_batch for one image (src/dataset/imdb.py:85-97): float32, subtract the
  BGR means in place, THEN resize; returns the image and (x_scale, y_scale)."""
  import cv2
  im = cv2.imread(path).astype(np.float32, copy=False)
  im -= mc.BGR_MEANS
  orig_h, orig_w = float(im.shape[0]), float(im.shape[1])
  im = cv2.resize(im, (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT))
  return im, (mc.IMAGE_WIDTH / orig_w, mc.IMAGE_HEIGHT / orig_h)


def detections_to_all_boxes(records, count, scale, num_classes):
  """One image's filtered records -> per-class lists of [xmin, ymin, xmax, ymax, score]
  (eval.py:89-91).  `scale` = (x_scale, y_scale) still to be divided out, or None when the
  engine already rescaled the boxes before the filter (the reference order, eval.py:83-87).
  count < 0 is the filter's overflow marker (PROB_THRESH branch above the record capacity)."""
  from ._lib import SqdetError
  if count < 0:
    raise SqdetError(-6, 'more boxes above PROB_THRESH than the record capacity')
  out = [[] for _ in range(num_classes)]
  x_scale, y_scale = scale if scale is not None else (1.0, 1.0)
  for r in records[:count]:
    if scale is None:
      box = np.array([r['cx'], r['cy'], r['w'], r['h']], dtype=np.float32)
    else:
      box = np.array([r['cx'] / x_scale, r['cy'] / y_scale, r['w'] / x_scale, r['h'] / y_scale],
                     dtype=np.float32)
    out[int(r['cls'])].append(bbox_transform(box) + [r['prob']])
  return out


def _read_frame(path):
  """cv2.imread of one frame (uint8 BGR, original size) and the seconds it took."""
  import cv2
  t0 = time.time()
  frame = cv2.imread(path)
  return frame, time.time() - t0


def _charge(timer, seconds, images):
  """Adds `seconds` spent on `images` images to `timer`, keeping its average per image."""
  timer.total_time += seconds
  timer.calls += images
  timer.average_time = timer.total_time / timer.calls


# where oracle/build_kitti_eval.sh puts the devkit's own scorer, against which the tests check
# the GPU scorer's files; eval_once does not run it
EVAL_TOOL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle',
                         '_ref', 'evaluate_object')


def eval_once(flags):
  from . import config as cfg
  from . import nets
  from .utils import checkpoint as ckpt, synth
  assert flags.dataset == 'KITTI', 'Currently only supports KITTI dataset'
  assert flags.net in NETS, 'Selected neural net architecture not supported: {}'.format(flags.net)
  cls_name, cfg_name = NETS[flags.net]
  mc = getattr(cfg, cfg_name)()
  k = int(flags.batch_size)
  assert k >= 1, '--batch_size must be at least 1'
  mc.BATCH_SIZE = k                     # 1: the reference evaluates image by image (eval.py:150)
  mc.LOAD_PRETRAINED_MODEL = False
  model = getattr(nets, cls_name)(mc, int(flags.gpu))
  if flags.checkpoint_path == 'synthetic':
    model.load_weights(synth.synthetic_weights(synth.model_param_specs(model), seed=0))
  else:
    model.load_weights(ckpt.load_weights_file(flags.checkpoint_path, names=model.param_names()))

  with open(os.path.join(flags.data_path, 'ImageSets', flags.image_set + '.txt')) as f:
    image_ids = [x.strip() for x in f.readlines()]
  image_dir = os.path.join(flags.data_path, 'training', 'image_2')
  num_images = len(image_ids)
  all_boxes = [[[] for _ in range(num_images)] for _ in range(mc.CLASSES)]
  # every timer is an average per image: im_read = cv2.imread time, im_detect = host time spent
  # in the submit and wait calls, misc = records -> all_boxes
  _t = {'im_detect': Timer(), 'im_read': Timer(), 'misc': Timer()}
  from ._lib import DET_DTYPE, PinnedArray
  groups = [list(range(s, min(s + k, num_images))) for s in range(0, num_images, k)]
  # one pinned result slot per group in flight (pinned, so the copies back stay asynchronous)
  dets_buf = [PinnedArray((k, model.max_dets), DET_DTYPE) for _ in range(2)]
  counts_buf = [PinnedArray((k,), np.int32) for _ in range(2)]
  # every image's records, for the scorer
  all_dets = np.zeros((num_images, model.max_dets), DET_DTYPE)
  all_counts = np.zeros((num_images,), np.int32)

  def collect(gi):
    """The results of group gi, after its wait()."""
    dets, counts = dets_buf[gi & 1].array, counts_buf[gi & 1].array
    for j, i in enumerate(groups[gi]):
      _t['misc'].tic()
      all_dets[i], all_counts[i] = dets[j], counts[j]
      per_class = detections_to_all_boxes(dets[j], int(counts[j]), None, mc.CLASSES)
      for c in range(mc.CLASSES):
        all_boxes[c][i] = per_class[c]
      _t['misc'].toc()
      print('im_detect: {:d}/{:d} im_read: {:.3f}s detect: {:.3f}s misc: {:.3f}s'.format(
          i + 1, num_images, _t['im_read'].average_time, _t['im_detect'].average_time,
          _t['misc'].average_time))

  with ThreadPoolExecutor(max_workers=max(1, min(k, os.cpu_count() or 1, 8))) as pool:
    def start_read(gi):
      return [pool.submit(_read_frame, os.path.join(image_dir, image_ids[i] + '.png'))
              for i in groups[gi]]

    in_flight = collections.deque()        # (group, its frames), oldest first
    reading = start_read(0) if groups else []
    for gi in range(len(groups)):
      read = [f.result() for f in reading]
      _charge(_t['im_read'], sum(s for _, s in read), len(read))
      frames = [f for f, _ in read]
      if gi + 1 < len(groups):
        reading = start_read(gi + 1)       # decodes while this group runs on the GPU
      t0 = time.time()
      # imdb.py:85-97 pre-processing, forward, eval.py:83-84 rescale, filter: one GPU pass
      model.submit_frames(frames, dets_buf[gi & 1].ptr, counts_buf[gi & 1].ptr, order='eval',
                          rescale=True)
      in_flight.append((gi, frames))
      done = None
      if len(in_flight) == 2:
        model.wait()
        done = in_flight.popleft()[0]
      _charge(_t['im_detect'], time.time() - t0, len(frames))
      if done is not None:
        collect(done)
    while in_flight:
      t0 = time.time()
      model.wait()
      done = in_flight.popleft()[0]
      _charge(_t['im_detect'], time.time() - t0, len(groups[done]))
      collect(done)
  for buf in dets_buf + counts_buf:
    buf.free()

  det_dir = os.path.join(flags.eval_dir, 'detection_files_{:s}'.format('0'), 'data')
  result_dir = write_kitti_detections(det_dir, image_ids, mc.CLASS_NAMES, all_boxes)
  from . import kitti
  labels = None
  try:
    labels = kitti.read_labels(os.path.join(flags.data_path, 'training', 'label_2'), image_ids)
  except (OSError, ValueError) as e:
    # as evaluate_object did: an error naming the file, no stats files, APs of 0
    print('ERROR: Couldn\'t read the ground truth: {}'.format(e))
  else:
    scores = kitti.evaluate_device(all_dets, all_counts, mc.CLASS_NAMES, labels,
                                   device='cuda:{:d}'.format(int(flags.gpu)))
    kitti.write_stats(result_dir, scores)
  aps, names = parse_kitti_ap_files(result_dir, mc.CLASS_NAMES)
  for ap, name in zip(aps, names):
    print('    {}: {:.3f}'.format(name, ap))
  print('    Mean average precision: {:.3f}'.format(float(np.mean(aps))))
  if labels is not None:
    analyze(flags, image_ids, mc.CLASS_NAMES, all_dets, all_counts, labels, result_dir)
  return all_boxes, aps, names


def analyze(flags, image_ids, class_names, all_dets, all_counts, labels, result_dir):
  """eval.py:128-130: the detection analysis of every image's records, printed, and
  <result_dir>/error_analysis/det_error_file.txt.  A label box the reference asserts against
  prints an error naming the image, and no error file is written."""
  from . import kitti
  print('Analyzing detections...')
  try:
    stats, lines = kitti.analyze_device(all_dets, all_counts, class_names, labels,
                                        device='cuda:{:d}'.format(int(flags.gpu)))
  except ValueError as e:
    msg = str(e)
    if msg.startswith('image '):
      k = int(msg.split(':')[0].split()[1])
      msg = '{} ({}.txt){}'.format(msg.split(':')[0], image_ids[k], msg[msg.index(':'):])
    print('ERROR: Couldn\'t analyze the detections: {}'.format(msg))
    return None
  print(kitti.analysis_text(stats), end='')
  kitti.write_error_file(os.path.join(result_dir, 'error_analysis', 'det_error_file.txt'),
                         image_ids, class_names, lines)
  return stats


def main(argv=None):
  eval_once(parse_flags(argv))


if __name__ == '__main__':
  main()
