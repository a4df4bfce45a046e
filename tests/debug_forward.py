"""GPU debug driver: one profiled (non-graph) forward at the bench configuration."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from squeezedet_b200 import _lib, nets
from squeezedet_b200 import config as cfg
from squeezedet_b200.utils import synth

net = sys.argv[1] if len(sys.argv) > 1 else 'squeezeDet'
batch = int(sys.argv[2]) if len(sys.argv) > 2 else 20
cls, cf = {'squeezeDet': ('SqueezeDet', 'kitti_squeezeDet_config'),
           'squeezeDet+': ('SqueezeDetPlus', 'kitti_squeezeDetPlus_config'),
           'vgg16': ('VGG16ConvDet', 'kitti_vgg16_config'),
           'resnet50': ('ResNet50ConvDet', 'kitti_res50_config')}[net]
mc = getattr(cfg, cf)()
mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = 1242, 375, batch
mc.ANCHOR_BOX = cfg.set_anchors(mc)
model = getattr(nets, cls)(mc, 0)
model.load_weights(synth.synthetic_weights(synth.model_param_specs(model), seed=0))
x = _lib.DeviceBuffer.from_numpy(synth.synthetic_images(batch, 375, 1242))
model.forward_profiled(x.ptr)          # warm-up
sys.stderr.write('---- second pass ----\n')
rows = model.forward_profiled(x.ptr)
tot = 0
for (name, fl, pa, by), ms in rows:
  tot += ms
  print('%-18s %8.4f ms  %8.1f GB/s  %7.2f TFLOP/s' % (name, ms, by / ms / 1e6, fl / ms / 1e9))
print('total %.4f ms -> %.0f img/s' % (tot, batch / tot * 1e3))
