"""GPU debug driver: end-to-end accuracy of the SqueezeDet forward against the fp64 oracle
(truth) next to the fp32 oracle's own error, at the smoke() configuration.
Usage: python tests/debug_accuracy.py [tc|simt]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import oracle
from squeezedet_b200 import _lib
from squeezedet_b200 import config as cfg
from squeezedet_b200.nets import SqueezeDet
from squeezedet_b200.utils import synth

mode = sys.argv[1] if len(sys.argv) > 1 else 'tc'
width, height, batch = 416, 128, 2
mc = cfg.kitti_squeezeDet_config()
mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT, mc.BATCH_SIZE = width, height, batch
grid = oracle.layer_table('squeezeDet', height, width)[-1][2]
mc.GRID_H, mc.GRID_W = grid[0], grid[1]
mc.ANCHOR_BOX = cfg.set_anchors(mc)
mc.ANCHORS = len(mc.ANCHOR_BOX)
model = SqueezeDet(mc, 0, math_mode=_lib.MATH_TF32X3_TC if mode == 'tc' else _lib.MATH_FP32_SIMT)
weights = synth.synthetic_weights(synth.model_param_specs(model), seed=0)
model.load_weights(weights)
images = synth.synthetic_images(batch, height, width, seed=1234)
boxes, probs, cls = model.detect(images)
got_preds = model.read_tensor('conv12')

def run(dtype):
  preds = oracle.forward('squeezeDet', weights, images, dtype=dtype)
  return preds, oracle.interpret_output(preds, mc.ANCHOR_BOX, mc.CLASSES, mc.ANCHOR_PER_GRID,
                                        width, height, mc.EXP_THRESH, dtype)
p32, (b32, s32, c32) = run(np.float32)
p64, (b64, s64, c64) = run(np.float64)
sc = np.abs(p64).max()
print('mode %s' % mode)
print('preds  max|gpu-f64|/max %.3e   max|f32-f64|/max %.3e   mean signed (gpu-f64)/|f64| %.3e'
      % (np.abs(got_preds - p64).max() / sc, np.abs(p32 - p64).max() / sc,
         np.mean((got_preds - p64) * np.sign(p64)) / np.mean(np.abs(p64))))
def viol(a, b):
  return int((np.abs(a - b) > 1e-3 + 1e-4 * np.abs(b)).sum())
print('boxes  max|gpu-f64| %.3e  max|f32-f64| %.3e  max|gpu-f32| %.3e'
      % (np.abs(boxes - b64).max(), np.abs(b32 - b64).max(), np.abs(boxes - b32).max()))
print('boxes  strict-tol violations: gpu vs f32 %d   gpu vs f64 %d   f32 vs f64 %d   of %d'
      % (viol(boxes, b32), viol(boxes, b64), viol(b32, b64), boxes.size))
print('scores max|gpu-f64| %.3e  max|f32-f64| %.3e' % (np.abs(probs - s64).max(), np.abs(s32 - s64).max()))
print('class mismatches gpu vs f64 %d, f32 vs f64 %d' % (int((cls != c64).sum()), int((c32 != c64).sum())))
