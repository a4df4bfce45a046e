"""What the engine runs, layer by layer.  Small nets are built from a FireNetBase table
(squeezedet_b200/nets/squeezeDet.py), every tensor the engine can hand back is checked against a
chained numpy oracle, and launches_per_forward() tells which kernel path each op took:
  * the first layer: Cin = 3 stride-2 conv + 3x3/2 pool as one FFMA kernel, at every width the
    fused kernel accepts (16..96) and one above it;
  * a fire module as one kernel (16-channel squeeze on a grid of >= 4 tiles per SM) against the
    squeeze conv + expand pair (two launches), and the SIMT path (three launches).
Bar per tensor (test_gpu_e2e.test_layerwise_parity_small_image): within 1e-4 of the fp32
reference, and no further from fp64 than 4x the fp32 reference's own distance."""
import numpy as np
import pytest

import oracle
from squeezedet_b200 import _lib
from squeezedet_b200.utils import synth
from gpu_util import (MODES, ONE_KERNEL_MIN_TILES, PAIR_MAX_TILES, POST_LAUNCHES, TOL,
                      assert_fused_away, body_grid, build, engine_tensor, fire_oracle, fire_tiles,
                      rel_err)

pytestmark = pytest.mark.gpu


def oracle_layers(body, weights, images, dtype, bn_convs=(), eps=1e-5):
  """{tensor name: oracle value} for every body row, each fire's squeeze output and the head."""
  out = {}
  x = np.asarray(images, dtype)
  for row in body:
    kind, name = row[0], row[1]
    if kind == 'conv':
      _, k, s, pad = row[2:]
      kern, bias = weights[name + '/kernels'], weights[name + '/biases']
      if name in bn_convs:
        y = oracle.conv2d(x, kern, bias, s, 'SAME', False, dtype)
        y = oracle.batch_norm_frozen(y, weights[name + '/mean'], weights[name + '/var'],
                                     weights[name + '/beta'], weights[name + '/gamma'], eps)
        x = oracle.relu(y).astype(dtype)
      else:
        x = oracle.conv2d(x, kern, bias, s, pad, True, dtype)
    elif kind == 'pool':
      x = oracle.max_pool(x, *row[2:])
    else:
      p = [weights[name + sub] for sub in ('/squeeze1x1/kernels', '/squeeze1x1/biases',
                                           '/expand1x1/kernels', '/expand1x1/biases',
                                           '/expand3x3/kernels', '/expand3x3/biases')]
      out[name + '/squeeze1x1'] = oracle.conv2d(x, p[0], p[1], 1, 'SAME', True, dtype)
      x = fire_oracle(x, *p, dtype=dtype)
    out[name] = x
  out['conv12'] = oracle.conv2d(x, weights['conv12/kernels'], weights['conv12/biases'], 1, 'SAME',
                                False, dtype)
  return out


def assert_layer(model, name, want64, want32):
  got = model.read_tensor(engine_tensor(model, name))
  assert got.shape == want64[name].shape, name
  assert rel_err(got, want32[name]) < TOL, (name, rel_err(got, want32[name]))
  e_gpu, e_ref = rel_err(got, want64[name]), rel_err(want32[name], want64[name])
  assert e_gpu < max(4 * e_ref, 2e-5), (name, e_gpu, e_ref)


def run(body, batch, height, width, math_mode, device, bn_convs=()):
  mc, model, weights = build(body, batch, height, width, math_mode, device, bn_convs)
  images = synth.synthetic_images(batch, height, width, seed=11)
  model.detect(images)
  want64 = oracle_layers(body, weights, images, np.float64, bn_convs, mc.BATCH_NORM_EPSILON)
  want32 = oracle_layers(body, weights, images, np.float32, bn_convs, mc.BATCH_NORM_EPSILON)
  return model, want64, want32


# ---- first layer: conv (Cin = 3, stride 2) -> 3x3/2 max-pool ---------------------------------
FIRST_LAYER_CASES = [
    # Cout, conv size, conv padding, pool padding, frozen-BN epilogue
    (16, 3, 'SAME', 'SAME', False),
    (16, 7, 'VALID', 'VALID', False),
    (32, 7, 'VALID', 'SAME', False),
    (48, 3, 'VALID', 'VALID', False),
    (64, 7, 'SAME', 'VALID', True),      # ResNet-50 conv1 + pool1
    (80, 3, 'SAME', 'VALID', False),
    (80, 7, 'SAME', 'SAME', False),
    (96, 7, 'VALID', 'VALID', False),
    (112, 3, 'SAME', 'SAME', False),     # wider than the fused kernel takes: conv, then pool
]


@pytest.mark.parametrize('math_mode', MODES)
@pytest.mark.parametrize('cout,size,cpad,ppad,bn', FIRST_LAYER_CASES)
def test_first_layer_conv_pool(cout, size, cpad, ppad, bn, math_mode, gpu_device):
  body = [('conv', 'conv1', cout, size, 2, cpad), ('pool', 'pool1', 3, 2, ppad)]
  bn_convs = ('conv1',) if bn else ()
  model, want64, want32 = run(body, 2, 61, 93, math_mode, gpu_device, bn_convs)
  fused = cout <= 96
  # conv1 [+ pool1] + head + post-processing
  assert model.launches_per_forward() == 1 + (0 if fused else 1) + 1 + POST_LAUNCHES
  if fused:
    assert_fused_away(model, 'conv1')
  else:
    assert_layer(model, 'conv1', want64, want32)
  assert_layer(model, 'pool1', want64, want32)
  assert_layer(model, 'conv12', want64, want32)


# ---- fire modules: one kernel vs squeeze + expand pair ---------------------------------------
@pytest.mark.parametrize('math_mode', MODES)
@pytest.mark.parametrize('cin', [32, 48])
def test_fire_one_kernel_layerwise(cin, math_mode, gpu_device):
  """A 16-channel squeeze on a 2 x 128 x 528 grid (1056 tiles): one kernel on the tensor-core
  path, so its squeeze tensor is never written and reads as not found.  The stride-1 3x3 first
  conv runs in gather mode; Cin = 48 reaches the KCI = 16 variant of the one-kernel fire."""
  batch, height, width = 2, 128, 528
  assert fire_tiles(batch, height, width) >= ONE_KERNEL_MIN_TILES
  body = [('conv', 'conv1', cin, 3, 1, 'SAME'), ('fire', 'fire2', 16, 64, 64),
          ('pool', 'pool2', 3, 2, 'SAME')]
  model, want64, want32 = run(body, batch, height, width, math_mode, gpu_device)
  fire_launches = 1 if math_mode == _lib.MATH_TF32X3_TC else 3
  # conv1 + fire2 + pool2 + head + post-processing
  assert model.launches_per_forward() == 1 + fire_launches + 1 + 1 + POST_LAUNCHES
  for name in ('conv1', 'fire2', 'pool2', 'conv12'):
    assert_layer(model, name, want64, want32)
  if math_mode == _lib.MATH_TF32X3_TC:
    assert_fused_away(model, 'fire2/squeeze1x1')
  else:
    assert_layer(model, 'fire2/squeeze1x1', want64, want32)


@pytest.mark.parametrize('math_mode', MODES)
def test_fire_expand_pair_layerwise(math_mode, gpu_device):
  """Fires on a 2 x 24 x 40 grid (18 tiles): squeeze conv, then the expand pair as one launch
  (tensor cores) or two SIMT convs.  S = 16; S = 48 (K chunks of 16 in the expand); E1 != E3 with
  ragged widths.  Every squeeze tensor is materialised and matches the oracle."""
  batch, height, width = 2, 96, 160
  body = [('conv', 'conv1', 64, 3, 2, 'SAME'), ('pool', 'pool1', 3, 2, 'SAME'),
          ('fire', 'fire2', 16, 64, 64), ('fire', 'fire3', 48, 64, 64),
          ('fire', 'fire4', 32, 40, 88)]
  assert fire_tiles(batch, *body_grid(body, height, width)) < PAIR_MAX_TILES
  model, want64, want32 = run(body, batch, height, width, math_mode, gpu_device)
  fire_launches = 2 if math_mode == _lib.MATH_TF32X3_TC else 3
  # conv1+pool1 (one kernel) + 3 fires + head + post-processing
  assert model.launches_per_forward() == 1 + 3 * fire_launches + 1 + POST_LAUNCHES
  assert_fused_away(model, 'conv1')
  for name in ('pool1', 'fire2/squeeze1x1', 'fire2', 'fire3/squeeze1x1', 'fire3',
               'fire4/squeeze1x1', 'fire4', 'conv12'):
    assert_layer(model, name, want64, want32)
