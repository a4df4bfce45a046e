"""The fused first layer (conv_pool_simt_kernel) against the unfused FFMA path, bitwise, across the
strip geometry: each CTA walks a strip of an even number of pooled rows (2 .. 16, chosen by the
launcher from the batch and the device) over 31 pooled columns, two pooled rows per step, and
carries the conv row two pooled rows share from one step to the next.

The rows reach:
  * strips of several steps: at these sizes a strip of 2 would take more CTAs than the device
    holds at once, so the launcher picks a taller one and the carried row is used;
  * a short last strip: an odd pooled height is never a multiple of an even strip height, so the
    last strip is short and ends on a half-used step;
  * a single pooled row, a single pooled pixel, and pooled widths that are a multiple of 31, one
    more than a multiple, and other remainders;
  * both conv and pool paddings for k = 3 and 7, the frozen-BN epilogue, and the four kernel
    instances (k = 3 / 7 by 256 / 384 threads, 64 threads per 16 channels);
  * uint8 input at byte offsets 0 .. 3, which must match the fp32 instance on the converted images.
"""
import numpy as np
import pytest

import oracle
from gpu_util import assert_fused_away, build, conv2d_gpu, maxpool_gpu
from squeezedet_b200 import _lib
from squeezedet_b200._lib import DeviceBuffer
from squeezedet_b200.utils import synth

# (Cout, ksize, conv padding, pool padding, frozen BN, H, W, B)
ROWS = [
    (64, 3, 'VALID', 'VALID', False, 375, 1242, 3),   # SqueezeDet: 93 x 310 pooled, 10 x 31 exactly
    (64, 3, 'SAME', 'SAME', False, 371, 1242, 3),     # 93 x 311: a last column tile 1 wide
    (64, 7, 'SAME', 'VALID', True, 375, 1242, 2),     # ResNet-50's conv1 + pool1: 93 x 310
    (96, 7, 'VALID', 'VALID', False, 375, 1242, 2),   # SqueezeDet+: 92 x 308
    (96, 3, 'SAME', 'VALID', False, 301, 700, 3),     # 75 x 174
    (48, 7, 'VALID', 'SAME', False, 333, 509, 4),     # 82 x 126, 192 threads
    (16, 3, 'SAME', 'SAME', False, 255, 380, 4),      # 64 x 95, 64 threads
    (32, 3, 'VALID', 'VALID', False, 7, 900, 2),      # a single pooled row, 1 x 224
    (80, 3, 'VALID', 'SAME', False, 5, 6, 3),         # a single pooled pixel
    (80, 7, 'SAME', 'SAME', False, 97, 130, 3),       # 25 x 33 on 320 threads
    (32, 3, 'SAME', 'VALID', True, 150, 200, 3),      # 37 x 49, BN on 128 threads
]
U8_ROWS = [ROWS[0], ROWS[2], ROWS[3], ROWS[4]]


def row_id(r):
  return '%dc-k%d-%s-%s%s-%dx%d-b%d' % (r[0], r[1], r[2], r[3], '-bn' if r[4] else '', r[5], r[6],
                                        r[7])


def fused_model(row, device):
  cout, k, cpad, ppad, bn, height, width, B = row
  body = [('conv', 'conv1', cout, k, 2, cpad), ('pool', 'pool1', 3, 2, ppad)]
  mc, model, weights = build(body, B, height, width, _lib.MATH_TF32X3_TC, device,
                             ('conv1',) if bn else ())
  return mc, model, weights


def fused_pool1(model, images):
  buf = DeviceBuffer.from_numpy(np.ascontiguousarray(images, np.float32), model.gpu_id)
  model.forward_device(buf.ptr, None)
  _lib.check(model._lib.sqdet_stream_sync(model.gpu_id, None))
  buf.free()
  return model.read_tensor('pool1')


def bn_affine(weights, eps):
  """The engine's fold of a frozen BN into a per-channel scale and shift, in float32."""
  g, b, m, v = [np.asarray(weights['conv1/' + n], np.float32) for n in ('gamma', 'beta', 'mean',
                                                                       'var')]
  inv = (np.float32(1.0) / np.sqrt(v + np.float32(eps))) * g
  return inv, b - m * inv


def test_rows_reach_the_strip_classes():
  """What the table above claims to reach, from the pooled geometry alone."""
  seen = []
  for cout, k, cpad, ppad, bn, height, width, B in ROWS:
    hc = oracle.conv_geometry(height, k, 2, cpad)[0]
    wc = oracle.conv_geometry(width, k, 2, cpad)[0]
    hp = oracle.conv_geometry(hc, 3, 2, ppad)[0]
    wp = oracle.conv_geometry(wc, 3, 2, ppad)[0]
    seen.append(dict(hp=hp, wp=wp, k=k, pads=(cpad, ppad), bn=bn, wide=4 * cout > 256,
                     many=B * ((hp + 1) // 2) * ((wp + 30) // 31) > 132 * 8))
  assert any(s['hp'] % 2 and s['many'] for s in seen)          # short last strip, several steps
  assert any(s['hp'] == 1 and s['wp'] > 31 for s in seen)
  assert any(s['hp'] == s['wp'] == 1 for s in seen)
  assert {s['wp'] % 31 for s in seen} >= {0, 1} and len({s['wp'] % 31 for s in seen}) > 4
  assert {(s['k'], s['pads']) for s in seen} == {(k, (cp, pp)) for k in (3, 7)
                                                 for cp in ('SAME', 'VALID')
                                                 for pp in ('SAME', 'VALID')}
  assert {(s['k'], s['wide']) for s in seen} == {(k, w) for k in (3, 7) for w in (False, True)}
  assert {s['k'] for s in seen if s['bn']} == {3, 7}
  assert all(s['pads'][0] == 'SAME' for s in seen if s['bn'])      # _conv_bn_layer: SAME only
  assert all(16 <= r[0] <= 96 and r[0] % 16 == 0 for r in ROWS)


@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=row_id)
def test_fused_equals_unfused(row, gpu_device):
  """pool1 of the fused kernel equals sqdet_conv2d in the SIMT math mode (bias, BN as the engine
  folds it, ReLU) followed by sqdet_maxpool_nhwc, bit for bit."""
  cout, k, cpad, ppad, bn, height, width, B = row
  mc, model, weights = fused_model(row, gpu_device)
  images = synth.synthetic_images(B, height, width, seed=height + width + cout)
  pooled = fused_pool1(model, images)
  assert_fused_away(model, 'conv1')
  scale, shift = bn_affine(weights, mc.BATCH_NORM_EPSILON) if bn else (None, None)
  conv = conv2d_gpu(images, weights['conv1/kernels'], weights.get('conv1/biases'), 2, cpad,
                    relu=True, scale=scale, shift=shift, math_mode=_lib.MATH_FP32_SIMT,
                    device=gpu_device)
  unfused = maxpool_gpu(conv, 3, 2, ppad, device=gpu_device)
  assert pooled.shape == unfused.shape
  diff = np.argwhere(pooled.view(np.uint32) != unfused.view(np.uint32))
  assert len(diff) == 0, ('fused and unfused first layer differ', len(diff), tuple(diff[0]),
                          float(pooled[tuple(diff[0])]), float(unfused[tuple(diff[0])]))


@pytest.mark.gpu
@pytest.mark.parametrize('row', U8_ROWS, ids=row_id)
def test_u8_equals_fp32(row, gpu_device):
  """The uint8 instance at byte offsets 0 .. 3 against the fp32 instance on the converted images."""
  cout, k, cpad, ppad, bn, height, width, B = row
  mc, model, _ = fused_model(row, gpu_device)
  u8 = np.random.default_rng(height * width + cout).integers(0, 256, (B, height, width, 3),
                                                             dtype=np.uint8)
  conv = (u8.astype(np.float64) - np.asarray(mc.BGR_MEANS, np.float64).reshape(3)).astype(
      np.float32)
  want = fused_pool1(model, conv)
  for offset in range(4):
    flat = np.concatenate([np.full(offset, 0xA5, np.uint8), u8.ravel(), np.full(7, 0x5A, np.uint8)])
    buf = DeviceBuffer.from_numpy(flat, gpu_device)
    model.forward_device_u8(buf.ptr + offset, None)
    _lib.check(model._lib.sqdet_stream_sync(gpu_device, None))
    buf.free()
    got = model.read_tensor('pool1')
    assert got.tobytes() == want.tobytes(), ('offset', offset)
