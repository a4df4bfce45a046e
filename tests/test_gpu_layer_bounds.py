"""Every layer of the benchmark networks checked on its own, per element, against fp64.

The oracle of each layer is fed the engine's own read-back input for that layer (teacher
forcing), so errors do not compound from layer to layer and the per-element bound of the
stage-isolated tests (gpu_util.adv_tol) applies unchanged at the benchmark's shapes,
batch and dispatch:

    |got - want64| <= tol(K) * (|x| (*) |w| + |b|),    tol(K) = 1.2e-7 * sqrt(K),  K = k*k*Cin.

LayerChecker is a tracer for oracle.nets.NET_BUILDERS, like oracle.torch_port._TorchTracer: each
conv / conv_bn / pool / fire call computes that one layer in fp64 (torch on the CPU, with the TF
SAME padding of _TorchTracer) on the engine's input, compares the engine's output with it, and
returns the engine's tensor, so the next layer is fed what the GPU computed.  ResNet's
`S.relu(sc + y)` then runs on the engine's fp32 tensors, which is exactly add_relu_kernel.

Rules per layer kind:
  * conv [+ ReLU], the head: the bound above (ReLU is 1-Lipschitz);
  * conv + frozen BN: the conv term scaled by the fp64 BN scale, plus BN_ULPS ulps of the affine
    (derived at BN_ULPS);
  * conv fused with the 3x3/2 pool (the conv tensor reads as not found): max_pool of the fp64 conv
    against max_pool of the conv bound (a max over a window moves by at most the largest move of
    its inputs);
  * one-kernel fire (the squeeze tensor reads as not found): gpu_util.fire_oracle in fp64,
    per element against the bar of test_gpu_fire.fire_bound_ratio;
  * squeeze + expand pair, or three SIMT convs: the conv rule for the squeeze on the fire input and
    for each expand on the engine's squeeze tensor;
  * max-pool and add + ReLU: bitwise equal.

Only the first and the last image of each tensor are checked on the CPU; the GPU runs the whole
batch, and the last image exercises the batch offsets.  The numpy fp32 oracle (oracle.conv2d in
float32, a plain fp32 sum), run on the same engine input, must meet every bound too: a check of the
bar itself.  It runs on the first checked image only."""
import numpy as np
import pytest
import torch

import oracle
from oracle.nets import NET_BUILDERS
from oracle.torch_port import _TorchTracer
from squeezedet_b200 import _lib
from squeezedet_b200.utils import synth
from gpu_util import (ERR_NOT_FOUND, MODES, ONE_KERNEL_MIN_TILES, PAIR_MAX_TILES, adv_tol,
                      assert_fused_away, bound_ratio, build, conv2d_gpu, engine_tensor,
                      fire_error_bound, fire_oracle, fire_tiles, make_net, maxpool_gpu)

U = 2.0 ** -24         # unit roundoff of fp32 round-to-nearest

# Frozen BN.  The engine computes scale' = fl(fl(1 / fl(sqrtf(fl(var + eps)))) * gamma) and
# shift' = fl(beta - fl(mean * scale')) in fp32 on the host (engine.cu prepare_params), then
# y' = fl(t * scale' + shift') after the conv (an FMA or a multiply and an add), where t is the
# conv + bias with |t - c| <= the conv bound E.  With s = gamma / sqrt(var + eps) and
# h = beta - mean * s exact, to first order in U:
#   |scale' - s| <= 4U |s|: eps in fp32 and the add (2U on var + eps, U after the square root),
#                           the square root, the reciprocal and the product with gamma (U each);
#   |shift' - h| <= U |beta| + 6U |mean s|: 4U |mean s| from scale', U from the product, and the
#                           subtraction's U |shift'| <= U (|beta| + |mean s|);
#   affine rounding <= U |t s| + U |y'| <= 2U |c s| + U |beta| + U |mean s|.
# With E carried through the scale, |y' - y| <= |s| E + 6U |c s| + 2U |beta| + 7U |mean s|
#                                            <= |s| E + 7U (|c s| + |beta| + |mean s|).
# The second-order terms (U^2, U E) are covered by rounding 7 up to 8.  The numpy fp32 oracle
# (oracle.batch_norm_frozen in float32) takes the same steps, so the same bound holds for it.
BN_ULPS = 8


def _nchw(x):
  return torch.from_numpy(np.ascontiguousarray(x)).permute(0, 3, 1, 2).to(torch.float64)


def _nhwc(t):
  return t.permute(0, 2, 3, 1).contiguous().numpy()


class _Fused:
  """A conv the engine never writes (it is fused into the pool that follows): its fp64 value and
  per-element bar on the checked images, K, and the numpy fp32 oracle on the first image."""

  def __init__(self, want, bar, K, want32):
    self.want, self.bar, self.K, self.want32 = want, bar, K, want32


class LayerChecker:
  """Tracer for oracle.nets.NET_BUILDERS that checks each layer on the engine's own input.

  `read(name)` returns the engine's tensor `name` restricted to the checked images (batch indices
  `images`), or None when the engine never materialises it.  `rows[name]` = (rule, worst ratio of
  error to bar, K) for every checked layer; `failures` collects one message per failing layer."""

  def __init__(self, weights, read, images, keep_bars=False):
    self.w = weights
    self.read = read
    self.images = list(images)
    self.t64 = _TorchTracer(weights, np.float64)
    self.tabs = _TorchTracer({k: np.abs(v) for k, v in weights.items()}, np.float64)
    self.rows = {}
    self.failures = []
    self.bars = {} if keep_bars else None

  # ---- comparisons -----------------------------------------------------------------------------
  def _need(self, name):
    got = self.read(name)
    assert got is not None, '%s: the engine did not materialise this tensor' % name
    return got

  def _bounded(self, name, rule, got, want, bar, K, record=True):
    if got.shape != want.shape:
      self.failures.append('%s (%s): shape %s, want %s' % (name, rule, got.shape, want.shape))
      return
    ratio = bound_ratio(got, want, bar)
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    r = float(ratio[worst])
    if record:
      self.rows[name] = (rule, r, K)
      if self.bars is not None:
        self.bars[name] = bar
    if not r < 1.0:
      self.failures.append(
          '%s (%s): image %d, element (y, x, c) = %s: |got - want| = %.4g is %.3g x the bar %.4g '
          '(got %r, want %r), K = %d' % (name, rule, self.images[worst[0]],
                                          tuple(int(v) for v in worst[1:]),
                                          abs(float(got[worst]) - want[worst]), r,
                                          bar[worst], float(got[worst]), float(want[worst]), K))

  def _sanity(self, name, rule, want32, want, bar, K):
    """The numpy fp32 oracle on the same input (first checked image) meets the same bar."""
    self._bounded(name + ' [numpy fp32 oracle]', rule, want32, want[:1], bar[:1], K, record=False)

  def _bitwise(self, name, rule, got, want):
    self.rows[name] = (rule, 0.0, 0)
    if got.shape != want.shape:
      self.failures.append('%s (%s): shape %s, want %s' % (name, rule, got.shape, want.shape))
    elif not np.array_equal(got, want):
      bad = np.argwhere(got != want)
      i = tuple(int(v) for v in bad[0])
      self.rows[name] = (rule, np.inf, 0)
      self.failures.append('%s (%s): %d elements differ; first at image %d, (y, x, c) = %s: got '
                           '%r, want %r' % (name, rule, len(bad), self.images[i[0]], i[1:],
                                            float(got[i]), float(want[i])))

  # ---- layer oracles ---------------------------------------------------------------------------
  def _conv64(self, scope, x, size, stride, padding, bias):
    """fp64 conv (+ bias) of the engine's input, and its magnitude |x| (*) |w| (+ |b|)."""
    xt = _nchw(x)
    want = self.t64._conv(scope, xt, size, stride, padding, bias)
    mag = self.tabs._conv(scope, xt.abs(), size, stride, padding, bias)
    return _nhwc(want), _nhwc(mag)

  def _conv(self, name, x, size, stride, padding, relu, got):
    """The conv rule for `got` (None: fused into the next pool, returns a _Fused)."""
    K = size * size * x.shape[3]
    want, mag = self._conv64(name, x, size, stride, padding, True)
    if relu:
      want = np.maximum(want, 0)
    bar = adv_tol(K) * mag
    want32 = oracle.conv2d(x[:1], self.w[name + '/kernels'], self.w[name + '/biases'], stride,
                           padding, relu, np.float32)
    if got is None:
      return _Fused(want, bar, K, want32)
    self._bounded(name, 'conv', got, want, bar, K)
    self._sanity(name, 'conv', want32, want, bar, K)
    return got

  def conv(self, name, x, filters, size, stride, padding='SAME', relu=True):
    return self._conv(name, x, size, stride, padding, relu, self.read(name))

  def conv_bn(self, scope, x, filters, size, stride, relu=True, bias=False, eps=1e-5):
    K = size * size * x.shape[3]
    c, mag = self._conv64(scope, x, size, stride, 'SAME', bias)
    mean, var, beta, gamma = [self.w[scope + '/' + k] for k in ('mean', 'var', 'beta', 'gamma')]
    want = oracle.batch_norm_frozen(c, *[np.asarray(v, np.float64) for v in (mean, var, beta,
                                                                           gamma)], eps)
    s = np.asarray(gamma, np.float64) / np.sqrt(np.asarray(var, np.float64) + eps)
    bar = (np.abs(s) * adv_tol(K) * mag +
           BN_ULPS * U * (np.abs(c * s) + np.abs(np.asarray(beta, np.float64)) +
                          np.abs(np.asarray(mean, np.float64) * s)))
    y32 = oracle.conv2d(x[:1], self.w[scope + '/kernels'],
                        self.w[scope + '/biases'] if bias else None, stride, 'SAME', False,
                        np.float32)
    want32 = oracle.batch_norm_frozen(y32, mean, var, beta, gamma, eps)
    if relu:
      want, want32 = np.maximum(want, 0), np.maximum(want32, 0).astype(np.float32)
    got = self.read(scope)
    if got is None:
      return _Fused(want, bar, K, want32)
    self._bounded(scope, 'conv + BN', got, want, bar, K)
    self._sanity(scope, 'conv + BN', want32, want, bar, K)
    return got

  def pool(self, name, x, size, stride, padding='SAME'):
    got = self._need(name)
    if isinstance(x, _Fused):
      want = oracle.max_pool(x.want, size, stride, padding)
      bar = oracle.max_pool(x.bar, size, stride, padding)
      self._bounded(name, 'conv + pool', got, want, bar, x.K)
      self._sanity(name, 'conv + pool', oracle.max_pool(x.want32, size, stride, padding), want,
                   bar, x.K)
    else:
      self._bitwise(name, 'max-pool', got, oracle.max_pool(x, size, stride, padding))
    return got

  def fire(self, name, x, s1x1, e1x1, e3x3):
    got = self._need(name)
    q = self.read(name + '/squeeze1x1')
    if q is None:
      ws, bs, w1, b1, w3, b3 = [self.w[name + sub] for sub in (
          '/squeeze1x1/kernels', '/squeeze1x1/biases', '/expand1x1/kernels',
          '/expand1x1/biases', '/expand3x3/kernels', '/expand3x3/biases')]
      want = fire_oracle(x, ws, bs, w1, b1, w3, b3, dtype=np.float64)
      q64 = oracle.conv2d(x, ws, bs, 1, 'SAME', True, np.float64)
      # test_gpu_fire.fire_bound_ratio's bar, element by element
      K = max(x.shape[3], 9 * s1x1)
      bar = adv_tol(K) * fire_error_bound(x, ws, w1, w3, q64)
      self._bounded(name, 'fire, one kernel', got, want, bar, K)
      self._sanity(name, 'fire, one kernel',
                   fire_oracle(x[:1], ws, bs, w1, b1, w3, b3, dtype=np.float32), want, bar, K)
      return got
    q = self._conv(name + '/squeeze1x1', x, 1, 1, 'SAME', True, q)
    self._conv(name + '/expand1x1', q, 1, 1, 'SAME', True, got[..., :e1x1])
    self._conv(name + '/expand3x3', q, 3, 1, 'SAME', True, got[..., e1x1:])
    return got

  def _rec(self, name, kind, y, flops=0, params=0):
    """ResNet's relu(shortcut + branch), computed by the builder on the engine's fp32 tensors."""
    assert kind == 'add_relu' and y.dtype == np.float32, (name, kind, y.dtype)
    got = self._need(name)
    self._bitwise(name, 'add + ReLU', got, y)
    return got

  # ---- results -----------------------------------------------------------------------------------
  def assert_ok(self):
    assert not self.failures, '\n'.join(self.failures)

  def worst(self):
    """(layer, rule, ratio, K) of the largest err / bar among the bounded layers."""
    name = max(self.rows, key=lambda n: self.rows[n][1])
    return (name,) + self.rows[name]


def engine_reader(model, images):
  """read() for LayerChecker over an engine: the tensor's checked images, or None when the engine
  reports it as not materialised (fused into its consumer)."""
  def read(name):
    try:
      full = model.read_tensor(engine_tensor(model, name))
    except _lib.SqdetError as exc:
      assert exc.code == ERR_NOT_FOUND, (name, exc)
      return None
    return full[images]
  return read


def checked_images(batch):
  return sorted({0, batch - 1})


def report(tag, t):
  name, rule, ratio, K = t.worst()
  print('\n%s: %d layers, worst err / bar %.3f at %s (%s, K = %d)'
        % (tag, len(t.rows), ratio, name, rule, K))


# ---- the benchmark configurations (1242 x 375) --------------------------------------------------
CONFIGS = [('squeezeDet', 20), ('squeezeDet', 1), ('squeezeDet+', 20), ('resnet50', 8),
           ('vgg16', 8)]
HEIGHT, WIDTH = 375, 1242


@pytest.mark.gpu
@pytest.mark.parametrize('math_mode', MODES)
@pytest.mark.parametrize('net,batch', CONFIGS)
def test_benchmark_layers_within_fp64_bound(net, batch, math_mode, gpu_device):
  """Each layer of the net at 1242 x 375 and the batch the benchmark runs, with the dispatch this
  check is meant to see asserted first."""
  model, weights = make_net(net, WIDTH, HEIGHT, batch, gpu_device, math_mode, seed=0)
  mc = model.mc
  images = synth.synthetic_images(batch, HEIGHT, WIDTH, seed=1234)
  model.detect(images)
  tc = math_mode == _lib.MATH_TF32X3_TC
  one_kernel = ()
  if net != 'vgg16':
    # conv1 + pool1 as one kernel: SqueezeDet 3x3 SAME / SAME pool, SqueezeDet+ 7x7 VALID at 96
    # channels (the 384-thread instance), ResNet-50 7x7 SAME + BN / VALID pool
    assert_fused_away(model, 'conv1')
  if net == 'squeezeDet':
    tiles = fire_tiles(batch, 94, 311)
    if batch == 20:
      assert tiles >= ONE_KERNEL_MIN_TILES
      one_kernel = ('fire2', 'fire3') if tc else ()
    else:
      assert tiles < PAIR_MAX_TILES
    for fire in one_kernel:
      assert_fused_away(model, fire + '/squeeze1x1')
  idx = checked_images(batch)
  t = LayerChecker(weights, engine_reader(model, idx), idx)
  NET_BUILDERS[net](t, images[idx], mc.ANCHOR_PER_GRID * (mc.CLASSES + 5))
  # the checker took the paths asserted above, and no other
  if net != 'vgg16':
    assert t.rows['pool1'][0] == 'conv + pool'
  else:
    assert t.rows['conv1/conv1_1'][0] == 'conv'
  fires = [n for n, row in t.rows.items() if row[0] == 'fire, one kernel']
  assert fires == list(one_kernel), fires
  if net.startswith('squeezeDet'):
    squeezes = {n for n in t.rows if n.endswith('/squeeze1x1')}
    assert squeezes == {'fire%d/squeeze1x1' % i for i in range(2, 12)} - \
        {f + '/squeeze1x1' for f in one_kernel}
  if net == 'resnet50':
    assert sum(row[0] == 'add + ReLU' for row in t.rows.values()) == 13
  report('%s b=%d %s' % (net, batch, 'tf32x3' if tc else 'simt'), t)
  t.assert_ok()


# ---- the fused first layer across its geometry ---------------------------------------------------
# (Cout, ksize, conv padding, pool padding, frozen BN, H, W), B = 3 and a 72-channel ConvDet head.
# test_host_logic.test_first_layer_table_reaches_every_class checks what the rows reach.
FIRST_LAYER_ROWS = [
    (64, 3, 'SAME', 'SAME', False, 130, 257),
    (96, 3, 'SAME', 'VALID', False, 41, 128),
    (32, 3, 'VALID', 'SAME', False, 5, 6),        # pools to a single pixel
    (80, 3, 'VALID', 'VALID', False, 64, 263),
    (48, 7, 'SAME', 'SAME', False, 32, 256),
    (64, 7, 'SAME', 'VALID', True, 45, 99),       # ResNet-50's conv1 + pool1
    (96, 7, 'VALID', 'VALID', False, 20, 50),     # less than one 4 x 16 pooled tile
    (80, 7, 'VALID', 'SAME', False, 77, 140),
]
FIRST_LAYER_BATCH = 3


@pytest.mark.gpu
@pytest.mark.parametrize('math_mode', MODES)
@pytest.mark.parametrize('row', FIRST_LAYER_ROWS, ids=lambda r: '%dc-k%d-%s-%s%s-%dx%d' % (
    r[0], r[1], r[2], r[3], '-bn' if r[4] else '', r[5], r[6]))
def test_first_layer_conv_pool_bounds(row, math_mode, gpu_device):
  """conv_pool_simt_kernel on one geometry: the per-element bound of the fused conv + pool, and
  for rows without BN, value equality with the unfused FFMA path (sqdet_conv2d in the SIMT math
  mode, then sqdet_maxpool_nhwc).  Both kernels sum the same products in the same order (one fmaf
  per K index in HWIO order from 0, then the bias, then the ReLU) and max is exact, so the two
  must agree exactly."""
  cout, k, cpad, ppad, bn, height, width = row
  body = [('conv', 'conv1', cout, k, 2, cpad), ('pool', 'pool1', 3, 2, ppad)]
  bn_convs = ('conv1',) if bn else ()
  B = FIRST_LAYER_BATCH
  mc, model, weights = build(body, B, height, width, math_mode, gpu_device, bn_convs)
  images = synth.synthetic_images(B, height, width, seed=11)
  model.detect(images)
  assert_fused_away(model, 'conv1')
  idx = checked_images(B)
  t = LayerChecker(weights, engine_reader(model, idx), idx)
  x = images[idx]
  if bn:
    x = t.conv_bn('conv1', x, cout, k, 2, relu=True, bias=True, eps=mc.BATCH_NORM_EPSILON)
  else:
    x = t.conv('conv1', x, cout, k, 2, cpad)
  x = t.pool('pool1', x, 3, 2, ppad)
  t.conv('conv12', x, mc.ANCHOR_PER_GRID * (mc.CLASSES + 5), 3, 1, 'SAME', relu=False)
  assert t.rows['pool1'][0] == 'conv + pool'
  print('\nfirst layer %s: pool1 err / bar %.3f' % (row, t.rows['pool1'][1]))
  t.assert_ok()
  if not bn:
    pooled = model.read_tensor('pool1')
    conv = conv2d_gpu(images, weights['conv1/kernels'], weights['conv1/biases'], 2, cpad,
                      relu=True, math_mode=_lib.MATH_FP32_SIMT, device=gpu_device)
    unfused = maxpool_gpu(conv, 3, 2, ppad, device=gpu_device)
    assert pooled.shape == unfused.shape
    diff = np.argwhere(pooled != unfused)
    assert len(diff) == 0, ('fused and unfused first layer differ', len(diff),
                            tuple(diff[0]), float(pooled[tuple(diff[0])]),
                            float(unfused[tuple(diff[0])]))


# ---- the checker itself, with the numpy fp32 oracle standing in for the engine -------------------
SELF_TEST_SIZES = {'squeezeDet': (67, 118), 'squeezeDet+': (69, 117), 'vgg16': (48, 80),
                   'resnet50': (67, 99)}
SELF_TEST_BATCH = 3
FUSED_IN_SELF_TEST = ('conv1', 'fire2/squeeze1x1', 'fire3/squeeze1x1')


def stand_in(net, move=None, ulp=None, keep_bars=False):
  """A LayerChecker run over the numpy fp32 oracle's tensors, as the engine would hand them back,
  with conv1 and the first two fire squeezes reading as fused away.  `move` = (layer, index):
  push that element of the stand-in away from fp64 by twice its bar (from a clean run);
  `ulp` = (layer, index): move that element up by one ulp.  `keep_bars`: keep every bounded
  layer's bar in the checker's `bars`."""
  height, width = SELF_TEST_SIZES[net]
  weights = synth.synthetic_weights(oracle.param_specs(net), seed=2)
  images = synth.synthetic_images(SELF_TEST_BATCH, height, width, seed=5)
  keep = {}
  oracle.forward(net, weights, images, dtype=np.float32, keep=keep)
  idx = checked_images(SELF_TEST_BATCH)
  tensors = {n: np.array(v[idx]) for n, v in keep.items() if n not in FUSED_IN_SELF_TEST}
  if move is not None:
    name, i, delta = move
    tensors[name][i] += np.float32(delta)
  if ulp is not None:
    name, i = ulp
    tensors[name][i] = np.nextafter(tensors[name][i], np.float32(np.inf))
  t = LayerChecker(weights, tensors.get, idx, keep_bars)
  NET_BUILDERS[net](t, images[idx], 72)
  return t


@pytest.mark.parametrize('net', sorted(SELF_TEST_SIZES))
def test_layer_checker_self_test(net):
  """Without a GPU: every layer of the fp32 oracle passes; one element moved by twice its bar fails
  and the message names the layer and the element; a bitwise layer one ulp off fails."""
  t = stand_in(net, keep_bars=True)
  t.assert_ok()
  assert t.rows, net
  if net.startswith('squeezeDet'):
    assert t.rows['pool1'][0] == 'conv + pool'
    assert t.rows['fire2'][0] == t.rows['fire3'][0] == 'fire, one kernel'
    assert t.rows['fire4/squeeze1x1'][0] == 'conv'
  if net == 'resnet50':
    assert t.rows['pool1'][0] == 'conv + pool'
  # move one element of a bounded layer in the last image by 2x its bar
  layer = {'squeezeDet': 'fire5/squeeze1x1', 'squeezeDet+': 'fire9/squeeze1x1',
           'vgg16': 'conv4/conv4_2',
           'resnet50': 'conv3_x/res3b/res3b_branch2/res3b_branch2b'}[net]
  bar = t.bars[layer]
  i = (1,) + tuple(int(n) // 2 for n in bar.shape[1:])
  assert bar[i] > 0
  bad = stand_in(net, move=(layer, i, 2 * bar[i]))
  # the layer fails first; its consumer may fail too, because the stand-in's next tensor was not
  # computed from the moved element, as an engine's would be
  assert bad.failures and bad.failures[0].startswith(layer + ' ('), bad.failures
  assert 'image %d, element (y, x, c) = %s' % (SELF_TEST_BATCH - 1, i[1:]) in bad.failures[0]
  assert 'is 2 x the bar' in bad.failures[0], bad.failures[0]
  # a bitwise layer one ulp off
  bitwise = {'squeezeDet': 'pool3', 'squeezeDet+': 'pool4', 'vgg16': 'pool2',
             'resnet50': 'res2b'}[net]
  bad = stand_in(net, ulp=(bitwise, (0, 1, 2, 3)))
  assert bad.failures and bad.failures[0].startswith(bitwise + ' ('), bad.failures
  assert '1 elements differ; first at image 0, (y, x, c) = (1, 2, 3)' in bad.failures[0]

