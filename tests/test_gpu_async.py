"""The engine's asynchronous paths against synchronous runs.

The engine issues work on its own non-blocking compute stream, a copy stream and the caller's
stream, and keeps four CUDA graphs keyed by (input, stream, n, box-scale table).  These tests leave
work queued while the next call changes engine state (a weight reload, a graph eviction, another
engine's thread) and compare every result bitwise with a synchronous run: a fresh engine with the
same weights, or the same engine on the legacy stream, which never uses a graph.  The kernels are
deterministic and the plan is the same, so any difference is an ordering bug, not rounding.

To make the in-flight window certain rather than a matter of timing, a stream is first held by a
bounded GPU spin (torch.cuda._sleep, torch and the library sharing the process and the device).
An event recorded behind the spin must still be pending when the racing call returns; otherwise
the run did not exercise the ordering and the test fails saying so."""
import functools
import threading

import numpy as np
import pytest
import torch

import oracle
from squeezedet_b200 import _lib
from squeezedet_b200.utils import synth
from gpu_util import MODES, assert_fused_away, fire_tiles, forward_n, make_net

pytestmark = pytest.mark.gpu

SPIN_CYCLES = 1_000_000_000      # 0.5 s at 1.98 GHz, longer at the clocks of a power-capped card
W1, W2 = 31, 32                  # weight seeds before and after a reload
# (height, width, batch).  SqueezeDet: fire2 and fire3 read 3 x 12 x 20 = 720 tiles of pool1's
# output, at least 4 per SM, so on tensor cores each runs as one kernel with its own weight pack.
# ResNet-50: frozen BN on tensor-core and SIMT convs, add+ReLU and strided convs.
SIZES = {'squeezeDet': (384, 1248, 3), 'resnet50': (99, 131, 2)}


@functools.lru_cache(maxsize=None)
def weights(net, seed):
  return synth.synthetic_weights(oracle.param_specs(net), seed=seed)


def sync(model, stream):
  _lib.check(model._lib.sqdet_stream_sync(model.gpu_id, stream))


def engine(net, mode, seed, device, size=None, scales=None):
  """An engine with weights `seed`, warmed by one forward on the legacy stream.  That forward is
  ordered behind the parameter uploads, so nothing is in flight afterwards."""
  h, w, b = size or SIZES[net]
  model, _ = make_net(net, w, h, b, device, mode, seed)
  if scales is not None:
    model.set_box_scale(scales)
  forward_n(model, np.zeros((b, h, w, 3), np.float32))
  return model


@pytest.fixture(scope='module')
def fresh():
  """fresh(net, mode, seed): a freshly built, warmed engine, shared by the tests of this module
  and only ever run synchronously."""
  cache = {}

  def get(net, mode, seed, device):
    key = (net, mode, seed)
    if key not in cache:
      cache[key] = engine(net, mode, seed, device)
    return cache[key]
  yield get
  cache.clear()


class Hold:
  """A bounded spin queued on `stream`: what is enqueued behind it stays in flight until the spin
  ends, about 0.5 s later."""

  def __init__(self, stream, device):
    s = torch.cuda.ExternalStream(stream, device=device)
    with torch.cuda.stream(s):
      torch.cuda._sleep(SPIN_CYCLES)
    self.done = torch.cuda.Event()
    self.done.record(s)

  def assert_active(self, after):
    assert not self.done.query(), (
        'the stream hold had ended when %s returned: the run did not race queued work, so it '
        'tested nothing' % after)


def records(dets, counts):
  """Each image's filtered records up to its count, and the counts, as one bytes value."""
  counts = np.asarray(counts)
  cap = dets.shape[1]
  return counts.tobytes() + b''.join(dets[i][:min(max(int(c), 0), cap)].tobytes()
                                     for i, c in enumerate(counts))


def pinned_records(model, n):
  return (_lib.PinnedArray((n, model.max_dets), _lib.DET_DTYPE),
          _lib.PinnedArray((n,), np.int32))


class Results:
  """Pinned host copies of rows [0, n) of every result buffer of a forward."""

  def __init__(self, model, n=None):
    B, A = model.det_probs.shape
    self.n = n or B
    self.bufs = {'det_boxes': _lib.PinnedArray((self.n, A, 4), np.float32),
                 'det_probs': _lib.PinnedArray((self.n, A), np.float32),
                 'det_class': _lib.PinnedArray((self.n, A), np.int64),
                 'dets': _lib.PinnedArray((self.n, model.max_dets), _lib.DET_DTYPE),
                 'counts': _lib.PinnedArray((self.n,), np.int32)}

  def copy(self, model, stream):
    """Enqueue the copies on `stream` (asynchronous: the buffers are pinned)."""
    dev = model.results_device()
    for key, p in self.bufs.items():
      _lib.check(model._lib.sqdet_memcpy_d2h(p.ptr, dev[key], p.array.nbytes, stream))

  def value(self):
    a = {k: p.array for k, p in self.bufs.items()}
    return (records(a['dets'], a['counts']) + a['det_boxes'].tobytes() +
            a['det_probs'].tobytes() + a['det_class'].tobytes())


def legacy_forward(model, images_dev, n=None):
  """The synchronous result: a forward on the legacy stream (never graph-captured)."""
  r = Results(model, n)
  model.forward_device(images_dev.ptr, None, n)
  r.copy(model, None)
  sync(model, None)
  return r.value()


def pinned(arr):
  p = _lib.PinnedArray(arr.shape, arr.dtype)
  p.array[...] = arr
  return p


def assert_same(got, want, other, what):
  """`got` equals `want`; on a mismatch, say whether it equals the other weights' result."""
  if got == want:
    return
  if got == other:
    pytest.fail('%s: its result is that of the weights loaded after it was enqueued' % what)
  pytest.fail('%s: its result differs from the synchronous run' % what)


# ---- the paths a reload can race: two submissions each, 0 before and 1 after the reload --------
# Every buffer a submission needs is allocated, and every graph captured, before the stream is
# held: a cudaFree or a pinned free inside the window would synchronise the device.
class Submit:
  """sqdet_submit of fp32 or uint8 images from pinned memory, records back to pinned memory."""

  def __init__(self, model, device, u8):
    B, H, W = model.mc.BATCH_SIZE, model.mc.IMAGE_HEIGHT, model.mc.IMAGE_WIDTH
    rng = np.random.default_rng(40)
    self.model, self.stream, self.u8 = model, model.engine_stream(), u8
    self.images = [pinned(rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8) if u8
                          else synth.synthetic_images(B, H, W, seed=41 + i)) for i in range(2)]
    self.out = [pinned_records(model, B) for _ in range(2)]

  def enqueue(self, i):
    d, c = self.out[i]
    self.model.submit(self.images[i].ptr, d.ptr, c.ptr, _lib.IMG_U8 if self.u8 else _lib.IMG_F32)

  def finish(self):
    self.model.wait()
    self.model.wait()

  def result(self, i):
    return records(self.out[i][0].array, self.out[i][1].array)

  def reference(self, eng, i):
    x = self.images[i].array
    return records(*(eng.detect_u8(x) if self.u8 else eng.detect_records(x)))


class SubmitFrames(Submit):
  """sqdet_submit_frames_n of B - 1 pinned frames of other sizes.  Only the second submission
  rescales: the scale table goes up as a pageable copy on the engine stream, and such a copy may
  block until a held stream reaches it."""

  def __init__(self, model, device):
    B, H, W = model.mc.BATCH_SIZE, model.mc.IMAGE_HEIGHT, model.mc.IMAGE_WIDTH
    rng = np.random.default_rng(45)
    sizes = [(H + 17, W - 24), (H - 9, W + 40), (H + 3, W + 5)]
    self.model, self.stream, self.n = model, model.engine_stream(), B - 1
    self.frames = [[pinned(rng.integers(0, 256, sizes[(i + j) % 3] + (3,), dtype=np.uint8))
                    for j in range(self.n)] for i in range(2)]
    self.out = [pinned_records(model, self.n) for _ in range(2)]

  def enqueue(self, i):
    d, c = self.out[i]
    self.model.submit_frames([f.array for f in self.frames[i]], d.ptr, c.ptr, 'eval',
                             rescale=i == 1)

  def reference(self, eng, i):
    return records(*eng.detect_frames([f.array for f in self.frames[i]], 'eval', rescale=i == 1))


class ForwardDevice:
  """forward_device on `stream` (a caller's, by default), every result copied to pinned memory on
  that stream behind it."""

  def __init__(self, model, device, stream=None):
    B, H, W = model.mc.BATCH_SIZE, model.mc.IMAGE_HEIGHT, model.mc.IMAGE_WIDTH
    self.caller = torch.cuda.Stream(device=device)
    self.model, self.stream = model, stream or self.caller.cuda_stream
    self.images = [_lib.DeviceBuffer.from_numpy(synth.synthetic_images(B, H, W, seed=51 + i), device)
                   for i in range(2)]
    self.out = [Results(model) for _ in range(2)]

  def enqueue(self, i):
    self.model.forward_device(self.images[i].ptr, self.stream)
    self.out[i].copy(self.model, self.stream)

  def finish(self):
    sync(self.model, self.stream)

  def result(self, i):
    return self.out[i].value()

  def reference(self, eng, i):
    return legacy_forward(eng, self.images[i])


PATHS = {
    'submit_f32': lambda m, d: Submit(m, d, u8=False),
    'submit_u8': lambda m, d: Submit(m, d, u8=True),
    'submit_frames_n': SubmitFrames,
    'forward_device': ForwardDevice,
}


@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('math_mode', MODES)
@pytest.mark.parametrize('net', list(SIZES))
def test_reload_with_forwards_in_flight(net, math_mode, path, fresh, gpu_device):
  """Hold the path's stream, then: enqueue A with W1, load W2, enqueue B, wait for both.  A must
  give what a W1 engine gives, B what a W2 engine gives: the forward after a reload waits for A
  before overwriting the weights, and its own kernels read the uploaded ones."""
  model = engine(net, math_mode, W1, gpu_device)
  if net == 'squeezeDet' and math_mode == _lib.MATH_TF32X3_TC:
    h, w, b = SIZES[net]
    pool1 = {r[0]: r[2] for r in oracle.layer_table(net, h, w)}['pool1']
    assert fire_tiles(b, pool1[0], pool1[1]) >= 4 * 132
    assert_fused_away(model, 'fire2/squeeze1x1')
    assert_fused_away(model, 'fire3/squeeze1x1')
  run = PATHS[path](model, gpu_device)
  for i in (0, 1):                 # both submissions once: graphs captured, buffers sized
    run.enqueue(i)
  run.finish()
  w2 = weights(net, W2)            # outside the hold: ResNet-50's table takes over 0.2 s to make
  hold = Hold(run.stream, gpu_device)
  run.enqueue(0)
  model.load_weights(w2)
  hold.assert_active('the reload')
  run.enqueue(1)
  run.finish()
  want = {s: [run.reference(fresh(net, math_mode, s, gpu_device), i) for i in (0, 1)]
          for s in (W1, W2)}
  assert want[W1][0] != want[W2][0] and want[W1][1] != want[W2][1], 'W1 and W2 give one result'
  assert_same(run.result(0), want[W1][0], want[W2][0], 'the forward enqueued before the reload')
  assert_same(run.result(1), want[W2][1], want[W1][1], 'the forward enqueued after the reload')


@pytest.mark.parametrize('math_mode', MODES)
@pytest.mark.parametrize('net', list(SIZES))
def test_reload_between_graph_replays(net, math_mode, fresh, gpu_device):
  """Nothing in flight: a forward on the engine stream captures its graph, the weights change,
  and the next forward of the same key replays that graph with the new weights, BN scale/shift
  and tensor-core packs included."""
  model = engine(net, math_mode, W1, gpu_device)
  run = ForwardDevice(model, gpu_device, model.engine_stream())
  got = []
  for seed in (W1, W2):
    if seed == W2:
      model.load_weights(weights(net, W2))
    run.enqueue(0)
    run.finish()
    got.append(run.result(0))
  for seed, g in zip((W1, W2), got):
    assert g == run.reference(fresh(net, math_mode, seed, gpu_device), 0), seed
  assert got[0] != got[1]


def test_graph_cache_keys(gpu_device):
  """24 keys (3 inputs, n in {B, 1}, the engine stream and a caller's, the box-scale table set or
  not) through the 4-entry cache, twice, in scrambled orders: each forward equals the legacy-stream
  forward of its input.  Then five new keys on a held stream: the fifth capture evicts the graph of
  the first, whose launch is still queued, and all five still give the synchronous results."""
  h, w, b = 112, 208, 3
  model = engine('squeezeDet', _lib.MATH_TF32X3_TC, W1, gpu_device, size=(h, w, b))
  table = np.array([[1.25, 0.8], [0.5, 2.0], [1.0, 1.5]], np.float32)
  inputs = [_lib.DeviceBuffer.from_numpy(synth.synthetic_images(b, h, w, seed=60 + i), gpu_device)
            for i in range(3)]
  caller, held = torch.cuda.Stream(device=gpu_device), torch.cuda.Stream(device=gpu_device)
  streams = {'engine': model.engine_stream(), 'caller': caller.cuda_stream}
  assert len({*streams.values(), held.cuda_stream}) == 3

  want = {}
  for scaled in (False, True):
    model.set_box_scale(table if scaled else None)
    for i in range(3):
      for n in (b, 1):
        want[i, n, scaled] = legacy_forward(model, inputs[i], n)
  assert len(set(want.values())) == len(want)

  res = {n: Results(model, n) for n in (b, 1)}
  keys = [(i, n, s, scaled) for i in range(3) for n in (b, 1) for s in streams
          for scaled in (False, True)]
  rng = np.random.default_rng(5)
  scaled_now = True
  for rnd in range(2):
    for k in rng.permutation(len(keys)):
      i, n, s, scaled = keys[k]
      if scaled != scaled_now:
        model.set_box_scale(table if scaled else None)
        scaled_now = scaled
      r = res[n]
      model.forward_device(inputs[i].ptr, streams[s], n)
      r.copy(model, streams[s])
      sync(model, streams[s])
      assert r.value() == want[i, n, scaled], (rnd, keys[k])

  five = [(i, n) for i in range(3) for n in (b, 1)][:5]
  outs = [Results(model, n) for _, n in five]
  hold = Hold(held.cuda_stream, gpu_device)
  for (i, n), r in zip(five, outs):
    model.forward_device(inputs[i].ptr, held.cuda_stream, n)
    r.copy(model, held.cuda_stream)
  hold.assert_active('five forwards on new keys')
  sync(model, held.cuda_stream)
  for (i, n), r in zip(five, outs):
    assert r.value() == want[i, n, scaled_now], (i, n)


def test_waits_cover_only_the_engines_own_work(gpu_device):
  """A reload, read_tensor and set_box_scale wait for the engine's own forwards, not for the
  device: synchronising the device is invalid while another thread captures a graph, and would
  invalidate that capture.  With a stream the engine never uses held, a reload, a forward,
  read_tensor and set_box_scale all return, and the forward gives the new weights' result."""
  h, w, b = 112, 208, 2
  table = np.linspace(0.7, 1.6, 2 * b).astype(np.float32)
  model = engine('squeezeDet', _lib.MATH_TF32X3_TC, W1, gpu_device, (h, w, b), table)
  x = _lib.DeviceBuffer.from_numpy(synth.synthetic_images(b, h, w, seed=65), gpu_device)
  r = Results(model)
  foreign = torch.cuda.Stream(device=gpu_device)
  stream = model.engine_stream()
  assert foreign.cuda_stream != stream
  w2 = weights('squeezeDet', W2)
  hold = Hold(foreign.cuda_stream, gpu_device)
  model.load_weights(w2)
  model.forward_device(x.ptr, stream)
  r.copy(model, stream)
  sync(model, stream)
  preds = model.read_tensor(model.preds)
  model.set_box_scale(table)
  assert not hold.done.query(), 'the engine waited for work on a stream it never used'
  ref = engine('squeezeDet', _lib.MATH_TF32X3_TC, W2, gpu_device, (h, w, b), table)
  assert r.value() == legacy_forward(ref, x)
  assert preds.tobytes() == ref.read_tensor(ref.preds).tobytes()


# ---- two engines, two host threads -------------------------------------------------------------
ITERS = 10
THREAD_NETS = [('squeezeDet', _lib.MATH_TF32X3_TC, (112, 208, 2)),
               ('resnet50', _lib.MATH_FP32_SIMT, (99, 131, 2))]


class Worker:
  """One thread's loop over detect, pipelined submit_frames_n, forward_device on its own stream
  and read_tensor, re-setting the box-scale table each time; its input buffers and keys."""

  def __init__(self, net, mode, size, device):
    h, w, b = size
    self.net, self.mode, self.size, self.b = net, mode, size, b
    self.table = np.linspace(0.6, 1.7, 2 * b).astype(np.float32)
    self.images = [synth.synthetic_images(b, h, w, seed=70 + i) for i in range(3)]
    self.inputs = [_lib.DeviceBuffer.from_numpy(x, device) for x in self.images]
    rng = np.random.default_rng(75)
    self.frames = [[pinned(rng.integers(0, 256, (h + 11 * j + 5, w - 7 * k + 9, 3), dtype=np.uint8))
                    for j in range(n)] for k, n in enumerate((b, 1))]
    self.stream = torch.cuda.Stream(device=device)
    self.out = self.results = None

  def step(self, model, it):
    """Iteration `it`: its results as bytes values.  The forward_device key cycles through six
    (input, n) pairs, so with the engine stream's keys the cache recaptures every iteration."""
    i, n = it % 3, (self.b if it % 2 == 0 else 1)
    if self.out is None:            # the first step runs on a reference engine, before the threads
      self.out = [pinned_records(model, self.b) for _ in range(2)]
      self.results = {m: Results(model, m) for m in (self.b, 1)}
    boxes, probs, cls, dets, counts = model.detect(self.images[i], want_dets=True)
    got = [boxes.tobytes() + probs.tobytes() + cls.tobytes() + records(dets, counts)]
    for k, frames in enumerate(self.frames):
      d, c = self.out[k]
      model.submit_frames([f.array for f in frames], d.ptr, c.ptr, 'eval', rescale=k == 1)
    for k, frames in enumerate(self.frames):
      model.wait()
      d, c = self.out[k]
      got.append(records(d.array[:len(frames)], c.array[:len(frames)]))
    r = self.results[n]
    s = self.stream.cuda_stream
    model.forward_device(self.inputs[i].ptr, s, n)
    r.copy(model, s)
    sync(model, s)
    got.append(r.value())
    got.append(model.read_tensor(model.preds)[:n].tobytes())
    model.set_box_scale(self.table)
    return got


def test_two_engines_two_threads(gpu_device):
  """Two engines with different nets, sizes and math modes, each driven by its own host thread
  (ctypes releases the GIL, so the threads overlap): one thread captures graphs in thread-local
  mode while the other waits for its own forwards in read_tensor, set_box_scale and, halfway, its
  weight reload, and copies on the legacy stream.  Every result equals that engine's
  single-threaded run."""
  workers = [Worker(net, mode, size, gpu_device) for net, mode, size in THREAD_NETS]
  want = []
  for wk in workers:
    refs = [engine(wk.net, wk.mode, s, gpu_device, wk.size, wk.table) for s in (W1, W2)]
    want.append([wk.step(refs[it >= ITERS // 2], it) for it in range(ITERS)])
  models = [engine(wk.net, wk.mode, W1, gpu_device, wk.size, wk.table) for wk in workers]
  got = [[] for _ in workers]
  errors = []
  barrier = threading.Barrier(len(workers), timeout=60)

  def loop(k):
    try:
      wk, model = workers[k], models[k]
      barrier.wait()
      for it in range(ITERS):
        if it == ITERS // 2:
          model.load_weights(weights(wk.net, W2))
        got[k].append(wk.step(model, it))
    except BaseException as exc:      # re-raised in the main thread
      errors.append(exc)

  threads = [threading.Thread(target=loop, args=(k,), daemon=True) for k in range(len(workers))]
  for t in threads:
    t.start()
  for t in threads:
    t.join(timeout=120)
  assert not any(t.is_alive() for t in threads), 'a worker thread did not finish in 120 s'
  if errors:
    raise errors[0]
  names = ['detect', 'submit_frames_n (B)', 'submit_frames_n (1, rescaled)', 'forward_device',
           'read_tensor']
  for wk, g, w in zip(workers, got, want):
    assert len(g) == ITERS
    for it in range(ITERS):
      for name, a, b in zip(names, g[it], w[it]):
        assert a == b, (wk.net, it, name)
