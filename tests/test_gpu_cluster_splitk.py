"""The K split of the ConvDet head (conv_tc.cu, 72-wide halo-mode tile): a cluster of S CTAs shares
one output tile, each rank sums a contiguous range of the conv's 32-channel chunks, and the ranks
add their partial tiles in rank order through distributed shared memory.  The engine chooses S
from its batch and the device's resident clusters; sqdet_conv2d_k_split forces it.  Each element
is checked against the fp64 oracle with the bar gpu_util.adv_tol, repeat runs bitwise, and
forwards of fewer images than the engine's batch bitwise against the full batch's rows."""
import numpy as np
import pytest

from squeezedet_b200 import _lib
from squeezedet_b200.utils import synth
from gpu_util import (assert_rows_equal, assert_within_bound, conv_oracle, fetch_results,
                      forward_n, make_net)

pytestmark = pytest.mark.gpu
TC = _lib.MATH_TF32X3_TC


def conv_k_split(x, w, b, k_split, relu=False, scale=None, shift=None, y_cstride=None, y_coff=0,
                 device=0):
  """sqdet_conv2d_k_split of a stride-1 SAME 3x3 conv on host arrays; channels outside the
  window keep the value 7."""
  lib = _lib.load()
  B, H, W, Cin = x.shape
  Cout = w.shape[3]
  cs = y_cstride or Cout
  bufs = [_lib.DeviceBuffer.from_numpy(np.ascontiguousarray(a, np.float32), device)
          if a is not None else None for a in (x, w, b, scale, shift)]
  dy = _lib.DeviceBuffer.from_numpy(np.full((B, H, W, cs), 7.0, np.float32), device)
  ptr = [bf.ptr if bf else None for bf in bufs]
  _lib.check(lib.sqdet_conv2d_k_split(ptr[0], ptr[1], ptr[2], ptr[3], ptr[4], dy.ptr, B, H, W, Cin,
                                      Cout, 3, 1, _lib.PAD_SAME, int(relu), cs, y_coff, TC,
                                      k_split, None))
  _lib.check(lib.sqdet_stream_sync(device, None))
  return dy.to_numpy(np.float32, (B, H, W, cs))


CASES = [
    # B, H, W, Cin, Cout, y_cstride, y_coff
    (1, 24, 78, 768, 72, 72, 0),    # the SqueezeDet head's grid and K: 24 channel chunks
    (2, 13, 37, 224, 66, 80, 7),    # 7 chunks (divides by no S), Cout < 72, a channel window
]


@pytest.mark.parametrize('k_split', [2, 3, 4])
@pytest.mark.parametrize('case', CASES)
def test_forced_k_split_vs_oracle(case, k_split, gpu_device):
  B, H, W, Cin, Cout, cs, coff = case
  rng = np.random.default_rng(sum(case) + k_split)
  x = rng.normal(size=(B, H, W, Cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, Cin, Cout)) / np.sqrt(9 * Cin)).astype(np.float32)
  b = rng.normal(size=Cout).astype(np.float32)
  affine = cs != Cout
  sc = rng.uniform(0.5, 1.5, Cout).astype(np.float32) if affine else None
  sh = rng.normal(size=Cout).astype(np.float32) if affine else None
  want, bound = conv_oracle(x, w, b, scale=sc, shift=sh)
  got = conv_k_split(x, w, b, k_split, scale=sc, shift=sh, y_cstride=cs, y_coff=coff,
                     device=gpu_device)
  win = got[..., coff:coff + Cout]
  assert not np.isnan(win).any()
  assert_within_bound(win, want, bound, 9 * Cin, (case, k_split))
  assert np.all(got[..., :coff] == 7.0) and np.all(got[..., coff + Cout:] == 7.0)
  again = conv_k_split(x, w, b, k_split, scale=sc, shift=sh, y_cstride=cs, y_coff=coff,
                       device=gpu_device)
  assert got.tobytes() == again.tobytes()
  # an image's tiles do not depend on the batch around it
  first = conv_k_split(x[:1], w, b, k_split, scale=sc, shift=sh, y_cstride=cs, y_coff=coff,
                       device=gpu_device)
  assert first.tobytes() == got[:1].tobytes()


def test_k_split_rejected_where_not_planned(gpu_device):
  """A K split needs the 72-wide tile and at least one channel chunk per rank."""
  rng = np.random.default_rng(0)
  x = rng.normal(size=(1, 8, 16, 64)).astype(np.float32)
  for cout, k_split in ((64, 2), (72, 3), (72, 5)):   # 64 wide; 2 chunks < 3 ranks; S > 4
    w = rng.normal(size=(3, 3, 64, cout)).astype(np.float32)
    with pytest.raises(_lib.SqdetError) as exc:
      conv_k_split(x, w, None, k_split, device=gpu_device)
    assert exc.value.code == -1, (cout, k_split)


def forward(model, images, n, device):
  """The head's output and the det tensors of a forward of the first n images."""
  forward_n(model, images, n)
  res = fetch_results(model, device)
  return {'preds': model.read_tensor(model.preds),
          **{key: res[key] for key in ('det_probs', 'det_boxes', 'det_class')}}


def test_squeezedet_head_splits_at_the_benchmark_size(gpu_device):
  """SqueezeDet at 1242 x 375, b = 20: 300 head tiles on 2 x 132 CTA slots leave most of a second
  wave idle, so the plan splits the head's K.  Two forwards are bitwise equal, and a forward
  of 7 images gives bitwise the first 7 rows of the full batch."""
  B, H, W = 20, 375, 1242
  model, _ = make_net('squeezeDet', W, H, B, gpu_device, seed=5)
  splits = model.op_k_splits()
  assert list(splits) == ['conv12'] and splits['conv12'] > 1, splits
  images = synth.synthetic_images(B, H, W, seed=2)
  full = forward(model, images, B, gpu_device)
  assert_rows_equal(forward(model, images, B, gpu_device), full, B)
  assert_rows_equal(forward(model, images, 7, gpu_device), full, 7)


@pytest.mark.parametrize('net', ['resnet50', 'vgg16'])
def test_only_the_head_splits(net, gpu_device):
  """At b = 8 the 120 head tiles fill fewer than half of the two CTA slots per SM, so the plan
  splits the head's K; no other op of the net is planned with a split."""
  model, _ = make_net(net, 1242, 375, 8, gpu_device, seed=5)
  splits = model.op_k_splits()
  head = model.op_table()[-3][0]          # the last plan op, before interpret and filter
  assert list(splits) == [head] and 1 < splits[head] <= 4, splits


def test_split_head_rows_follow_full_batch(gpu_device):
  """A small grid (2 head tiles an image) splits the head four ways; forwards of n = 1, 2 of the
  3 images, and a repeat of the full batch, give bitwise the full forward's rows."""
  B, H, W = 3, 96, 320
  model, _ = make_net('squeezeDet', W, H, B, gpu_device, seed=8)
  assert model.op_k_splits().get('conv12', 1) > 1
  images = synth.synthetic_images(B, H, W, seed=4)
  full = forward(model, images, B, gpu_device)
  for n in (1, 2, 3):
    assert_rows_equal(forward(model, images, n, gpu_device), full, n)
