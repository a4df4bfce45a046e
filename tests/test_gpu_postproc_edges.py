"""interpret_output and the top-N / NMS filter at their numerical edges, each against a plain
reference, through the C ABI.

interpret_kernel (csrc/postproc.cu) restates oracle.interpret_output operation for operation in
fp32, with no contracted FMA:
  * with every dw and dh above EXP_THRESH no exp enters the box chain, so det_boxes equal the fp32
    oracle's bit for bit;
  * everywhere else scores and boxes stay within a per-element bound derived from the operation
    chain (check_interpret_bounds) of an fp64 evaluation of the same chain;
  * an edge table: the EXP_THRESH boundary, exp underflow, logits that overflow expf without the
    max subtraction, exact class ties, a saturated sigmoid, boxes decoded outside the image, and a
    one-pixel-wide image.
filter_kernel (sqdet_topk_nms) equals oracle.filter_prediction bit for bit on signed zeros, NaN
of either sign, +-inf, subnormals, scores at PROB_THRESH and IoUs at NMS_THRESH, zero-area and
identical boxes, top_n in {A, A + 1}, and a batch where only some images overflow the threshold
branch.  The rank order is probability descending, -0.0 == +0.0, NaN last, ties by ascending
anchor (oracle.postproc._rank_order); test_order_key_ranks_as_oracle checks the kernel's sort key
against it without a GPU.

Not pinned here: non-finite values inside interpret_kernel (NaN logits or deltas, where fmaxf
drops a NaN that numpy propagates).  No fixture pins the reference's TensorFlow semantics there.
"""
import numpy as np
import pytest

import oracle
from gpu_util import assert_classes_match, interpret_gpu, topk_nms_gpu

gpu = pytest.mark.gpu
U = 2.0 ** -24                       # float32 unit roundoff
FLT_MIN = 2.0 ** -126                # smallest normal float32
SHAPES = oracle.postproc.ANCHOR_SHAPES_SQUEEZE
F32 = np.float32


# ---- interpret_output ---------------------------------------------------------------------------
def interpret_f64(preds, anchors, K, C, W, H, t):
  """interpret_output's chain in fp64 from the fp32 preds -> (scores [B,A], boxes [B,A,4],
  M [B,A,4]).  Two intermediates stay fp32 because the kernel and the fp32 oracle form each with
  the same IEEE operations, and one rounding there can cost far more than an ulp of the result:
  the max-subtracted logits z = lg - max(lg) (an exp of z scales the rounding by |z|) and the
  centres cx = ax + dx * aw (ax + dx * aw may cancel).  M is the pre-clip magnitude
  max(|c|, b / 2) of each output's axis, which sets its bound."""
  p = np.asarray(preds, F32)
  B = p.shape[0]
  A = p.shape[1] * p.shape[2] * K
  an = np.asarray(anchors, np.float64).astype(F32)
  lg = p[..., :K * C].reshape(B, A, C)
  e = np.exp((lg - lg.max(axis=2, keepdims=True)).astype(np.float64))
  x = p[..., K * C:K * C + K].reshape(B, A).astype(np.float64)
  with np.errstate(over='ignore'):
    conf = 1.0 / (1.0 + np.exp(-x))
  scores = (e / e.sum(axis=2, keepdims=True) * conf[..., None]).max(axis=2)
  d = p[..., K * C + K:].reshape(B, A, 4)
  cx = (an[:, 0] + d[..., 0] * an[:, 2]).astype(np.float64)
  cy = (an[:, 1] + d[..., 1] * an[:, 3]).astype(np.float64)

  def safe_exp(w):
    w64 = w.astype(np.float64)
    with np.errstate(over='ignore'):
      return np.where(w > F32(t), np.exp(t) * (w64 - t + 1.0), np.exp(np.minimum(w64, t)))

  def axis(c, size, m1):
    lo = np.minimum(np.maximum(0.0, c - size / 2), m1)
    hi = np.maximum(np.minimum(m1, c + size / 2), 0.0)
    s = hi - lo + 1.0
    return lo + 0.5 * s, s, np.maximum(np.abs(c), size / 2)

  ox, ow, mx = axis(cx, an[:, 2] * safe_exp(d[..., 2]), W - 1.0)
  oy, oh, my = axis(cy, an[:, 3] * safe_exp(d[..., 3]), H - 1.0)
  return scores, np.stack([ox, oy, ow, oh], -1), np.stack([mx, my, mx, my], -1)


def assert_within(got, want, tol, what):
  err = np.abs(np.asarray(got, np.float64) - want)
  bad = ~(err <= tol)
  if bad.any():
    i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(tol, 1e-300), -1)), err.shape)
    raise AssertionError('%s: %d elements out of bound; worst at %s: got %r want %r bound %r'
                         % (what, int(bad.sum()), i, float(np.asarray(got)[i]), float(want[i]),
                            float(tol[i])))


def check_interpret_bounds(got, preds, anchors, K, C, W, H, t):
  """Scores and boxes of the kernel against interpret_f64, per element (u = 2^-24; first order):

  score = (e_c / sum_c e_c) * conf with e_c = expf(z_c) and conf = 1 / (1 + expf(-x)).  CUDA's
  expf is within 2 ulp (4u relative); every other operation rounds once (u).  e_c: 4u; the sum of
  C positive terms: 4u + (C - 1)u; the quotient: (C + 8)u; conf: 4u + u + u = 6u; the product:
  (C + 15)u.  Below FLT_MIN results carry absolute error, and for x < -88.7 expf(-x) overflows so
  conf is 0 where the exact value is below 2^-127: 2 * FLT_MIN absolute covers both.

  box, per axis, M = max(|c|, b / 2) with c the shared fp32 centre: b = a * expf(w) or
  a * slope * (w - t + 1) carries 5u relative, so b / 2 carries 5uM; lo = c - b / 2 rounds once
  on a value below 2M: 7uM, clipping does not grow it; hi - lo: 16uM; + 1: 18uM + u (the width);
  lo + width / 2 rounds once on a value below 3M + 1: 19uM + 2u (the centre).  Bound: 20u(M + 1),
  ~10-20 ulp of M."""
  gb, gp, gc = got
  rp, rb, M = interpret_f64(preds, anchors, K, C, W, H, t)
  assert_within(gp, rp, (C + 15) * U * np.abs(rp) + 2 * FLT_MIN, 'scores')
  assert_within(gb, rb, 20 * U * (M + 1), 'boxes')


def deltas(preds, K, C):
  """preds' (dx, dy, dw, dh) as a writable view [..., K, 4]."""
  d = preds[..., K * C + K:].reshape(preds.shape[:-1] + (K, 4))
  assert np.shares_memory(d, preds)
  return d


def run_interpret(preds, anchors, K, C, W, H, t):
  got = interpret_gpu(preds, anchors, K, C, W, H, t)
  with np.errstate(over='ignore', under='ignore'):
    want = oracle.interpret_output(preds, anchors, C, K, W, H, t)
  return got, want


@gpu
@pytest.mark.parametrize('W,H', [(1242, 375), (4001, 1207)])
@pytest.mark.parametrize('K', [9, 1])
@pytest.mark.parametrize('C', [1, 3, 20])
def test_exp_free_box_decode_bit_exact(C, K, W, H, gpu_device):
  """Every dw and dh above EXP_THRESH: safe_exp is slope * (w - t + 1) with slope cast from
  float64, so the box chain has no exp and det_boxes equal the fp32 oracle's bit for bit.  A
  contracted FMA in cx = ax + dx * aw, or any reordering, shows here."""
  B, gh, gw, t = 2, 7, 11, 1.0
  rng = np.random.default_rng(C * 100 + K + W)
  preds = (rng.normal(size=(B, gh, gw, K * (C + 5))) * 1.5).astype(F32)
  dwh = deltas(preds, K, C)[..., 2:]
  dwh[...] = np.maximum(F32(t) + rng.uniform(0, 3, dwh.shape).astype(F32),
                        np.nextafter(F32(t), F32(np.inf)))
  anchors = oracle.set_anchors(W, H, gh, gw, SHAPES[:K])
  got, want = run_interpret(preds, anchors, K, C, W, H, t)
  assert got[0].tobytes() == want[0].tobytes()
  check_interpret_bounds(got, preds, anchors, K, C, W, H, t)
  assert_classes_match(got[2], want[2], preds.astype(np.float64), K, C, (C + 15) * U)


@gpu
@pytest.mark.parametrize('classes,K,gh,gw', [(3, 9, 24, 78), (20, 9, 5, 7), (3, 9, 22, 76),
                                             (3, 1, 24, 78), (3, 5, 13, 41), (1, 9, 11, 37)])
def test_interpret_within_derived_bound(classes, K, gh, gw, gpu_device):
  """Random preds with exp in the chain: scores and boxes within check_interpret_bounds."""
  rng = np.random.default_rng(classes * 7 + K)
  B, W, H, t = 2, 1242, 375, 1.0
  preds = (rng.normal(size=(B, gh, gw, K * (classes + 5))) * 1.5).astype(F32)
  preds[0, 0, 0, K * classes + K + 2] = 3.0         # dw above EXP_THRESH: the linear tail
  preds[0, 0, 1, K * classes + K + 3] = -40.0
  anchors = oracle.set_anchors(W, H, gh, gw, SHAPES[:K])
  got, want = run_interpret(preds, anchors, K, classes, W, H, t)
  check_interpret_bounds(got, preds, anchors, K, classes, W, H, t)
  assert_classes_match(got[2], want[2], preds.astype(np.float64), K, classes,
                       (classes + 15) * U)


# An edge-table row: class logits (C = 3), confidence logit, deltas (dx, dy, dw, dh), and what the
# row asserts beyond the bounds: the class id, a box bit-equal to the fp32 oracle's, box values
# that must come out exactly (None: not pinned), a score of exactly +0.
BASE = dict(logits=(0.25, -0.5, 1.0), conf=0.3, d=(0.1, -0.2, 0.3, -0.4), cls=2, box_oracle=False,
            box=None, score_zero=False)


def row(name, **kw):
  r = dict(BASE, name=name, **kw)
  if 'd' in kw:
    r['d'] = tuple(BASE['d'][i] if v is None else v for i, v in enumerate(kw['d']))
  return r


def edge_rows(t, W, H):
  below, above = (float(np.nextafter(F32(t), F32(s))) for s in (-np.inf, np.inf))
  wm1, hm1 = W - 1.0, H - 1.0
  return [
      row('dw, dh at EXP_THRESH', d=(None, None, t, t)),
      row('dw, dh one ulp below EXP_THRESH', d=(None, None, below, below)),
      row('dw, dh one ulp above EXP_THRESH', d=(None, None, above, above), box_oracle=True),
      row('dw, dh = +50', d=(None, None, 50.0, 50.0), box_oracle=True),
      # exp(-100) underflows: the box has no extent, so the clipped width and height are 1
      row('dw, dh = -100', d=(None, None, -100.0, -100.0), box_oracle=True,
          box=(None, None, 1.0, 1.0)),
      row('box covering the image', d=(None, None, 1e3, 1e3), box=(W / 2, H / 2, W, H)),
      row('centre far left', d=(-1e3, None, None, None), box=(0.5, None, 1.0, None)),
      row('centre far right', d=(1e3, None, None, None), box=(wm1 + 0.5, None, 1.0, None)),
      row('centre far above', d=(None, -1e3, None, None), box=(None, 0.5, None, 1.0)),
      row('centre far below', d=(None, 1e3, None, None), box=(None, hm1 + 0.5, None, 1.0)),
      # without the max subtraction the sum of three exp(88) overflows, and exp(1e4) is inf
      row('class logits all +88', logits=(88.0, 88.0, 88.0), cls=0),
      row('class logits all -88', logits=(-88.0, -88.0, -88.0), cls=0),
      row('class logits -88, +88, -88', logits=(-88.0, 88.0, -88.0), cls=1),
      row('class logits -1e4, +1e4, -1e4', logits=(-1e4, 1e4, -1e4), cls=1),
      # exact ties: the first maximum wins (tf.argmax)
      row('all classes tied', logits=(0.7, 0.7, 0.7), cls=0),
      row('classes 1 and 2 tied', logits=(0.1, 2.0, 2.0), cls=1),
      # expf(100) overflows: conf = 0, every class scores +0 and class 0 wins the tie
      row('confidence logit -100', conf=-100.0, cls=0, score_zero=True),
      row('confidence logit +100', conf=100.0),
  ]


def put(preds, b, a, K, C, r):
  cell, k = divmod(a, K)
  v = preds[b, cell // preds.shape[2], cell % preds.shape[2]]
  v[k * C:(k + 1) * C] = r['logits']
  v[K * C + k] = r['conf']
  v[K * C + K + 4 * k:K * C + K + 4 * k + 4] = r['d']


@gpu
@pytest.mark.parametrize('W,H', [(1242, 375), (4001, 1207)])
@pytest.mark.parametrize('t', [0.5, 1.0, 2.0])
def test_interpret_edge_table(t, W, H, gpu_device):
  """Each row of edge_rows at one anchor (image 0 in table order, image 1 reversed), every other
  anchor the base row: the bounds hold everywhere, the class id equals the fp32 oracle's at every
  anchor (each row's top-2 margin is exactly 0 or far above fp noise), and each row's own
  assertion holds."""
  B, K, C = 2, 9, 3
  rows = edge_rows(t, W, H)
  gw = -(-len(rows) // K) + 1
  A = gw * K
  preds = np.zeros((B, 1, gw, K * (C + 5)), F32)
  for b in range(B):
    for a in range(A):
      put(preds, b, a, K, C, BASE)
  at = [list(range(len(rows))), [A - 1 - i for i in range(len(rows))]]
  for b in range(B):
    for i, r in enumerate(rows):
      put(preds, b, at[b][i], K, C, r)
  anchors = oracle.set_anchors(W, H, 1, gw, SHAPES)
  got, want = run_interpret(preds, anchors, K, C, W, H, t)
  gb, gp, gc = got
  check_interpret_bounds(got, preds, anchors, K, C, W, H, t)
  assert gc.dtype == np.int64
  assert np.array_equal(gc, want[2])
  for b in range(B):
    for i, r in enumerate(rows):
      a = at[b][i]
      assert gc[b, a] == r['cls'], (r['name'], b, gc[b, a])
      if r['box_oracle']:
        assert gb[b, a].tobytes() == want[0][b, a].tobytes(), (r['name'], b, gb[b, a])
      if r['box'] is not None:
        for j, v in enumerate(r['box']):
          assert v is None or gb[b, a, j] == F32(v), (r['name'], b, j, gb[b, a], r['box'])
      if r['score_zero']:
        assert gp[b, a] == 0 and not np.signbit(gp[b, a]), (r['name'], b, gp[b, a])


# thresholds on a 1/16 grid (exact in float32), 1.0 and 2.0 among them
THRESH_SWEEP = [0.5 + i / 16 for i in range(56)]


@gpu
def test_exp_thresh_boundary_takes_exp_branch(gpu_device):
  """safe_exp's test is strict (w > thresh): at w == thresh it returns exp(w).  So every box
  decoded with dw = dh = t under EXP_THRESH t equals, bit for bit, the box decoded from the same
  preds under the next float32 above t, where w < thresh and only exp(w) can apply.  A '>=' would
  return slope = float32(e^t) instead, which differs from expf(t) in the last bit for some t.
  576 anchors of distinct sizes per t, each box inside the image with its low edge between 5 %
  and 150 % of its size from 0, let such a bit reach the output.  Both launches also stay within
  check_interpret_bounds."""
  B, gh, gw, K, C, W, H = 1, 8, 8, 9, 3, 65536, 65536
  rng = np.random.default_rng(9)
  A = gh * gw * K
  preds = rng.normal(size=(B, gh, gw, K * (C + 5))).astype(F32)
  deltas(preds, K, C)[..., :2] = 0
  for t in THRESH_SWEEP:
    deltas(preds, K, C)[..., 2:] = t
    size = rng.uniform(1, 400, (A, 2))
    anchors = np.concatenate([size * np.exp(t) * rng.uniform(0.55, 2, (A, 2)), size], 1)
    t_up = float(np.nextafter(F32(t), F32(np.inf)))
    at_t = interpret_gpu(preds, anchors, K, C, W, H, t)
    check_interpret_bounds(at_t, preds, anchors, K, C, W, H, t)
    above = interpret_gpu(preds, anchors, K, C, W, H, t_up)
    check_interpret_bounds(above, preds, anchors, K, C, W, H, t_up)
    assert at_t[0].tobytes() == above[0].tobytes(), t


@gpu
def test_interpret_one_pixel_wide_image(gpu_device):
  """W = 1, so W - 1 = 0: both clip bounds are 0 and every box is x = 0.5, width 1 exactly."""
  B, gh, gw, K, C, W, H, t = 2, 3, 5, 9, 3, 1, 375, 1.0
  rng = np.random.default_rng(21)
  preds = (rng.normal(size=(B, gh, gw, K * (C + 5))) * 1.5).astype(F32)
  anchors = oracle.set_anchors(W, H, gh, gw, SHAPES)
  got, want = run_interpret(preds, anchors, K, C, W, H, t)
  assert np.all(got[0][..., 0] == 0.5) and np.all(got[0][..., 2] == 1.0)
  check_interpret_bounds(got, preds, anchors, K, C, W, H, t)
  assert_classes_match(got[2], want[2], preds.astype(np.float64), K, C, 18 * U)


# ---- filter_prediction / NMS --------------------------------------------------------------------
CLASSES = 3
PROB_THRESH = float(F32(0.005))      # exact in float32, so the oracle and the kernel share it
NMS_THRESH = 0.4
NAN_NEG = -np.float32(np.nan)
NAN_PAYLOAD = np.array([0x7fc12345], np.uint32).view(F32)[0]
TINY = np.array([1], np.uint32).view(F32)[0]             # smallest subnormal
SUB_MAX = np.array([0x007fffff], np.uint32).view(F32)[0]  # largest subnormal


def check_filter_bits(dets, count, boxes, probs, cls, top_n, prob_thresh=PROB_THRESH,
                      nms_thresh=NMS_THRESH):
  """One image's records against oracle.filter_prediction, bit for bit: scores are compared as
  bit patterns, so a -0.0 or a NaN comes back as the caller gave it.  Returns the kept anchors
  (None when the threshold branch overflows, which must be reported, not truncated)."""
  max_dets = len(dets)
  with np.errstate(invalid='ignore'):
    fb, fp, fc, src = oracle.filter_prediction(boxes, probs, cls, CLASSES, top_n, prob_thresh,
                                               nms_thresh)
  if not 0 < top_n < len(probs) and (probs > prob_thresh).sum() > min(1024, max_dets):
    assert count == -1
    assert np.all(dets['anchor'] == -1)
    return None
  n = len(src)
  assert count == n, (count, n)
  d = dets[:n]
  assert d['anchor'].tolist() == src
  assert d['cls'].tolist() == fc
  assert d['prob'].tobytes() == np.asarray(fp, F32).reshape(n).tobytes()
  got = np.stack([d['cx'], d['cy'], d['w'], d['h']], 1)
  assert got.tobytes() == np.asarray(fb, F32).reshape(n, 4).tobytes()
  assert np.all(dets[n:]['anchor'] == -1)
  return src


def run_filter(boxes, probs, cls, top_n, prob_thresh=PROB_THRESH, nms_thresh=NMS_THRESH,
               max_dets=None):
  dets, counts = topk_nms_gpu(boxes[None], probs[None], cls[None], CLASSES, top_n, prob_thresh,
                              nms_thresh, max_dets=max_dets)
  return check_filter_bits(dets[0], int(counts[0]), boxes, probs, cls, top_n, prob_thresh,
                           nms_thresh)


def scattered_boxes(A, rng):
  """Boxes over a 1242 x 375 image (few overlap) and class ids."""
  boxes = np.stack([rng.uniform(0, 1242, A), rng.uniform(0, 375, A), rng.uniform(8, 60, A),
                    rng.uniform(8, 40, A)], 1).astype(F32)
  return boxes, rng.integers(0, CLASSES, A).astype(np.int64)


def pair_up(boxes, cls, idx):
  """Anchors idx (ascending) in consecutive pairs, the second of each pair the first's box moved
  half a pixel and its class: IoU far above NMS_THRESH, so which one survives follows their rank,
  and for equal scores their anchors."""
  idx = np.sort(idx)
  first, second = idx[0::2][:len(idx) // 2], idx[1::2]
  boxes[second] = boxes[first] + np.array([0.5, 0.5, 0, 0], F32)
  cls[second] = cls[first]


def signed_zeros(n, rng):
  return np.where(rng.random(n) < 0.5, F32(-0.0), F32(0.0)).astype(F32)


@gpu
@pytest.mark.parametrize('A', [3000, 30000])   # scores in registers (A <= 24576) and from L2
def test_filter_signed_zeros_tie(A, gpu_device):
  """40 positive scores, then a run of mixed +0.0 / -0.0 where the top-64 cut falls, then
  negative scores.  -0.0 == +0.0, so the cut takes the lowest zero-scored anchors whatever their
  sign, and of two overlapping zero-scored boxes the lower anchor suppresses the other."""
  rng = np.random.default_rng(A)
  boxes, cls = scattered_boxes(A, rng)
  probs = signed_zeros(A, rng)
  idx = rng.permutation(A)
  probs[idx[:40]] = rng.uniform(0.01, 1, 40)
  probs[idx[40:140]] = -rng.uniform(0.01, 1, 100)
  pair_up(boxes, cls, np.nonzero(probs == 0)[0])
  src = run_filter(boxes, probs, cls, 64)
  kept = probs[src]
  assert np.any((kept == 0) & np.signbit(kept)) and np.any((kept == 0) & ~np.signbit(kept))


@gpu
@pytest.mark.parametrize('A', [3000, 30000])
@pytest.mark.parametrize('top_n', [150, 0])
def test_filter_nan_scores_rank_last(A, top_n, gpu_device):
  """Most scores NaN of either sign or with a payload, 100 finite.  top_n = 150: the 100 finite
  scores and then the 50 NaN-scored anchors lowest in index, NaN ranking last and by anchor in
  NMS too.  top_n = 0 (threshold branch): a NaN is never above PROB_THRESH."""
  rng = np.random.default_rng(A + top_n)
  boxes, cls = scattered_boxes(A, rng)
  probs = rng.choice(np.array([np.nan, NAN_NEG, NAN_PAYLOAD], F32), A)
  idx = rng.permutation(A)
  probs[idx[:100]] = np.concatenate([rng.uniform(0.01, 1, 60), signed_zeros(20, rng),
                                     -rng.uniform(0.01, 1, 15), [-np.inf] * 5]).astype(F32)
  pair_up(boxes, cls, np.nonzero(np.isnan(probs))[0])
  pair_up(boxes, cls, np.nonzero(probs == 0)[0])
  src = run_filter(boxes, probs, cls, top_n)
  kept = probs[src]
  if top_n:
    assert np.isnan(kept).sum() > 10 and len({v.tobytes() for v in kept[np.isnan(kept)]}) == 3
  else:
    assert np.all(kept > PROB_THRESH)


SPECIALS = np.array([np.inf, 1.0, np.nextafter(F32(PROB_THRESH), F32(1)), PROB_THRESH,
                     np.nextafter(F32(PROB_THRESH), F32(0)), FLT_MIN, SUB_MAX, TINY, 0.0, -0.0,
                     -TINY, -SUB_MAX, -np.inf], F32)


@gpu
@pytest.mark.parametrize('top_n,prob_thresh', [(170, PROB_THRESH), (590, PROB_THRESH),
                                               (0, PROB_THRESH), (0, -1.0)])
def test_filter_special_scores(top_n, prob_thresh, gpu_device):
  """+-inf, subnormals, FLT_MIN, +-0.0 and PROB_THRESH itself with its float32 neighbours, 20
  anchors each, over negative filler.  top_n = 170 cuts inside the zeros, 590 inside -inf; the
  threshold branch keeps only scores strictly above PROB_THRESH, and with a threshold of -1 it
  takes every zero and subnormal into NMS."""
  A = 600
  rng = np.random.default_rng(top_n + 3)
  boxes, cls = scattered_boxes(A, rng)
  probs = -rng.uniform(0.001, 1, A).astype(F32)
  idx = rng.permutation(A)
  probs[idx[:20 * len(SPECIALS)]] = np.repeat(SPECIALS, 20)
  for v in SPECIALS[~((SPECIALS == 0) & np.signbit(SPECIALS))]:   # zeros pair across signs
    pair_up(boxes, cls, np.nonzero(probs == v)[0])
  src = run_filter(boxes, probs, cls, top_n, prob_thresh)
  if top_n == 0 and prob_thresh == PROB_THRESH:
    assert set(probs[src].tolist()) <= {np.inf, 1.0, float(SPECIALS[2])}


@gpu
@pytest.mark.parametrize('extra', [0, 1])
def test_filter_top_n_not_below_anchor_count(extra, gpu_device):
  """top_n == A and top_n == A + 1 run the threshold branch (nn_skeleton.py:711)."""
  A = 500
  rng = np.random.default_rng(extra)
  boxes, cls = scattered_boxes(A, rng)
  probs = rng.uniform(0, 0.004, A).astype(F32)
  probs[rng.permutation(A)[:100]] = rng.uniform(0.5, 1, 100)
  src = run_filter(boxes, probs, cls, A + extra)
  assert np.all(probs[src] > PROB_THRESH)


@gpu
@pytest.mark.parametrize('top_n', [0, 2])
@pytest.mark.parametrize('a_first', [True, False])
@pytest.mark.parametrize('wider', [False, True])
def test_filter_iou_at_nms_thresh(wider, a_first, top_n, gpu_device):
  """a = (0, 0, 2, 1) and b = (0, 0, 5, 1) have IoU 2 / 5, exactly float32(0.4): not above
  NMS_THRESH, so both stay.  With a's width one ulp wider the IoU is 0.40000004 and the
  higher-ranked box suppresses the other.  A third, distant box makes A = 3."""
  aw = np.nextafter(F32(2), F32(3)) if wider else F32(2)
  boxes = np.array([[0, 0, aw, 1], [0, 0, 5, 1], [100, 100, 5, 5]], F32)
  probs = np.array([0.9, 0.8, 0.7] if a_first else [0.8, 0.9, 0.7], F32)
  cls = np.zeros(3, np.int64)
  iou = oracle.batch_iou(boxes[1:2], boxes[0])[0]
  assert iou.dtype == F32 and (iou > F32(NMS_THRESH)) == wider
  assert wider or iou == F32(NMS_THRESH)
  src = run_filter(boxes, probs, cls, top_n)
  assert len(src) == (3 if top_n == 0 else 2) - int(wider)


@gpu
@pytest.mark.parametrize('top_n', [0, 8])
def test_filter_zero_area_and_identical_boxes(top_n, gpu_device):
  """Identical boxes of one class: IoU 1, the lower-ranked goes (also at equal scores, where the
  lower anchor ranks first).  Identical zero-area boxes: IoU 0 / 0 = NaN, which does not
  suppress.  A zero-area box inside a real one: IoU 0.  Another class never suppresses."""
  boxes = np.array([[10, 10, 20, 20], [10, 10, 20, 20], [50, 50, 0, 10], [50, 50, 0, 10],
                    [50, 50, 10, 10], [80, 80, 0, 0], [80, 80, 0, 0], [10, 10, 20, 20],
                    [10, 10, 20, 20]], F32)
  probs = np.array([0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3, 0.9, 0.9], F32)
  cls = np.array([0, 0, 0, 0, 0, 0, 0, 1, 0], np.int64)
  src = run_filter(boxes, probs, cls, top_n)
  assert src == ([0, 2, 3, 4, 5, 6, 7] if top_n == 0 else [0, 2, 3, 4, 5, 7])


@gpu
def test_filter_batch_with_some_images_overflowing(gpu_device):
  """Ten images in one launch of the threshold branch with max_dets = 100: the images with more
  than 100 scores above PROB_THRESH report count -1 with every record's anchor -1, the others are
  filtered normally, and each image's records equal its own single-image launch."""
  A, max_dets = 3000, 100
  n_above = [0, 1, 50, 99, 100, 101, 200, 3000, 64, 100]
  rng = np.random.default_rng(8)
  B = len(n_above)
  boxes, probs, cls = [], [], []
  for n in n_above:
    bx, c = scattered_boxes(A, rng)
    p = rng.uniform(0, 0.004, A).astype(F32)
    p[rng.permutation(A)[:n]] = rng.uniform(0.5, 1, n)
    boxes.append(bx)
    probs.append(p)
    cls.append(c)
  boxes, probs, cls = np.stack(boxes), np.stack(probs), np.stack(cls)
  dets, counts = topk_nms_gpu(boxes, probs, cls, CLASSES, 0, PROB_THRESH, NMS_THRESH,
                              max_dets=max_dets)
  for i in range(B):
    one, one_count = topk_nms_gpu(boxes[i:i + 1], probs[i:i + 1], cls[i:i + 1], CLASSES, 0,
                                  PROB_THRESH, NMS_THRESH, max_dets=max_dets)
    assert dets[i].tobytes() == one[0].tobytes() and counts[i] == one_count[0], i
    check_filter_bits(dets[i], int(counts[i]), boxes[i], probs[i], cls[i], 0)
  assert [i for i in range(B) if counts[i] == -1] == [5, 6, 7]


# ---- the filter's sort key, restated (no GPU) ---------------------------------------------------
def filter_sort_key(probs):
  """filter_kernel's 64-bit rank key: order_key(prob) << 32 | ~anchor, where order_key maps a
  float to an unsigned key that grows with it, -0.0 to the key of +0.0, and NaN to 0."""
  f = np.asarray(probs, F32)
  u = f.view(np.uint32).astype(np.uint64)
  key = np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000)
  key = np.where(f == 0, np.uint64(0x80000000), key)
  key = np.where(np.isnan(f), np.uint64(0), key)
  anchor = np.arange(len(f), dtype=np.uint64)
  return (key << np.uint64(32)) | (~anchor & np.uint64(0xffffffff))


def test_order_key_ranks_as_oracle():
  """Sorting by the kernel's key, descending, gives oracle.postproc._rank_order on special
  values: +-0, +-inf, NaN of either sign and with a payload, subnormals, and ties."""
  example = np.array([0, -0.0, np.nan, -np.nan, 0.5, -np.inf, np.nan, 0], F32)
  assert oracle.postproc._rank_order(example).tolist() == [4, 0, 1, 7, 5, 2, 3, 6]
  assert np.argsort(filter_sort_key(example))[::-1].tolist() == [4, 0, 1, 7, 5, 2, 3, 6]
  pool = np.concatenate([SPECIALS, np.array([np.nan, NAN_NEG, NAN_PAYLOAD, 0.5, -0.5, 3e38, -3e38],
                                            F32)])
  rng = np.random.default_rng(0)
  for n in (2, 7, 64, 1000):
    for _ in range(20):
      p = rng.choice(pool, n).astype(F32)
      assert np.array_equal(np.argsort(filter_sort_key(p))[::-1],
                            oracle.postproc._rank_order(p)), p
