// The KITTI 2-D object scorer (the reference's evaluate_object, src/dataset/kitti-eval/cpp/
// evaluate_object.cpp, restated in oracle/kitti_eval.py) on the engine's filtered records: the
// per-(class, difficulty, threshold) TP / FP / FN counts and ordered similarity sums from which
// the host forms precision, AOS and AP exactly as the binary does.  Five launches on the caller's
// stream, no host wait:
//   prepare_kernel    the values the binary reads back from eval.py's text (corners
//                     rint(v * 100) / 100, scores k / 1000 as bins k), class codes, record checks
//   recall_kernel     one warp per (image, class, difficulty): computeStatistics without FP
//                     (:345-437) into a 1001-bin histogram of TP scores, and n_gt
//   threshold_kernel  one CTA per (class, difficulty): getThresholds (:239-272) as a histogram
//                     suffix sum and one binary search per threshold
//   pr_kernel         one warp per (image, class, difficulty): computeStatistics with FP
//                     (:345-498) at each threshold
//   sum_kernel        the similarity of each threshold summed in image order (:540-555)
// In the warp kernels the gt loop is serial and lane l owns detections l, l + 32, ..., so with at
// most 1024 records per image each lane's assigned flags are one 32-bit word.  Every double
// operation whose rounding decides a comparison is an explicit _rn intrinsic, so --fmad=true
// cannot contract it.
//
// The detection error analysis (the reference's analyze_detections, src/dataset/kitti.py:182-296,
// restated in oracle/kitti_analysis.py) reads the records back through the same read_back and
// runs in three launches: rank_kernel, line_scan_kernel and line_kernel (see below).
#include "common.cuh"
#include "scan.cuh"

namespace sqdet {
namespace {

constexpr int kCd = 9;                  // 3 classes x 3 difficulties, index 3 * class + difficulty
constexpr int kBins = 1001;             // scores k / 1000, k in 0..1000
constexpr int kMaxThresholds = SQDET_KITTI_MAX_THRESHOLDS;
constexpr int kMaxDets = 1024;
constexpr int kWarpsPerBlock = 8;

// class id k -> 0 car, 1 pedestrian, 2 cyclist or -1, stored + 1 in 2 bits at bit 2 (k % 32) of
// word k / 32 (no array, so reading it needs no stack frame)
struct ClassMap {
  uint64_t lo, hi;
  int classes;
  __device__ int code(int k) const { return (int)(((k < 32 ? lo : hi) >> (2 * (k & 31))) & 3) - 1; }
};

struct Scratch {
  double* box;          // [n * max_dets][4] x1 y1 x2 y2 as the binary reads them
  int32_t* meta;        // [n * max_dets] code << 16 | score bin, or -1 (not car/pedestrian/cyclist)
  int32_t* hist;        // [kCd][kBins] TP scores of the recall pass
  int32_t* thr;         // [kCd][kMaxThresholds] threshold score bins
  double* sim;          // [kCd][kMaxThresholds][n] per-image similarity
};

Scratch carve(Carver& c, int n, int max_dets) {
  const int64_t recs = (int64_t)n * max_dets;
  Scratch s;
  s.box = c.take<double>(recs * 4);
  s.meta = c.take<int32_t>(recs);
  s.hist = c.take<int32_t>(kCd * kBins);
  s.thr = c.take<int32_t>(kCd * kMaxThresholds);
  s.sim = c.take<double>((int64_t)kCd * kMaxThresholds * n);
  return s;
}

int64_t scratch_bytes(int n, int max_dets) {
  Carver c;
  carve(c, n, max_dets);
  return c.offset;
}

__device__ __forceinline__ void refuse(sqdet_kitti_result* out, int image, int reason) {
  atomicMin(reinterpret_cast<unsigned*>(&out->status), (unsigned)(image * 8 + reason));
}

// std::max / std::min as the binary calls them: (a < b) ? b : a and (b < a) ? b : a
__device__ __forceinline__ double dmax(double a, double b) { return a < b ? b : a; }
__device__ __forceinline__ double dmin(double a, double b) { return b < a ? b : a; }

// boxoverlap (:203-237): criterion -1 (union) for det vs gt, 0 (det area) for det vs DontCare
template <bool kUnion>
__device__ __forceinline__ double box_overlap(const double* a, const sqdet_kitti_obj& b) {
  const double w = __dsub_rn(dmin(a[2], b.x2), dmax(a[0], b.x1));
  const double h = __dsub_rn(dmin(a[3], b.y2), dmax(a[1], b.y1));
  if (w <= 0 || h <= 0) return 0;
  const double inter = __dmul_rn(w, h);
  const double a_area = __dmul_rn(__dsub_rn(a[2], a[0]), __dsub_rn(a[3], a[1]));
  if (!kUnion) return __ddiv_rn(inter, a_area);
  const double b_area = __dmul_rn(__dsub_rn(b.x2, b.x1), __dsub_rn(b.y2, b.y1));
  return __ddiv_rn(inter, __dsub_rn(__dadd_rn(a_area, b_area), inter));
}

__device__ __forceinline__ double min_overlap(int c) { return c == 0 ? 0.7 : 0.5; }   // :37

// cleanData's ignored_gt entry (:277-320): 0 counted, 1 ignored, -1 skipped
__device__ __forceinline__ int gt_state(const sqdet_kitti_obj& g, int c, int d) {
  const int valid = g.type == c ? 1
                  : ((c == 0 && g.type == SQDET_KITTI_VAN) ||
                     (c == 1 && g.type == SQDET_KITTI_PERSON_SITTING)) ? 0 : -1;
  const int min_height = d == 0 ? 40 : 25;                          // :28
  const double max_trunc = d == 0 ? 0.15 : d == 1 ? 0.3 : 0.5;      // :30
  const double height = __dsub_rn(g.y2, g.y1);
  const bool ignore = g.occlusion > d || g.truncation > max_trunc || height < min_height;   // :29
  if (valid == 1 && !ignore) return 0;
  if (valid == 0 || (ignore && valid == 1)) return 1;
  return -1;
}

__device__ __forceinline__ int clamp_count(int c, int max_dets) {
  return c < 0 ? 0 : c > max_dets ? max_dets : c;
}

__device__ __forceinline__ bool bad_range(int64_t a, int64_t b, int64_t n_objects) {
  return a < 0 || b < a || b > n_objects;
}

// Image i's objects [g0, g1): empty when its offsets are refused, so that a bad range only sets
// the status word and no kernel reads outside objs (which may be null when n_objects is 0).
__device__ __forceinline__ void object_range(const int64_t* offsets, int i, int64_t n_objects,
                                             int64_t& g0, int64_t& g1) {
  g0 = offsets[i];
  g1 = offsets[i + 1];
  if (bad_range(g0, g1, n_objects)) g0 = g1 = 0;
}

__device__ __forceinline__ bool bad_count(int count, int max_dets) {
  return count < 0 || count > max_dets;
}

// One record as eval.py's detection file gives it back: the corners x1 y1 x2 y2 and the score bin.
struct ReadBack {
  double box[4];
  int bin;
};

// What a reader gets back from `{:.2f}` / `{:.3f}` of the float32 values (v * 100 and p * 1000
// are exact in double, so rint, round-half-even like Python's formatting of exact ties, gives the
// printed decimal; divided back it is strtod's double).  0, or the SQDET_KITTI_* reason the
// record is refused for.
__device__ __forceinline__ int read_back(const sqdet_det& d, int classes, ReadBack& rb) {
  if (d.cls < 0 || d.cls >= classes) return SQDET_KITTI_BAD_CLASS;
  if (!isfinite(d.prob) || !isfinite(d.cx) || !isfinite(d.cy) || !isfinite(d.w) || !isfinite(d.h))
    return SQDET_KITTI_NOT_FINITE;
  if (!(d.prob >= 0.f && d.prob <= 1.f)) return SQDET_KITTI_BAD_SCORE;
  // bbox_transform in float32 (utils/util.py): cx - w / 2 etc., not contracted
  const float hw = __fdiv_rn(d.w, 2.f), hh = __fdiv_rn(d.h, 2.f);
  const float v[4] = {__fsub_rn(d.cx, hw), __fsub_rn(d.cy, hh), __fadd_rn(d.cx, hw),
                      __fadd_rn(d.cy, hh)};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double c = rint(__dmul_rn((double)v[k], 100.0));
    if (!isfinite(c)) return SQDET_KITTI_NOT_FINITE;
    rb.box[k] = __ddiv_rn(c, 100.0);
  }
  rb.bin = (int)rint(__dmul_rn((double)d.prob, 1000.0));
  return 0;
}

// One thread per record: the read-back values and the record checks.
__global__ void prepare_kernel(const sqdet_det* __restrict__ dets, const int32_t* __restrict__ counts,
                               const int64_t* __restrict__ offsets, int64_t n_objects, int n,
                               int max_dets, ClassMap map, Scratch s, sqdet_kitti_result* out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= (int64_t)n * max_dets) return;
  const int i = (int)(r / max_dets), j = (int)(r % max_dets);
  const int count = counts[i];
  if (j == 0) {
    if (bad_count(count, max_dets)) refuse(out, i, SQDET_KITTI_BAD_COUNT);
    const int64_t a = offsets[i], b = offsets[i + 1];
    if (bad_range(a, b, n_objects)) refuse(out, i, SQDET_KITTI_BAD_OFFSETS);
  }
  s.meta[r] = -1;
  if (j >= count) return;
  const sqdet_det d = dets[r];
  ReadBack rb;
  const int why = read_back(d, map.classes, rb);
  if (why) { refuse(out, i, why); return; }
  double* box = s.box + r * 4;
#pragma unroll
  for (int k = 0; k < 4; ++k) box[k] = rb.box[k];
  const int code = map.code(d.cls);
  if (code < 0) return;
  s.meta[r] = code << 16 | rb.bin;
  out->evaluated[code] = 1;
}

// The recall pass (computeStatistics, compute_fp = false): each gt that is not skipped takes the
// unassigned detection of its class overlapping it by more than the minimum with the highest
// score, the first index on equal scores; a TP puts its score bin into the histogram.
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
recall_kernel(const int32_t* __restrict__ counts, const sqdet_kitti_obj* __restrict__ objs,
              const int64_t* __restrict__ offsets, int64_t n_objects, int n, int max_dets, Scratch s,
              sqdet_kitti_result* out) {
  const int w = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= n * kCd) return;
  const int i = w / kCd, cd = w % kCd, c = cd / 3, d = cd % 3;
  const int count = clamp_count(counts[i], max_dets);
  const int slots = (count + 31) >> 5;
  const int64_t base = (int64_t)i * max_dets;
  const double minov = min_overlap(c);
  uint32_t assigned = 0;
  int n_gt = 0;
  int64_t g0, g1;
  object_range(offsets, i, n_objects, g0, g1);
  for (int64_t g = g0; g < g1; ++g) {
    const sqdet_kitti_obj gt = objs[g];
    const int st = gt_state(gt, c, d);
    if (st == -1) continue;
    n_gt += st == 0;
    uint32_t key = 0;                  // (bin + 1) << 10 | (1023 - j): max = best score, first j
    for (int k = 0; k < slots; ++k) {
      const int j = lane + 32 * k;
      if (j >= count || (assigned >> k & 1)) continue;
      const int m = s.meta[base + j];
      if (m < 0 || (m >> 16) != c) continue;
      const uint32_t cand = (uint32_t)((m & 0xffff) + 1) << 10 | (uint32_t)(1023 - j);
      if (cand > key && box_overlap<true>(s.box + (base + j) * 4, gt) > minov) key = cand;
    }
    key = __reduce_max_sync(0xffffffffu, key);
    if (key == 0) continue;                                     // an FN when st == 0
    const int j = 1023 - (int)(key & 1023);
    if ((j & 31) == lane) assigned |= 1u << (j >> 5);
    if (st == 0 && lane == 0) atomicAdd(&s.hist[cd * kBins + (int)(key >> 10) - 1], 1);
  }
  if (lane == 0 && n_gt) atomicAdd(&out->n_gt[cd], n_gt);
}

// getThresholds: v (the TP scores) in descending order is the histogram read from bin 1000 down,
// so v[i] is the bin b with above[b + 1] <= i < above[b], above[b] = TPs scoring b or more.  Index
// i is skipped while it is not the last and (i + 2) / n - r < r - (i + 1) / n; both sides move
// monotonically with i, so the next index taken is one binary search.  r is the binary's running
// sum of 1 / 40.
__global__ void __launch_bounds__(1024) threshold_kernel(Scratch s, sqdet_kitti_result* out) {
  __shared__ int above[kBins + 1];
  const int cd = blockIdx.x;
  for (int b = threadIdx.x; b <= kBins; b += blockDim.x)
    above[b] = b < kBins ? s.hist[cd * kBins + b] : 0;
  __syncthreads();
  for (int step = 1; step < kBins; step <<= 1) {       // suffix sum, Hillis-Steele
    int v[2] = {0, 0};
    for (int t = 0; t < 2; ++t) {
      const int b = threadIdx.x + t * blockDim.x;
      if (b < kBins) v[t] = above[b] + (b + step < kBins ? above[b + step] : 0);
    }
    __syncthreads();
    for (int t = 0; t < 2; ++t) {
      const int b = threadIdx.x + t * blockDim.x;
      if (b < kBins) above[b] = v[t];
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  const int nv = above[0];
  const double n = (double)out->n_gt[cd];
  double r = 0;
  int nt = 0;
  auto skipped = [&](int i) {
    if (i >= nv - 1) return false;
    return __dsub_rn(__ddiv_rn((double)(i + 2), n), r) < __dsub_rn(r, __ddiv_rn((double)(i + 1), n));
  };
  for (int i = 0; i < nv; ++i) {
    int lo = i, hi = nv - 1;                 // the first index not skipped, in [i, nv - 1]
    while (lo < hi) {
      const int mid = lo + (hi - lo) / 2;
      if (skipped(mid)) lo = mid + 1; else hi = mid;
    }
    i = lo;
    int bl = 0, bh = kBins - 1;              // the largest bin b with above[b] > i
    while (bl < bh) {
      const int mid = bl + (bh - bl + 1) / 2;
      if (above[mid] > i) bl = mid; else bh = mid - 1;
    }
    if (nt == kMaxThresholds) {              // cannot happen (oracle/kitti_eval.get_thresholds)
      refuse(out, 0, SQDET_KITTI_TOO_MANY_THRESHOLDS);
      break;
    }
    s.thr[cd * kMaxThresholds + nt++] = bl;
    r = __dadd_rn(r, 1.0 / 40.0);
  }
  out->n_thresholds[cd] = nt;
}

// The PR pass (computeStatistics, compute_fp = true) at each threshold: detections scoring below
// it are left out, each gt takes the unassigned detection with the largest overlap above the
// minimum (the first index on equal overlaps), and FP counts the eligible detections left
// unassigned that no DontCare box holds by more than the minimum.  The similarity is 0.0 plus
// each TP's gt term in gt order.
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
pr_kernel(const int32_t* __restrict__ counts, const sqdet_kitti_obj* __restrict__ objs,
          const int64_t* __restrict__ offsets, int64_t n_objects, int n, int max_dets, Scratch s,
          sqdet_kitti_result* out) {
  const int w = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= n * kCd) return;
  const int i = w / kCd, cd = w % kCd, c = cd / 3, d = cd % 3;
  const int nt = out->n_thresholds[cd];
  if (nt == 0) return;
  const int count = clamp_count(counts[i], max_dets);
  const int slots = (count + 31) >> 5;
  const int64_t base = (int64_t)i * max_dets;
  int64_t g0, g1;
  object_range(offsets, i, n_objects, g0, g1);
  const double minov = min_overlap(c);
  uint32_t mine = 0, stuff = 0;          // this lane's detections of class c; held by DontCare
  for (int k = 0; k < slots; ++k) {
    const int j = lane + 32 * k;
    if (j >= count) break;
    const int m = s.meta[base + j];
    if (m < 0 || (m >> 16) != c) continue;
    mine |= 1u << k;
    for (int64_t g = g0; g < g1; ++g) {
      const sqdet_kitti_obj gt = objs[g];
      if (gt.type == SQDET_KITTI_DONTCARE && box_overlap<false>(s.box + (base + j) * 4, gt) > minov) {
        stuff |= 1u << k;
        break;
      }
    }
  }
  for (int t = 0; t < nt; ++t) {
    const int thr = s.thr[cd * kMaxThresholds + t];
    uint32_t elig = 0;
    for (int k = 0; k < slots; ++k)
      if ((mine >> k & 1) && (s.meta[base + lane + 32 * k] & 0xffff) >= thr) elig |= 1u << k;
    uint32_t assigned = 0;
    int tp = 0, fn = 0;
    double sim = 0;
    for (int64_t g = g0; g < g1; ++g) {
      const sqdet_kitti_obj gt = objs[g];
      const int st = gt_state(gt, c, d);
      if (st == -1) continue;
      double best = 0;
      int bj = kMaxDets;
      for (int k = 0; k < slots; ++k) {
        if (!((elig & ~assigned) >> k & 1)) continue;
        const int j = lane + 32 * k;
        const double o = box_overlap<true>(s.box + (base + j) * 4, gt);
        if (o > minov && o > best) { best = o; bj = j; }
      }
      for (int off = 16; off; off >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, off);
        if (ob > best || (ob == best && oj < bj)) { best = ob; bj = oj; }
      }
      if (bj == kMaxDets) {
        fn += st == 0;
        continue;
      }
      if ((bj & 31) == lane) assigned |= 1u << (bj >> 5);
      if (st == 0) {
        ++tp;
        sim = __dadd_rn(sim, gt.aos_term);
      }
    }
    int fp = __popc(elig & ~assigned & ~stuff);
    for (int off = 16; off; off >>= 1) fp += __shfl_xor_sync(0xffffffffu, fp, off);
    if (lane == 0) {
      const int o = cd * kMaxThresholds + t;
      if (tp) atomicAdd(&out->tp[0][0] + o, tp);
      if (fp) atomicAdd(&out->fp[0][0] + o, fp);
      if (fn) atomicAdd(&out->fn[0][0] + o, fn);
      s.sim[(int64_t)o * n + i] = sim;
    }
  }
}

// pr[t].similarity += the image's similarity, in image order (a sum of +0.0 changes nothing, so
// the images without TP or FP, whose similarity the binary skips, add their 0.0)
__global__ void sum_kernel(int n, Scratch s, sqdet_kitti_result* out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= kCd * kMaxThresholds || o % kMaxThresholds >= out->n_thresholds[o / kMaxThresholds]) return;
  const double* p = s.sim + (int64_t)o * n;
  double sum = 0;
  for (int i = 0; i < n; ++i) sum = __dadd_rn(sum, p[i]);
  (&out->similarity[0][0])[o] = sum;
}

// ---- detection error analysis (sqdet_kitti_analyze) -------------------------------------------
// Three launches: rank_kernel (one CTA per image: read-back, ranking, matching, counts),
// line_scan_kernel (one CTA: each image's first line), line_kernel (one CTA per image: the lines).

constexpr int kAnalyzeThreads = 256;
constexpr int kMaxAnalyzeImages = (1 << 27) - 1;
constexpr uint32_t kUnclaimed = 0xffffffffu;
enum { kLoc = SQDET_KITTI_ERR_LOC, kCls = SQDET_KITTI_ERR_CLS, kBg = SQDET_KITTI_ERR_BG,
       kHit = 4 };                 // IoU >= 0.5 with its own class: correct or repeated

// label type code -> class id (-1: not analyzed), stored + 1 in 2 bits per code
struct TypeMap {
  uint32_t bits;
  __device__ int class_of(int type) const {
    return type < 0 || type > SQDET_KITTI_OTHER ? -1 : (int)(bits >> (2 * type) & 3) - 1;
  }
};

struct AnalyzeScratch {
  double* box;          // [n * max_dets][4] x1 y1 x2 y2 as read back
  int32_t* slot;        // [n * max_dets] ranked detection t: j | type << 10 | bin << 13 | cls << 23
  uint32_t* claim;      // [n_objects] the first correct detection's rank, or kUnclaimed
  int32_t* kept;        // [n] counted detections
  int64_t* lines;       // [n] error lines, then the image's first line
};

AnalyzeScratch carve_analyze(Carver& c, int n, int max_dets, int64_t n_objects) {
  const int64_t recs = (int64_t)n * max_dets;
  AnalyzeScratch s;
  s.box = c.take<double>(recs * 4);
  s.slot = c.take<int32_t>(recs);
  s.claim = c.take<uint32_t>(n_objects);
  s.kept = c.take<int32_t>(n);
  s.lines = c.take<int64_t>(n);
  return s;
}

int64_t analyze_scratch_bytes(int n, int max_dets, int64_t n_objects) {
  Carver c;
  carve_analyze(c, n, max_dets, n_objects);
  return c.offset;
}

__device__ __forceinline__ void refuse16(sqdet_kitti_analysis* out, int image, int reason) {
  atomicMin(reinterpret_cast<unsigned*>(&out->status), (unsigned)(image * 16 + reason));
}

// bbox_transform_inv (utils/util.py:181-196) in double: w = (x2 - x1) + 1.0, cx = x1 + 0.5 * w
struct Center {
  double cx, cy, w, h;
};
__device__ __forceinline__ Center center_of(double x1, double y1, double x2, double y2) {
  Center c;
  c.w = __dadd_rn(__dsub_rn(x2, x1), 1.0);
  c.h = __dadd_rn(__dsub_rn(y2, y1), 1.0);
  c.cx = __dadd_rn(x1, __dmul_rn(0.5, c.w));
  c.cy = __dadd_rn(y1, __dmul_rn(0.5, c.h));
  return c;
}

__device__ __forceinline__ double dmax0(double a) { return a < 0 ? 0.0 : a; }

// batch_iou (utils/util.py:32-54) of one ground-truth box g and one detection d, in numpy's
// operation order; np.minimum / np.maximum agree with these on the finite values reaching here
__device__ __forceinline__ double batch_iou(const Center& g, const Center& d) {
  const double lr = dmax0(__dsub_rn(
      dmin(__dadd_rn(g.cx, __dmul_rn(0.5, g.w)), __dadd_rn(d.cx, __dmul_rn(0.5, d.w))),
      dmax(__dsub_rn(g.cx, __dmul_rn(0.5, g.w)), __dsub_rn(d.cx, __dmul_rn(0.5, d.w)))));
  const double tb = dmax0(__dsub_rn(
      dmin(__dadd_rn(g.cy, __dmul_rn(0.5, g.h)), __dadd_rn(d.cy, __dmul_rn(0.5, d.h))),
      dmax(__dsub_rn(g.cy, __dmul_rn(0.5, g.h)), __dsub_rn(d.cy, __dmul_rn(0.5, d.h)))));
  const double inter = __dmul_rn(lr, tb);
  const double uni = __dsub_rn(__dadd_rn(__dmul_rn(g.w, g.h), __dmul_rn(d.w, d.h)), inter);
  return __ddiv_rn(inter, uni);
}

// the reference's assertions on a label box of an analyzed class, and finite corners
__device__ __forceinline__ bool label_ok(const sqdet_kitti_obj& o) {
  return o.x1 >= 0 && o.x1 <= o.x2 && o.y1 >= 0 && o.y1 <= o.y2 && isfinite(o.x2) &&
         isfinite(o.y2);
}

// One CTA per image.  A record's rank is the number of records whose key (score bin, then lower
// class id, then lower index) is larger; the first G ranks are counted.  Each counted detection
// takes the first object of largest IoU; a hit claims its object with atomicMin of its rank, so
// the first claimant is the correct one and later ones are repeated.
__global__ void __launch_bounds__(kAnalyzeThreads)
rank_kernel(const sqdet_det* __restrict__ dets, const int32_t* __restrict__ counts,
            const sqdet_kitti_obj* __restrict__ objs, const int64_t* __restrict__ offsets,
            int64_t n_objects, int max_dets, int classes, TypeMap map, AnalyzeScratch s,
            sqdet_kitti_analysis* out) {
  __shared__ uint32_t key[kMaxDets];
  __shared__ int16_t kept[kMaxDets];
  __shared__ int8_t type[kMaxDets];
  __shared__ int64_t hit_gt[kMaxDets];
  __shared__ int tally[7];           // G, loc, cls, bg, hits, correct, missed
  const int i = blockIdx.x, tid = threadIdx.x;
  const int64_t base = (int64_t)i * max_dets;
  const int raw = counts[i];
  if (tid < 7) tally[tid] = 0;
  if (tid == 0) {
    if (bad_count(raw, max_dets)) refuse16(out, i, SQDET_KITTI_BAD_COUNT);
    if (bad_range(offsets[i], offsets[i + 1], n_objects)) refuse16(out, i, SQDET_KITTI_BAD_OFFSETS);
  }
  const int count = clamp_count(raw, max_dets);
  int64_t g0, g1;
  object_range(offsets, i, n_objects, g0, g1);
  __syncthreads();
  for (int64_t g = g0 + tid; g < g1; g += blockDim.x) {
    const sqdet_kitti_obj o = objs[g];
    if (map.class_of(o.type) < 0) continue;
    atomicAdd(&tally[0], 1);
    s.claim[g] = kUnclaimed;
    if (!label_ok(o)) refuse16(out, i, SQDET_KITTI_BAD_LABEL);
  }
  for (int j = tid; j < count; j += blockDim.x) {
    const sqdet_det d = dets[base + j];
    ReadBack rb;
    int why = read_back(d, classes, rb);
    if (!why && (d.w < 0.f || d.h < 0.f)) why = SQDET_KITTI_NEGATIVE_SIZE;
    if (why) {                           // the image is refused; keep the keys distinct
      refuse16(out, i, why);
      rb.bin = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) rb.box[k] = 0;
    }
    double* box = s.box + (base + j) * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) box[k] = rb.box[k];
    const int cls = why ? 0 : d.cls;
    key[j] = (uint32_t)rb.bin << 16 | (uint32_t)(63 - cls) << 10 | (uint32_t)(1023 - j);
  }
  __syncthreads();
  const int n_gt = tally[0];
  const int n_kept = n_gt < count ? n_gt : count;
  if (n_kept > 0) {
    for (int j = tid; j < count; j += blockDim.x) {
      const uint32_t mine = key[j];
      int rank = 0;
      for (int k = 0; k < count; ++k) rank += key[k] > mine;
      if (rank < n_kept) kept[rank] = (int16_t)j;
    }
    __syncthreads();
    for (int t = tid; t < n_kept; t += blockDim.x) {
      const int j = kept[t];
      const double* b = s.box + (base + j) * 4;
      const Center dc = center_of(b[0], b[1], b[2], b[3]);
      const uint32_t k = key[j];
      const int cls = 63 - (int)(k >> 10 & 63), bin = (int)(k >> 16);
      double best = -1.0;                // every IoU is >= 0 (+0.0 or -0.0)
      int64_t best_g = g0;
      int best_cls = -1;
      for (int64_t g = g0; g < g1; ++g) {
        const sqdet_kitti_obj o = objs[g];
        const int gc = map.class_of(o.type);
        if (gc < 0) continue;
        const double iou = batch_iou(center_of(o.x1, o.y1, o.x2, o.y2), dc);
        if (iou > best) { best = iou; best_g = g; best_cls = gc; }     // np.argmax: the first
      }
      int ty;
      if (best > 0.1) ty = best_cls != cls ? kCls : best >= 0.5 ? kHit : kLoc;
      else ty = kBg;
      if (ty == kHit) {
        atomicMin(&s.claim[best_g], (uint32_t)t);
        hit_gt[t] = best_g;
      }
      type[t] = (int8_t)ty;
      atomicAdd(&tally[ty == kHit ? 4 : 1 + ty], 1);
      s.slot[base + t] = j | ty << 10 | bin << 13 | cls << 23;
    }
    __syncthreads();
    for (int t = tid; t < n_kept; t += blockDim.x)
      if (type[t] == kHit && s.claim[hit_gt[t]] == (uint32_t)t) atomicAdd(&tally[5], 1);
  }
  for (int64_t g = g0 + tid; g < g1; g += blockDim.x)
    if (map.class_of(objs[g].type) >= 0 && s.claim[g] == kUnclaimed) atomicAdd(&tally[6], 1);
  __syncthreads();
  if (tid == 0) {
    s.kept[i] = n_kept;
    s.lines[i] = tally[1] + tally[2] + tally[3] + tally[6];
    typedef unsigned long long u64;
    const int64_t add[8] = {n_kept, n_gt, tally[5], tally[1], tally[2], tally[3],
                            tally[4] - tally[5], tally[5]};
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (add[k]) atomicAdd(reinterpret_cast<u64*>(&out->num_dets) + k, (u64)add[k]);
  }
}

// Each image's first line: an exclusive scan of the line counts in image order.
__global__ void __launch_bounds__(1024) line_scan_kernel(int n, AnalyzeScratch s,
                                                         sqdet_kitti_analysis* out) {
  __shared__ int64_t warp[32];
  int64_t run = 0;
  for (int c = 0; c < n; c += blockDim.x) {
    const int i = c + threadIdx.x;
    const int64_t v = i < n ? s.lines[i] : 0;
    int64_t total;
    const int64_t before = block_exclusive_scan(v, warp, &total);
    if (i < n) s.lines[i] = run + before;
    run += total;
  }
  if (threadIdx.x == 0) out->n_lines = run;
}

__device__ __forceinline__ void put_line(sqdet_kitti_error_line* lines, int64_t capacity,
                                         int64_t at, int image, int ty, int cls, const Center& c,
                                         double score) {
  if (at >= capacity) return;
  sqdet_kitti_error_line l;
  l.image = image;
  l.type = ty;
  l.cls = cls;
  l.reserved = 0;
  const double hw = __ddiv_rn(c.w, 2.0), hh = __ddiv_rn(c.h, 2.0);   // _save_detection's w / 2.
  l.x1 = __dsub_rn(c.cx, hw);
  l.y1 = __dsub_rn(c.cy, hh);
  l.x2 = __dadd_rn(c.cx, hw);
  l.y2 = __dadd_rn(c.cy, hh);
  l.score = score;
  lines[at] = l;
}

// One CTA per image: its loc / cls / bg detections in ranked order, then its unclaimed objects
// in label order, each at its first line plus a block scan of the flags before it.
__global__ void __launch_bounds__(kAnalyzeThreads)
line_kernel(const sqdet_kitti_obj* __restrict__ objs, const int64_t* __restrict__ offsets,
            int64_t n_objects, int max_dets, TypeMap map, AnalyzeScratch s,
            sqdet_kitti_error_line* __restrict__ lines, int64_t capacity) {
  __shared__ int64_t warp[kAnalyzeThreads / 32];
  const int i = blockIdx.x, tid = threadIdx.x;
  const int64_t base = (int64_t)i * max_dets;
  const int n_kept = s.kept[i];
  int64_t at = s.lines[i];
  for (int c = 0; c < n_kept; c += blockDim.x) {
    const int t = c + tid;
    const int v = t < n_kept ? s.slot[base + t] : 0;
    const int ty = v >> 10 & 7;
    const bool err = t < n_kept && ty != kHit;
    int64_t total;
    const int64_t before = block_exclusive_scan(err ? 1 : 0, warp, &total);
    if (err) {
      const double* b = s.box + (base + (v & 1023)) * 4;
      put_line(lines, capacity, at + before, i, ty, v >> 23, center_of(b[0], b[1], b[2], b[3]),
               __ddiv_rn((double)(v >> 13 & 1023), 1000.0));
    }
    at += total;
  }
  int64_t g0, g1;
  object_range(offsets, i, n_objects, g0, g1);
  for (int64_t c = g0; c < g1; c += blockDim.x) {
    const int64_t g = c + tid;
    int gc = -1;
    sqdet_kitti_obj o;
    if (g < g1) {
      o = objs[g];
      gc = map.class_of(o.type);
    }
    const bool missed = gc >= 0 && s.claim[g] == kUnclaimed;
    int64_t total;
    const int64_t before = block_exclusive_scan(missed ? 1 : 0, warp, &total);
    if (missed)
      put_line(lines, capacity, at + before, i, SQDET_KITTI_ERR_MISSED, gc,
               center_of(o.x1, o.y1, o.x2, o.y2), -1.0);
    at += total;
  }
}

}  // namespace
}  // namespace sqdet

using namespace sqdet;

int64_t sqdet_kitti_eval_scratch_bytes(int n, int max_dets, int64_t n_objects) {
  if (n < 1 || max_dets < 1 || max_dets > kMaxDets || n_objects < 0) {
    fail(SQDET_ERR_INVALID_ARG, "sqdet_kitti_eval_scratch_bytes: need n >= 1, max_dets in "
                                "[1, 1024] and n_objects >= 0");
    return -1;
  }
  return scratch_bytes(n, max_dets);
}

namespace {

// The checks both entry points make before any launch, in this order; fills `map`.
int check_args(const std::string& name, int n, int max_dets, const sqdet_det* dets,
               const int32_t* counts, int classes, const int32_t* class_map,
               const sqdet_kitti_obj* objs, const int64_t* offsets, int64_t n_objects,
               const void* scratch, const void* out, ClassMap& map) {
  if (n < 1) return fail(SQDET_ERR_INVALID_ARG, name + ": n must be at least 1");
  if (max_dets < 1 || max_dets > kMaxDets)
    return fail(SQDET_ERR_INVALID_ARG, name + ": max_dets must be in [1, 1024]");
  if (n_objects < 0) return fail(SQDET_ERR_INVALID_ARG, name + ": n_objects must be >= 0");
  if (!dets || !counts || !class_map || !offsets || !scratch || !out || (n_objects && !objs))
    return fail(SQDET_ERR_INVALID_ARG, name + ": null argument");
  if (classes < 1 || classes > SQDET_KITTI_MAX_CLASSES)
    return fail(SQDET_ERR_INVALID_ARG, name + ": classes must be in [1, 64]");
  map = ClassMap{};
  map.classes = classes;
  int seen[3] = {0, 0, 0};
  for (int k = 0; k < classes; ++k) {
    const int v = class_map[k];
    if (v < -1 || v > 2) return fail(SQDET_ERR_INVALID_ARG, name + ": class_map entries are -1, 0, 1 or 2");
    // the detection files group lines by class id, so two ids of one KITTI class would order
    // that class's detections differently from the records
    if (v >= 0 && seen[v]++)
      return fail(SQDET_ERR_INVALID_ARG, name + ": two class ids map to the same KITTI class");
    (k < 32 ? map.lo : map.hi) |= (uint64_t)(v + 1) << (2 * (k & 31));
  }
  if ((uintptr_t)scratch % 256)
    return fail(SQDET_ERR_INVALID_ARG, name + ": scratch must be 256-byte aligned");
  if ((uintptr_t)out % alignof(double) || (uintptr_t)offsets % alignof(int64_t) ||
      (uintptr_t)objs % alignof(double) || (uintptr_t)dets % alignof(int32_t) ||
      (uintptr_t)counts % alignof(int32_t))
    return fail(SQDET_ERR_INVALID_ARG, name + ": misaligned argument");
  return SQDET_OK;
}

// The records' device when every input lies inside one allocation on it, else -1.
int inputs_device(int n, int max_dets, const sqdet_det* dets, const int32_t* counts,
                  const sqdet_kitti_obj* objs, const int64_t* offsets, int64_t n_objects,
                  const void* scratch, int64_t scratch_bytes_) {
  const int device = pointer_device(dets);
  if (device < 0 || !device_range_ok(dets, (int64_t)n * max_dets * sizeof(sqdet_det), device) ||
      !device_range_ok(counts, (int64_t)n * 4, device) ||
      !device_range_ok(offsets, (int64_t)(n + 1) * 8, device) ||
      (n_objects && !device_range_ok(objs, n_objects * (int64_t)sizeof(sqdet_kitti_obj), device)) ||
      !device_range_ok(scratch, scratch_bytes_, device))
    return -1;
  return device;
}

}  // namespace

int sqdet_kitti_eval(int n, int max_dets, const sqdet_det* dets, const int32_t* counts,
                     int classes, const int32_t* class_map, const sqdet_kitti_obj* objs,
                     const int64_t* offsets, int64_t n_objects, void* scratch,
                     int64_t scratch_bytes_, sqdet_kitti_result* out, void* stream) {
  const std::string name = "sqdet_kitti_eval";
  ClassMap map;
  const int rc = check_args(name, n, max_dets, dets, counts, classes, class_map, objs, offsets,
                            n_objects, scratch, out, map);
  if (rc != SQDET_OK) return rc;
  if (scratch_bytes_ < scratch_bytes(n, max_dets))
    return fail(SQDET_ERR_INVALID_ARG, name + ": scratch_bytes is below sqdet_kitti_eval_scratch_bytes");
  const int device = inputs_device(n, max_dets, dets, counts, objs, offsets, n_objects, scratch,
                                   scratch_bytes_);
  if (device < 0 || !device_range_ok(out, sizeof(sqdet_kitti_result), device))
    return fail(SQDET_ERR_INVALID_ARG, name + ": dets, counts, objs, offsets, scratch and out must "
                                              "each lie inside one allocation on one device");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select the records' device");
  cudaStream_t st = (cudaStream_t)stream;
  Carver c{static_cast<uint8_t*>(scratch)};
  const Scratch s = carve(c, n, max_dets);
  SQ_CUDA(cudaMemsetAsync(out, 0, sizeof(sqdet_kitti_result), st));
  SQ_CUDA(cudaMemsetAsync(&out->status, 0xff, sizeof(out->status), st));
  SQ_CUDA(cudaMemsetAsync(s.hist, 0, kCd * kBins * 4, st));
  const int64_t recs = (int64_t)n * max_dets;
  prepare_kernel<<<(unsigned)((recs + 255) / 256), 256, 0, st>>>(dets, counts, offsets, n_objects, n,
                                                                 max_dets, map, s, out);
  SQ_CHECK_LAUNCH("kitti prepare_kernel");
  const unsigned warp_blocks = (unsigned)(((int64_t)n * kCd + kWarpsPerBlock - 1) / kWarpsPerBlock);
  recall_kernel<<<warp_blocks, kWarpsPerBlock * 32, 0, st>>>(counts, objs, offsets, n_objects, n, max_dets, s, out);
  SQ_CHECK_LAUNCH("kitti recall_kernel");
  threshold_kernel<<<kCd, 1024, 0, st>>>(s, out);
  SQ_CHECK_LAUNCH("kitti threshold_kernel");
  pr_kernel<<<warp_blocks, kWarpsPerBlock * 32, 0, st>>>(counts, objs, offsets, n_objects, n, max_dets, s, out);
  SQ_CHECK_LAUNCH("kitti pr_kernel");
  sum_kernel<<<(kCd * kMaxThresholds + 127) / 128, 128, 0, st>>>(n, s, out);
  SQ_CHECK_LAUNCH("kitti sum_kernel");
  return SQDET_OK;
}

int64_t sqdet_kitti_analyze_scratch_bytes(int n, int max_dets, int64_t n_objects) {
  if (n < 1 || n > kMaxAnalyzeImages || max_dets < 1 || max_dets > kMaxDets || n_objects < 0) {
    fail(SQDET_ERR_INVALID_ARG, "sqdet_kitti_analyze_scratch_bytes: need n in [1, 2^27 - 1], "
                                "max_dets in [1, 1024] and n_objects >= 0");
    return -1;
  }
  return analyze_scratch_bytes(n, max_dets, n_objects);
}

int sqdet_kitti_analyze(int n, int max_dets, const sqdet_det* dets, const int32_t* counts,
                        int classes, const int32_t* class_map, const sqdet_kitti_obj* objs,
                        const int64_t* offsets, int64_t n_objects, void* scratch,
                        int64_t scratch_bytes_, sqdet_kitti_analysis* out,
                        sqdet_kitti_error_line* lines, int64_t line_capacity, void* stream) {
  const std::string name = "sqdet_kitti_analyze";
  ClassMap cmap;
  const int rc = check_args(name, n, max_dets, dets, counts, classes, class_map, objs, offsets,
                            n_objects, scratch, out, cmap);
  if (rc != SQDET_OK) return rc;
  if (n > kMaxAnalyzeImages)        // out->status is 16 * image + reason
    return fail(SQDET_ERR_INVALID_ARG, name + ": n must be below 2^27");
  // a detection's class id is compared with its object's, so every id names an analyzed class
  TypeMap map{0};
  for (int k = 0; k < classes; ++k) {
    if (class_map[k] < 0)
      return fail(SQDET_ERR_INVALID_ARG, name + ": every class id must map to car, pedestrian "
                                                "or cyclist");
    map.bits |= (uint32_t)(k + 1) << (2 * class_map[k]);
  }
  if (line_capacity < 0 || (line_capacity && !lines))
    return fail(SQDET_ERR_INVALID_ARG, name + ": need line_capacity >= 0 and lines for it");
  if ((uintptr_t)lines % alignof(double))
    return fail(SQDET_ERR_INVALID_ARG, name + ": misaligned argument");
  if (scratch_bytes_ < analyze_scratch_bytes(n, max_dets, n_objects))
    return fail(SQDET_ERR_INVALID_ARG,
                name + ": scratch_bytes is below sqdet_kitti_analyze_scratch_bytes");
  const int device = inputs_device(n, max_dets, dets, counts, objs, offsets, n_objects, scratch,
                                   scratch_bytes_);
  if (device < 0 || !device_range_ok(out, sizeof(sqdet_kitti_analysis), device) ||
      (line_capacity &&
       !device_range_ok(lines, line_capacity * (int64_t)sizeof(sqdet_kitti_error_line), device)))
    return fail(SQDET_ERR_INVALID_ARG, name + ": dets, counts, objs, offsets, scratch, out and "
                                              "lines must each lie inside one allocation on one "
                                              "device");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select the records' device");
  cudaStream_t st = (cudaStream_t)stream;
  Carver c{static_cast<uint8_t*>(scratch)};
  const AnalyzeScratch s = carve_analyze(c, n, max_dets, n_objects);
  SQ_CUDA(cudaMemsetAsync(out, 0, sizeof(sqdet_kitti_analysis), st));
  SQ_CUDA(cudaMemsetAsync(&out->status, 0xff, sizeof(out->status), st));
  rank_kernel<<<n, kAnalyzeThreads, 0, st>>>(dets, counts, objs, offsets, n_objects, max_dets,
                                             classes, map, s, out);
  SQ_CHECK_LAUNCH("kitti rank_kernel");
  line_scan_kernel<<<1, 1024, 0, st>>>(n, s, out);
  SQ_CHECK_LAUNCH("kitti line_scan_kernel");
  line_kernel<<<n, kAnalyzeThreads, 0, st>>>(objs, offsets, n_objects, max_dets, map, s, lines,
                                             line_capacity);
  SQ_CHECK_LAUNCH("kitti line_kernel");
  return SQDET_OK;
}
