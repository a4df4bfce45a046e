// uint8 frames in any SQDET_FMT_* pixel format -> fp32 tensor 0: each crop converted to BGR as the
// format's cv2.cvtColor code does, then cv2.resize (float32, INTER_LINEAR) and the mean
// subtraction, bit for bit, in one batched launch per frames_per_launch(P) frames.  No BGR frame
// is written: each tap is fetched from the frame's planes and converted.
//
// One kernel template over the format code: taps<F> (frames.cuh, shared with jpeg.cu) picks the
// fetch from a FrameDesc<P> of the format's P planes, and resize_meansub_pixel does the arithmetic
// every format shares.
//
// It also owns the checks that frames and buffers coming from the caller get before any device
// work (accept_frames, device_range_ok), which every entry point taking device frames shares.
#include <cuda.h>

#include "frames.cuh"

namespace sqdet {

const PixFormat* pix_format(int format) {
  static_assert(SQDET_FMT_BGR == 0 && SQDET_FMT_RGB == 1 && SQDET_FMT_BGRA == 2 &&
                    SQDET_FMT_RGBA == 3 && SQDET_FMT_RGB_PLANAR == 4 && SQDET_FMT_NV12 == 5 &&
                    SQDET_FMT_I420 == 6,
                "the table is indexed by SQDET_FMT_*");
  static const PixFormat table[] = {
      {1, false, "3 * width", {{3, 0, 0}}},                                       // BGR
      {1, false, "3 * width", {{3, 0, 0}}},                                       // RGB
      {1, false, "4 * width", {{4, 0, 0}}},                                       // BGRA
      {1, false, "4 * width", {{4, 0, 0}}},                                       // RGBA
      {3, false, "the width", {{1, 0, 0}, {1, 0, 0}, {1, 0, 0}}},                 // RGB_PLANAR
      {2, true, "the width", {{1, 0, 0}, {2, 1, 1}}},                             // NV12
      {3, true, "the width (Y) or half of it (U, V)", {{1, 0, 0}, {1, 1, 1}, {1, 1, 1}}},  // I420
  };
  return format >= 0 && format < (int)(sizeof table / sizeof table[0]) ? &table[format] : nullptr;
}

namespace {

// cv2.resize (float32, INTER_LINEAR) and the mean subtraction, in the reference's two orders
// (src/demo.py:187-190: resize, then `- BGR_MEANS` in float64; src/dataset/imdb.py:87-91: float32
// `-= BGR_MEANS`, then resize).  Restates oracle/preproc.py
// operation for operation (double sampling position, float32 weight, clamps, horizontal pass then
// vertical pass, round-to-nearest multiplies and adds, no contraction).
// Output pixel (dx, dy) of one H0 x W0 frame whose source pixels `taps` fetches:
// taps(ys, xs, r, q, c) is channel c (B, G, R) of source pixel (ys[r], xs[q]), asked for channel 0
// of every tap first.
template <class Taps>
__device__ __forceinline__ void resize_meansub_pixel(const Taps& taps, int H0, int W0, int H, int W,
                                                     double scale_x, double scale_y,
                                                     const double (&mean)[3], int sub_first, int dx,
                                                     int dy, float* __restrict__ d) {
  int sx, sx1, y0, y1;
  float fx, fy;
  bool x_edge = false;
  if (W == W0 && H == H0) {                    // cv2.resize returns a copy for equal sizes
    sx = sx1 = dx; y0 = y1 = dy; fx = 0.f; fy = 0.f; x_edge = true;
  } else {
    // explicit round-to-nearest ops: an FMA contraction here could move a sampling position
    // across an integer relative to the restatement
    const double px = __dsub_rn(__dmul_rn(__dadd_rn((double)dx, 0.5), scale_x), 0.5);
    const double py = __dsub_rn(__dmul_rn(__dadd_rn((double)dy, 0.5), scale_y), 0.5);
    const double flx = floor(px), fly = floor(py);
    sx = (int)flx;
    fx = (float)(px - flx);
    if (sx < 0) { sx = 0; fx = 0.f; }
    if (sx >= W0 - 1) { sx = W0 - 1; fx = 0.f; x_edge = true; }
    sx1 = min(sx + 1, W0 - 1);
    const int sy = (int)fly;
    fy = (float)(py - fly);
    y0 = min(max(sy, 0), H0 - 1);
    y1 = min(max(sy + 1, 0), H0 - 1);
  }
  const float a0 = __fsub_rn(1.f, fx), a1 = fx, b0 = __fsub_rn(1.f, fy), b1 = fy;
  const bool same = (W == W0 && H == H0);
  float o[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float t[2][2];
    const int ys[2] = {y0, y1}, xs[2] = {sx, sx1};
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float v = taps(ys, xs, r, q, c);
        t[r][q] = sub_first ? (float)((double)v - mean[c]) : v;
      }
    float row[2];
#pragma unroll
    for (int r = 0; r < 2; ++r)
      row[r] = x_edge ? t[r][0] : __fadd_rn(__fmul_rn(t[r][0], a0), __fmul_rn(t[r][1], a1));
    const float v = same ? row[0] : __fadd_rn(__fmul_rn(row[0], b0), __fmul_rn(row[1], b1));
    o[c] = sub_first ? v : (float)((double)v - mean[c]);
  }
  d[0] = o[0]; d[1] = o[1]; d[2] = o[2];
}

// Frames per launch: the descriptors travel in the parameter block (no device table, no copy, no
// host synchronisation), and these many of them with the kernel's other 56 bytes of parameters
// fill the classic 4 KiB block.  sqdet_b200.h documents them.
constexpr int frames_per_launch(int planes) { return planes == 1 ? 64 : planes == 2 ? 56 : 45; }

template <int F>
struct FrameBatch {
  FrameDesc<kPlanes<F>> f[frames_per_launch(kPlanes<F>)];
};
static_assert(sizeof(FrameDesc<1>) == 56 && sizeof(FrameDesc<2>) == 72 && sizeof(FrameDesc<3>) == 88,
              "descriptor sizes");
static_assert(sizeof(FrameBatch<SQDET_FMT_BGR>) + 64 <= 4096 &&
                  sizeof(FrameBatch<SQDET_FMT_NV12>) + 64 <= 4096 &&
                  sizeof(FrameBatch<SQDET_FMT_I420>) + 64 <= 4096,
              "frame descriptors exceed 4 KiB of parameters");

// Up to the batch's frame count in one launch: blockIdx.y is the frame, x runs over its H x W
// output pixels, written as image blockIdx.y of the fp32 [count, H, W, 3] batch at dst.  With
// scales_xy, the frame's (x_scale, y_scale) box scales go to scales_xy[2 * frame].
template <int F>
__global__ void __launch_bounds__(256)
resize_meansub_u8_batch_kernel(const __grid_constant__ FrameBatch<F> batch, float* __restrict__ dst,
                               int H, int W, double m0, double m1, double m2, int sub_first,
                               float* __restrict__ scales_xy) {
  const auto& f = batch.f[blockIdx.y];
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (scales_xy && idx == 0) {
    scales_xy[2 * blockIdx.y] = f.box_scale_x;
    scales_xy[2 * blockIdx.y + 1] = f.box_scale_y;
  }
  if (idx >= (long long)H * W) return;
  const double mean[3] = {m0, m1, m2};
  resize_meansub_pixel(taps<F>(f), f.h, f.w, H, W, f.scale_x, f.scale_y, mean, sub_first,
                       (int)(idx % W), (int)(idx / W),
                       dst + ((long long)blockIdx.y * H * W + idx) * 3);
}

template <int F>
int launch_format(const PixFormat& pf, const FrameSource* frames, int n, float* dst, int H, int W,
                  unsigned blocks, const double* means, int sub_first, float* scales_xy,
                  cudaStream_t stream) {
  constexpr int P = kPlanes<F>, per_launch = frames_per_launch(P);
  const size_t pixels = (size_t)H * W;
  for (int g = 0; g < n; g += per_launch) {
    const int count = std::min(n - g, per_launch);
    FrameBatch<F> batch;
    for (int i = 0; i < count; ++i) batch.f[i] = frame_desc<P>(pf, frames[g + i], H, W);
    resize_meansub_u8_batch_kernel<F><<<dim3(blocks, (unsigned)count), 256, 0, stream>>>(
        batch, dst + (size_t)g * pixels * 3, H, W, means[0], means[1], means[2], sub_first,
        scales_xy ? scales_xy + 2 * g : nullptr);
    SQ_CHECK_LAUNCH("resize_meansub_u8_batch_kernel");
  }
  return SQDET_OK;
}

}  // namespace

int launch_resize_meansub_frames(int format, const FrameSource* frames, int n, float* dst, int H,
                                 int W, const double* means, int sub_first, float* scales_xy,
                                 cudaStream_t stream) {
  const PixFormat* pf = pix_format(format);
  if (!pf) return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_frames: unknown format");
  if (n <= 0 || H <= 0 || W <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_frames: non-positive image size");
  for (int i = 0; i < n; ++i)
    if (frames[i].h <= 0 || frames[i].w <= 0)
      return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_frames: non-positive crop size");
  const long long blocks = ((long long)H * W + 255) / 256;
  if (blocks > 0x7fffffffLL) return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_frames: image too large");
  return dispatch_format(format, [&](auto f) {
    return launch_format<decltype(f)::value>(*pf, frames, n, dst, H, W, (unsigned)blocks, means,
                                             sub_first, scales_xy, stream);
  });
}

// ---- frames and buffers from the caller ----------------------------------------------------------
int pointer_device(const void* p) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) == cudaSuccess && attr.type == cudaMemoryTypeDevice)
    return attr.device;
  (void)cudaGetLastError();      // an unknown pointer: no stale error for the next launch check
  return -1;
}

using MemGetAddressRangeFn = CUresult (*)(CUdeviceptr*, size_t*, CUdeviceptr);

bool device_range_ok(const void* p, int64_t bytes, int device) {
  static MemGetAddressRangeFn range = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      fn = nullptr;
    return reinterpret_cast<MemGetAddressRangeFn>(fn);
  }();
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
    (void)cudaGetLastError();      // an unknown pointer: no stale error for the next launch check
    return false;
  }
  if (attr.type != cudaMemoryTypeDevice || attr.device != device || !range) return false;
  CUdeviceptr base = 0;
  size_t size = 0;
  if (range(&base, &size, (CUdeviceptr)(uintptr_t)p) != CUDA_SUCCESS) return false;
  const uint64_t off = (uint64_t)(uintptr_t)p - (uint64_t)base;
  return off <= size && (uint64_t)bytes <= size - off;
}

int check_crop(const std::string& which, int64_t H, int64_t W, const int32_t* r, FrameSource& s) {
  s.x = r ? r[0] : 0;
  s.y = r ? r[1] : 0;
  s.w = r ? r[2] : (int)W;
  s.h = r ? r[3] : (int)H;
  if (s.w <= 0 || s.h <= 0) return fail(SQDET_ERR_INVALID_ARG, which + ": empty crop");
  if (s.x < 0 || s.y < 0 || (int64_t)s.x + s.w > W || (int64_t)s.y + s.h > H)
    return fail(SQDET_ERR_INVALID_ARG, which + ": crop outside the frame");
  return SQDET_OK;
}

int encode_crops(const std::string& name, const Encoder& enc, int n, const int32_t* heights,
                 const int32_t* widths, const int32_t* crops, std::vector<FrameSource>& fr) {
  if (!heights || !widths) return fail(SQDET_ERR_INVALID_ARG, name + ": null argument");
  if (n < 1 || n > enc.max_frames)
    return fail(SQDET_ERR_INVALID_ARG, name + ": n must be in [1, " + std::to_string(enc.max_frames) + "]");
  fr.assign((size_t)n, FrameSource{});
  for (int i = 0; i < n; ++i) {
    const std::string which = name + ": frame " + std::to_string(i);
    if (heights[i] <= 0 || widths[i] <= 0) return fail(SQDET_ERR_INVALID_ARG, which + " is empty");
    const int rc = check_crop(which, heights[i], widths[i], crops ? crops + 4 * i : nullptr, fr[(size_t)i]);
    if (rc) return rc;
    if (fr[(size_t)i].w > enc.max_side || fr[(size_t)i].h > enc.max_side)
      return fail(SQDET_ERR_INVALID_ARG, which + ": a " + enc.file + " is at most " +
                                             std::to_string(enc.max_side) + " pixels wide and high");
  }
  return SQDET_OK;
}

int accept_frames(const std::string& name, const PixFormat& pf, int n,
                  const uint8_t* const* planes, const int64_t* pitches, const int32_t* heights,
                  const int32_t* widths, const int32_t* crops,
                  const std::function<std::string(int)>& image, int* device,
                  std::vector<FrameSource>& fr) {
  auto which = [&](int i) { return name + ": " + (image ? image(i) : "frame " + std::to_string(i)); };
  fr.assign((size_t)n, FrameSource{});
  for (int i = 0; i < n; ++i) {
    const int64_t H = heights[i], W = widths[i];
    const std::string what = which(i);
    FrameSource& s = fr[(size_t)i];
    for (int p = 0; p < pf.planes; ++p) {
      s.plane[p] = planes[3 * (size_t)i + p];
      if (!s.plane[p])
        return fail(SQDET_ERR_INVALID_ARG, what + (pf.planes == 1 ? " is a null pointer" : " has a null plane"));
    }
    if (pf.even && (H <= 0 || W <= 0 || H % 2 || W % 2))
      return fail(SQDET_ERR_INVALID_ARG, what + ": height and width must be positive and even");
    if (H <= 0 || W <= 0) return fail(SQDET_ERR_INVALID_ARG, what + " is empty");
    for (int p = 0; p < pf.planes; ++p) {
      s.pitch[p] = pitches ? pitches[3 * (size_t)i + p] : pf.plane[p].row_bytes(W);
      if (s.pitch[p] < pf.plane[p].row_bytes(W))
        return fail(SQDET_ERR_INVALID_ARG, what + ": row pitch below " + pf.least_pitch);
    }
    const int rc = check_crop(what, H, W, crops ? crops + 4 * (size_t)i : nullptr, s);
    if (rc) return rc;
  }
  const char* where = *device == kFrame0Device ? "frame 0's device" : "the engine's device";
  if (*device == kFrame0Device) *device = pointer_device(fr[0].plane[0]);
  for (int i = 0; i < n; ++i) {
    const FrameSource& s = fr[(size_t)i];
    for (int p = 0; p < pf.planes; ++p) {
      // the plane's bytes end at (rows - 1) * pitch + row bytes; refused when that overflows int64
      const int64_t k = (int64_t)heights[i] >> pf.plane[p].y_shift, b = pf.plane[p].row_bytes(widths[i]);
      const bool fits = k == 1 || s.pitch[p] <= (INT64_MAX - b) / (k - 1);
      if (!fits || !device_range_ok(s.plane[p], (k - 1) * s.pitch[p] + b, *device))
        return fail(SQDET_ERR_INVALID_ARG,
                    which(i) + (pf.planes == 1 ? " is not inside" : ": a plane is not inside") +
                        " one device allocation on " + where);
    }
  }
  return SQDET_OK;
}

}  // namespace sqdet
