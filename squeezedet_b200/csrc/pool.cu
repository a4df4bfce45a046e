// NHWC max-pool and residual add+relu: pure-bandwidth kernels, 128-bit vectorised.
//
// Replaces tf.nn.max_pool (reference src/nn_skeleton.py:580-583; SAME never reads the
// padding: out-of-image taps are skipped, which equals a -inf pad) and
// tf.nn.relu(a + b) (src/nets/resnet50_convDet.py:55).
// Roofline: HBM.  Algorithmic bytes = 4*(B*H*W*C + B*Ho*Wo*C); each input element is
// read ~(k/stride)^2 times but the re-reads hit L1/L2 (adjacent threads share rows).
#include <math_constants.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace sqdet {
namespace {

__device__ __forceinline__ float4 ld_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

// One thread = one output pixel x 4 channels.
__global__ void __launch_bounds__(256)
maxpool_vec4_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W,
                    int C4, int k, int stride, int pad_t, int pad_l, int Ho, int Wo) {
  const long long total = (long long)B * Ho * Wo * C4;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(idx % C4);
    long long t = idx / C4;
    const int ow = (int)(t % Wo);
    t /= Wo;
    const int oh = (int)(t % Ho);
    const int n = (int)(t / Ho);
    const int iy0 = oh * stride - pad_t, ix0 = ow * stride - pad_l;
    float4 m = make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F);
    const float4* xin = reinterpret_cast<const float4*>(x) + (long long)n * H * W * C4;
    for (int u = 0; u < k; ++u) {
      const int iy = iy0 + u;
      if (iy < 0 || iy >= H) continue;
      for (int v = 0; v < k; ++v) {
        const int ix = ix0 + v;
        if (ix < 0 || ix >= W) continue;
        const float4 q = __ldg(xin + ((long long)iy * W + ix) * C4 + c4);
        m.x = fmaxf(m.x, q.x); m.y = fmaxf(m.y, q.y);
        m.z = fmaxf(m.z, q.z); m.w = fmaxf(m.w, q.w);
      }
    }
    reinterpret_cast<float4*>(y)[idx] = m;
  }
}

// Stride-2 windows of 2x2 or 3x3 (every pool of the four nets): all K*K loads of a thread are
// issued before the first max (addresses clamped into the image, out-of-image taps replaced by -inf
// afterwards), 32-bit index arithmetic.  The generic kernel below branches around each tap, which
// serialises its loads.
template <int K>
__global__ void __launch_bounds__(256)
maxpool_s2_vec4_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W,
                       int C4, int pad_t, int pad_l, int Ho, int Wo) {
  const int total = B * Ho * Wo * C4;
  const float4* __restrict__ x4 = reinterpret_cast<const float4*>(x);
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int c4 = idx % C4;
    int t = idx / C4;
    const int ow = t % Wo;
    t /= Wo;
    const int oh = t % Ho;
    const int n = t / Ho;
    const int iy0 = oh * 2 - pad_t, ix0 = ow * 2 - pad_l;
    const int base = n * H * W;
    float4 q[K * K];
#pragma unroll
    for (int u = 0; u < K; ++u) {
      const int iy = min(max(iy0 + u, 0), H - 1);
#pragma unroll
      for (int v = 0; v < K; ++v) {
        const int ix = min(max(ix0 + v, 0), W - 1);
        q[u * K + v] = __ldg(x4 + (size_t)(base + iy * W + ix) * C4 + c4);
      }
    }
    float4 m = make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F);
#pragma unroll
    for (int u = 0; u < K; ++u)
#pragma unroll
      for (int v = 0; v < K; ++v) {
        const bool ok = (unsigned)(iy0 + u) < (unsigned)H && (unsigned)(ix0 + v) < (unsigned)W;
        const float4 r = q[u * K + v];
        if (ok) {
          m.x = fmaxf(m.x, r.x); m.y = fmaxf(m.y, r.y);
          m.z = fmaxf(m.z, r.z); m.w = fmaxf(m.w, r.w);
        }
      }
    reinterpret_cast<float4*>(y)[idx] = m;
  }
}

__global__ void __launch_bounds__(256)
maxpool_scalar_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W,
                      int C, int k, int stride, int pad_t, int pad_l, int Ho, int Wo) {
  const long long total = (long long)B * Ho * Wo * C;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    long long t = idx / C;
    const int ow = (int)(t % Wo);
    t /= Wo;
    const int oh = (int)(t % Ho);
    const int n = (int)(t / Ho);
    const int iy0 = oh * stride - pad_t, ix0 = ow * stride - pad_l;
    float m = -CUDART_INF_F;
    for (int u = 0; u < k; ++u) {
      const int iy = iy0 + u;
      if (iy < 0 || iy >= H) continue;
      for (int v = 0; v < k; ++v) {
        const int ix = ix0 + v;
        if (ix < 0 || ix >= W) continue;
        m = fmaxf(m, __ldg(x + (((long long)n * H + iy) * W + ix) * C + c));
      }
    }
    y[idx] = m;
  }
}

__global__ void __launch_bounds__(256)
add_relu_kernel(const float* __restrict__ a, const float* __restrict__ b,
                float* __restrict__ y, long long n4, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n4) {
    const float4 p = ld_stream(reinterpret_cast<const float4*>(a) + i);
    const float4 q = ld_stream(reinterpret_cast<const float4*>(b) + i);
    float4 r;
    r.x = fmaxf(p.x + q.x, 0.f); r.y = fmaxf(p.y + q.y, 0.f);
    r.z = fmaxf(p.z + q.z, 0.f); r.w = fmaxf(p.w + q.w, 0.f);
    reinterpret_cast<float4*>(y)[i] = r;
  }
  if (i == 0) {  // tail (n not a multiple of 4)
    for (long long j = n4 * 4; j < n; ++j) y[j] = fmaxf(a[j] + b[j], 0.f);
  }
}

// uint8 BGR [H0, W0, 3] -> fp32 [H, W, 3]: cv2.resize (float32, INTER_LINEAR) and the mean
// subtraction, in the reference's two orders (src/demo.py:187-190: resize, then `- BGR_MEANS`
// in float64; src/dataset/imdb.py:87-91: float32 `-= BGR_MEANS`, then resize).  Restates
// oracle/preproc.py operation for operation (double sampling position, float32 weight, clamps,
// horizontal pass then vertical pass, round-to-nearest multiplies and adds, no contraction).
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

// The taps of a packed uint8 frame of kBpp bytes per pixel whose row r starts at src + r * pitch
// (any byte alignment), with B, G, R at byte offsets kB, kG, kR of a pixel (other bytes, such as
// alpha, are never read): a channel is a byte load served by L1.  The layout is a compile-time
// instance, so a tap costs the same address arithmetic as BGR's.
template <int kBpp, int kB, int kG, int kR>
struct PackedTaps {
  const uint8_t* __restrict__ src;
  long long pitch;
  __device__ __forceinline__ float operator()(const int (&ys)[2], const int (&xs)[2], int r, int q,
                                             int c) const {
    return (float)src[(long long)ys[r] * pitch + (long long)xs[q] * kBpp +
                      (c == 0 ? kB : c == 1 ? kG : kR)];
  }
};
using BgrTaps = PackedTaps<3, 0, 1, 2>;

// The taps of three uint8 planes holding R, G and B (torch's [3, h, w] image layout): channel c
// (B, G, R) of pixel (y, x) is byte x of row y of plane 2 - c, each plane at any byte and pitch.
struct PlanarTaps {
  const uint8_t* __restrict__ plane[3];
  long long pitch[3];
  __device__ __forceinline__ float operator()(const int (&ys)[2], const int (&xs)[2], int r, int q,
                                             int c) const {
    return (float)plane[2 - c][(long long)ys[r] * pitch[2 - c] + xs[q]];
  }
};

// The taps of a YUV 4:2:0 crop: one luma byte and the U,V samples of its 2x2 chroma block,
// converted as cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420) does (OpenCV's BT.601 limited-range
// ITUR_BT_601_* constants, 20 fraction bits; oracle.nv12.nv12_to_bgr).  kInterleaved: NV12, one
// chroma plane of U,V pairs at u; otherwise I420, separate U and V planes of half the width.
// Crop pixel (y, x) is frame pixel (y0 + y, x0 + x); luma and the chroma planes point at the crop
// origin's byte and chroma sample, and the origin's parity (x_odd, y_odd) picks the chroma block,
// so an odd origin reads the frame's own samples.  int32 suffices: every sum stays below 2^30 in
// magnitude.  Each tap is loaded and converted once, when its channel 0 is asked for.
template <bool kInterleaved>
struct Yuv420Taps {
  const uint8_t* __restrict__ luma;
  const uint8_t* __restrict__ u_plane;
  long long luma_pitch, u_pitch;
  int x_odd, y_odd;
  mutable float bgr[2][2][3];   // tap (r, q), converted at its channel 0
  // I420's V plane, last: with it after the fields NV12 uses, the NV12 instance compiles to the
  // code it had before I420 shared this struct
  const uint8_t* __restrict__ v_plane;
  long long v_pitch;
  __device__ __forceinline__ float operator()(const int (&ys)[2], const int (&xs)[2], int r, int q,
                                             int c) const {
    if (c == 0) {
      const int y = ys[r], x = xs[q];
      const int Y = luma[(long long)y * luma_pitch + x];
      const long long cy = (long long)((y + y_odd) >> 1);
      int u, v;
      if (kInterleaved) {
        const uint8_t* uv = u_plane + cy * u_pitch + ((x + x_odd) & ~1);
        u = (int)uv[0] - 128;
        v = (int)uv[1] - 128;
      } else {
        u = (int)u_plane[cy * u_pitch + ((x + x_odd) >> 1)] - 128;
        v = (int)v_plane[cy * v_pitch + ((x + x_odd) >> 1)] - 128;
      }
      const int yy = max(Y - 16, 0) * 1220542 + (1 << 19);
      bgr[r][q][0] = (float)min(max((yy + 2116026 * u) >> 20, 0), 255);
      bgr[r][q][1] = (float)min(max((yy - 852492 * v - 409993 * u) >> 20, 0), 255);
      bgr[r][q][2] = (float)min(max((yy + 1673527 * v) >> 20, 0), 255);
    }
    return bgr[r][q][c];
  }
};

// A packed RGB, BGRA or RGBA frame: ResizeFrame's descriptor, typed by its layout.
template <int kBpp, int kB, int kG, int kR>
struct PackedFrame : ResizeFrame {};
using RgbFrame = PackedFrame<3, 2, 1, 0>;
using BgraFrame = PackedFrame<4, 0, 1, 2>;
using RgbaFrame = PackedFrame<4, 2, 1, 0>;
// The h x w crop of a planar RGB or an I420 frame: plane[p] points at the crop origin's sample of
// plane p, and (x_odd, y_odd), the origin's parity, picks I420's chroma block.  88 bytes.
struct ThreePlaneFrame {
  const uint8_t* plane[3];
  int64_t pitch[3];
  double scale_x, scale_y;
  float box_scale_x, box_scale_y;
  int h, w;
  int x_odd, y_odd;
};
// Frames per launch: 45 descriptors of 88 bytes and the kernel's other parameters fill the
// classic 4 KiB parameter block.
constexpr int kThreePlaneFramesPerLaunch = 45;
struct PlanarFrame : ThreePlaneFrame {};
struct I420Frame : ThreePlaneFrame {};

__device__ __forceinline__ BgrTaps taps(const ResizeFrame& f) { return {f.src, f.pitch}; }
template <int kBpp, int kB, int kG, int kR>
__device__ __forceinline__ PackedTaps<kBpp, kB, kG, kR> taps(const PackedFrame<kBpp, kB, kG, kR>& f) {
  return {f.src, f.pitch};
}
__device__ __forceinline__ Yuv420Taps<true> taps(const Nv12Frame& f) {
  return {f.luma, f.chroma, f.luma_pitch, f.chroma_pitch, f.x_odd, f.y_odd, {}, nullptr, 0};
}
__device__ __forceinline__ PlanarTaps taps(const PlanarFrame& f) {
  return {{f.plane[0], f.plane[1], f.plane[2]}, {f.pitch[0], f.pitch[1], f.pitch[2]}};
}
__device__ __forceinline__ Yuv420Taps<false> taps(const I420Frame& f) {
  return {f.plane[0], f.plane[1], f.pitch[0], f.pitch[1], f.x_odd, f.y_odd, {}, f.plane[2],
          f.pitch[2]};
}

struct ResizeFrameBatch {
  ResizeFrame f[kResizeFramesPerLaunch];
};
struct Nv12FrameBatch {
  Nv12Frame f[kNv12FramesPerLaunch];
};
template <class Frame>
struct PackedFrameBatch {
  Frame f[kResizeFramesPerLaunch];
};
template <class Frame>
struct ThreePlaneFrameBatch {
  Frame f[kThreePlaneFramesPerLaunch];
};
// Descriptors travel in the parameter block: no device table, no copy, no host synchronisation.
static_assert(sizeof(ResizeFrameBatch) + 128 <= 4096, "resize descriptors exceed 4 KiB of parameters");
// The kernel's other parameters take 56 bytes.
static_assert(sizeof(Nv12FrameBatch) + 64 <= 4096, "NV12 descriptors exceed 4 KiB of parameters");
static_assert(sizeof(PackedFrameBatch<RgbaFrame>) == sizeof(ResizeFrameBatch),
              "packed descriptors are ResizeFrame's");
static_assert(sizeof(ThreePlaneFrameBatch<I420Frame>) + 64 <= 4096,
              "three-plane descriptors exceed 4 KiB of parameters");

// Up to the batch's frame count in one launch: blockIdx.y is the frame, x runs over its H x W
// output pixels, written as image blockIdx.y of the fp32 [count, H, W, 3] batch at dst.  With
// scales_xy, the frame's (x_scale, y_scale) box scales go to scales_xy[2 * frame].
template <class Batch>
__global__ void __launch_bounds__(256)
resize_meansub_u8_batch_kernel(const __grid_constant__ Batch batch, float* __restrict__ dst, int H,
                               int W, double m0, double m1, double m2, int sub_first,
                               float* __restrict__ scales_xy) {
  const auto& f = batch.f[blockIdx.y];
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (scales_xy && idx == 0) {
    scales_xy[2 * blockIdx.y] = f.box_scale_x;
    scales_xy[2 * blockIdx.y + 1] = f.box_scale_y;
  }
  if (idx >= (long long)H * W) return;
  const double mean[3] = {m0, m1, m2};
  resize_meansub_pixel(taps(f), f.h, f.w, H, W, f.scale_x, f.scale_y, mean, sub_first,
                       (int)(idx % W), (int)(idx / W),
                       dst + ((long long)blockIdx.y * H * W + idx) * 3);
}

// The frames in launches of the batch's frame count each (the frames' own checks are the
// caller's); `what` names the kernel in errors.
template <class Batch, class Frame>
int launch_batches(const char* what, const Frame* frames, int n, float* dst, int H, int W,
                   const double* means, int sub_first, float* scales_xy, cudaStream_t stream) {
  constexpr int per_launch = (int)(sizeof(Batch) / sizeof(Frame));
  const long long pixels = (long long)H * W;
  const long long blocks = (pixels + 255) / 256;
  if (blocks > 0x7fffffffLL) return fail(SQDET_ERR_INVALID_ARG, std::string(what) + ": image too large");
  for (int g = 0; g < n; g += per_launch) {
    const int count = std::min(n - g, per_launch);
    Batch batch;
    for (int i = 0; i < count; ++i) batch.f[i] = frames[g + i];
    resize_meansub_u8_batch_kernel<<<dim3((unsigned)blocks, (unsigned)count), 256, 0, stream>>>(
        batch, dst + (size_t)g * pixels * 3, H, W, means[0], means[1], means[2], sub_first,
        scales_xy ? scales_xy + 2 * g : nullptr);
    SQ_CHECK_LAUNCH(what);
  }
  return SQDET_OK;
}

}  // namespace

ResizeFrame resize_frame(const uint8_t* src, int64_t pitch, int h, int w, int H, int W) {
  ResizeFrame f;
  f.src = src;
  f.pitch = pitch;
  f.h = h;
  f.w = w;
  // cv::resize: inv_scale = dst / src, scale = 1 / inv_scale (both double)
  f.scale_x = 1.0 / ((double)W / (double)w);
  f.scale_y = 1.0 / ((double)H / (double)h);
  // eval.py:72-74 / imdb.py:93-95: x_scale = mc.IMAGE_WIDTH / orig_w (Python floats = double)
  f.box_scale_x = (float)((double)W / (double)w);
  f.box_scale_y = (float)((double)H / (double)h);
  return f;
}

Nv12Frame nv12_frame(const uint8_t* luma, int64_t luma_pitch, const uint8_t* chroma,
                     int64_t chroma_pitch, int x, int y, int h, int w, int H, int W) {
  const ResizeFrame r = resize_frame(nullptr, 0, h, w, H, W);
  Nv12Frame f;
  f.luma = luma + (int64_t)y * luma_pitch + x;
  f.chroma = chroma + (int64_t)(y >> 1) * chroma_pitch + (x & ~1);
  f.luma_pitch = luma_pitch;
  f.chroma_pitch = chroma_pitch;
  f.scale_x = r.scale_x;
  f.scale_y = r.scale_y;
  f.box_scale_x = r.box_scale_x;
  f.box_scale_y = r.box_scale_y;
  f.h = h;
  f.w = w;
  f.x_odd = x & 1;
  f.y_odd = y & 1;
  return f;
}

int launch_resize_meansub_u8_batch(const ResizeFrame* frames, int n, float* dst, int H, int W,
                                   const double* means, int sub_first, float* scales_xy,
                                   cudaStream_t stream) {
  if (n <= 0 || H <= 0 || W <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_u8: non-positive image size");
  for (int i = 0; i < n; ++i)
    if (frames[i].h <= 0 || frames[i].w <= 0)
      return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_u8: non-positive image size");
    else if (frames[i].pitch < 3 * (int64_t)frames[i].w)
      return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_u8: row pitch below 3 * width");
  return launch_batches<ResizeFrameBatch>("resize_meansub_u8_batch_kernel", frames, n, dst, H, W,
                                          means, sub_first, scales_xy, stream);
}

int launch_resize_meansub_nv12_batch(const Nv12Frame* frames, int n, float* dst, int H, int W,
                                     const double* means, int sub_first, float* scales_xy,
                                     cudaStream_t stream) {
  if (n <= 0 || H <= 0 || W <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_nv12: non-positive image size");
  for (int i = 0; i < n; ++i)
    if (frames[i].h <= 0 || frames[i].w <= 0)
      return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_nv12: non-positive crop size");
    else if (frames[i].luma_pitch < frames[i].w || frames[i].chroma_pitch < frames[i].w)
      return fail(SQDET_ERR_INVALID_ARG, "resize_meansub_nv12: row pitch below the crop width");
  return launch_batches<Nv12FrameBatch>("resize_meansub_u8_batch_kernel<Nv12FrameBatch>", frames,
                                        n, dst, H, W, means, sub_first, scales_xy, stream);
}

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

// The byte of plane p at the origin of frame s's crop.
const uint8_t* crop_origin(const PixFormat& pf, const FrameSource& s, int p) {
  const PixPlane& q = pf.plane[p];
  return s.plane[p] + (int64_t)(s.y >> q.y_shift) * s.pitch[p] +
         (int64_t)(s.x >> q.x_shift) * q.bytes_per_px;
}

template <class Frame>
int launch_packed(const char* what, const PixFormat& pf, const FrameSource* s, int n, float* dst,
                  int H, int W, const double* means, int sub_first, float* scales_xy,
                  cudaStream_t stream) {
  std::vector<Frame> fr((size_t)n);
  for (int i = 0; i < n; ++i)
    static_cast<ResizeFrame&>(fr[(size_t)i]) =
        resize_frame(crop_origin(pf, s[i], 0), s[i].pitch[0], s[i].h, s[i].w, H, W);
  return launch_batches<PackedFrameBatch<Frame>>(what, fr.data(), n, dst, H, W, means, sub_first,
                                                 scales_xy, stream);
}

template <class Frame>
int launch_three_plane(const char* what, const PixFormat& pf, const FrameSource* s, int n,
                       float* dst, int H, int W, const double* means, int sub_first,
                       float* scales_xy, cudaStream_t stream) {
  std::vector<Frame> fr((size_t)n);
  for (int i = 0; i < n; ++i) {
    const ResizeFrame r = resize_frame(nullptr, 0, s[i].h, s[i].w, H, W);
    Frame& f = fr[(size_t)i];
    for (int p = 0; p < 3; ++p) {
      f.plane[p] = crop_origin(pf, s[i], p);
      f.pitch[p] = s[i].pitch[p];
    }
    f.scale_x = r.scale_x;
    f.scale_y = r.scale_y;
    f.box_scale_x = r.box_scale_x;
    f.box_scale_y = r.box_scale_y;
    f.h = s[i].h;
    f.w = s[i].w;
    f.x_odd = s[i].x & 1;
    f.y_odd = s[i].y & 1;
  }
  return launch_batches<ThreePlaneFrameBatch<Frame>>(what, fr.data(), n, dst, H, W, means,
                                                     sub_first, scales_xy, stream);
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
  const FrameSource* s = frames;
  switch (format) {
    case SQDET_FMT_BGR: {
      std::vector<ResizeFrame> fr((size_t)n);
      for (int i = 0; i < n; ++i)
        fr[(size_t)i] = resize_frame(crop_origin(*pf, s[i], 0), s[i].pitch[0], s[i].h, s[i].w, H, W);
      return launch_resize_meansub_u8_batch(fr.data(), n, dst, H, W, means, sub_first, scales_xy,
                                            stream);
    }
    case SQDET_FMT_NV12: {
      std::vector<Nv12Frame> fr((size_t)n);
      for (int i = 0; i < n; ++i)
        fr[(size_t)i] = nv12_frame(s[i].plane[0], s[i].pitch[0], s[i].plane[1], s[i].pitch[1],
                                   s[i].x, s[i].y, s[i].h, s[i].w, H, W);
      return launch_resize_meansub_nv12_batch(fr.data(), n, dst, H, W, means, sub_first, scales_xy,
                                              stream);
    }
    case SQDET_FMT_RGB:
      return launch_packed<RgbFrame>("resize_meansub_u8_batch_kernel<RGB>", *pf, s, n, dst, H, W,
                                     means, sub_first, scales_xy, stream);
    case SQDET_FMT_BGRA:
      return launch_packed<BgraFrame>("resize_meansub_u8_batch_kernel<BGRA>", *pf, s, n, dst, H, W,
                                      means, sub_first, scales_xy, stream);
    case SQDET_FMT_RGBA:
      return launch_packed<RgbaFrame>("resize_meansub_u8_batch_kernel<RGBA>", *pf, s, n, dst, H, W,
                                      means, sub_first, scales_xy, stream);
    case SQDET_FMT_RGB_PLANAR:
      return launch_three_plane<PlanarFrame>("resize_meansub_u8_batch_kernel<PlanarFrame>", *pf, s,
                                             n, dst, H, W, means, sub_first, scales_xy, stream);
    default:
      return launch_three_plane<I420Frame>("resize_meansub_u8_batch_kernel<I420Frame>", *pf, s, n,
                                           dst, H, W, means, sub_first, scales_xy, stream);
  }
}

int launch_maxpool(const float* x, float* y, int B, int H, int W, int C, int size,
                   int stride, int padding, cudaStream_t stream) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || size <= 0 || stride <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "maxpool: non-positive dimension");
  const Geom gh = tf_geometry(H, size, stride, padding);
  const Geom gw = tf_geometry(W, size, stride, padding);
  if (gh.out <= 0 || gw.out <= 0) return fail(SQDET_ERR_INVALID_ARG, "maxpool: empty output");
  const bool vec = (C % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(y) & 15) == 0);
  const long long total = (long long)B * gh.out * gw.out * (vec ? C / 4 : C);
  long long blocks = (total + 255) / 256;
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long cap = (long long)sms * 8 * 16;   // grid-stride beyond 16 waves of 8 CTAs/SM
  if (blocks > cap) blocks = cap;
  const long long in_elems = (long long)B * H * W * (C / 4);
  if (vec && stride == 2 && (size == 2 || size == 3) && total < (1LL << 30) &&
      in_elems < (1LL << 30))
    (size == 3 ? maxpool_s2_vec4_kernel<3> : maxpool_s2_vec4_kernel<2>)<<<(unsigned)blocks, 256, 0, stream>>>(
        x, y, B, H, W, C / 4, gh.pad_before, gw.pad_before, gh.out, gw.out);
  else if (vec)
    maxpool_vec4_kernel<<<(unsigned)blocks, 256, 0, stream>>>(
        x, y, B, H, W, C / 4, size, stride, gh.pad_before, gw.pad_before, gh.out, gw.out);
  else
    maxpool_scalar_kernel<<<(unsigned)blocks, 256, 0, stream>>>(
        x, y, B, H, W, C, size, stride, gh.pad_before, gw.pad_before, gh.out, gw.out);
  SQ_CHECK_LAUNCH("maxpool_kernel");
  return SQDET_OK;
}

int launch_add_relu(const float* a, const float* b, float* y, int64_t n, cudaStream_t stream) {
  if (n <= 0) return fail(SQDET_ERR_INVALID_ARG, "add_relu: empty tensor");
  const bool aligned = (((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) |
                          reinterpret_cast<uintptr_t>(y)) & 15) == 0);
  const long long n4 = aligned ? n / 4 : 0;
  long long threads = n4 > 0 ? n4 : 1;
  add_relu_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(a, b, y, n4, n);
  SQ_CHECK_LAUNCH("add_relu_kernel");
  return SQDET_OK;
}

}  // namespace sqdet
