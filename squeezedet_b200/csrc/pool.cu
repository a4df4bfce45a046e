// NHWC max-pool and residual add+relu: pure-bandwidth kernels, 128-bit vectorised.
//
// Replaces tf.nn.max_pool (reference src/nn_skeleton.py:580-583; SAME never reads the
// padding: out-of-image taps are skipped, which equals a -inf pad) and
// tf.nn.relu(a + b) (src/nets/resnet50_convDet.py:55).
// Roofline: HBM.  Algorithmic bytes = 4*(B*H*W*C + B*Ho*Wo*C); each input element is
// read ~(k/stride)^2 times but the re-reads hit L1/L2 (adjacent threads share rows).
#include <math_constants.h>

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

}  // namespace

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
