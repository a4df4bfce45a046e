// Fused first layer: conv (Cin = 3, k x k, stride 2) + bias [+ frozen BN] + ReLU + 3x3/2
// max-pool in ONE kernel, fp32 FFMA.
//
// Replaces conv1 -> pool1 of every net (reference src/nets/squeezeDet.py:40-44,
// squeezeDetPlus.py:40-44, resnet50_convDet.py:41-46; layer code src/nn_skeleton.py:471-586).
// conv1's output is the largest tensor of the whole network (20 x 188 x 621 x 64 fp32 = 598 MB
// at the benchmark size); unfused it is written once and read once by pool1 (1.2 GB of the
// 4.7 GB a forward pass moves).  Here it never leaves the SM.
//
// K = 27 (or 147) with Cin = 3 is too thin for a tensor-core tile, so it stays on the FFMA pipe:
// exact fp32, same arithmetic as the reference's fp32 conv.
//
// CTA = one strip of strip_h pooled rows x 31 pooled columns of one image, walked top to bottom
// two pooled rows (four new conv rows) per step:
//   conv columns  64 per CTA, one per thread of each 16-channel group (the 64th is never pooled)
//   conv rows     each step computes conv rows 4s+1 .. 4s+4 of the strip (4 rows x 16 channels
//                 per thread); row 4s, shared with the pooled row above, is carried in registers
//                 from the step before (a one-row prologue computes row 0), so only the strip's
//                 first conv row and the 64th column are computed twice
//   vertical max  in registers: pooled row 2s = rows 4s..4s+2, 2s+1 = rows 4s+2..4s+4
//   horizontal    the two vertically pooled rows -> smem, 3-wide max, 128-bit coalesced stores
//   input         the step's 6 + k input rows -> smem with cp.async, issued one step ahead into
//                 the other of two buffers; each row stores even and odd pixels apart, so a
//                 warp's stride-2 pixel reads are unit-stride (3 words) and conflict free
//                 (uint8 input: the 4-byte words holding each row's bytes are staged, then each
//                 warp converts its rows to float32(double(byte) - mean[c]), 0 = pad)
// Threads: 64 per 16-channel group (Cout/16 groups).  Weights [k*k*3][Cout] live in smem.
#include <math_constants.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace sqdet {
namespace {

constexpr int CT_C = 64;                  // conv columns per CTA (one per thread of a group)
constexpr int PT_W = (CT_C - 1) / 2;      // 31 pooled columns: conv columns 0 .. 62
constexpr int NR = 4;                     // conv rows per thread and step: two pooled rows
constexpr int MAX_STRIP = 16;             // pooled rows per CTA, at most
// floats per channel group of s_vert ([2 pooled rows][CT_C][16]); the 16 extra put consecutive
// groups in opposite bank halves for the pool's reads
constexpr int VGS = 2 * CT_C * 16 + 16;

template <int KS>
struct PatchGeom {
  static constexpr int PX = 2 * (CT_C - 1) + KS;   // input pixels of a patch row
  static constexpr int HALF = (PX + 1) / 2;        // even pixels [0, HALF), odd pixels after
  static constexpr int ROWF = 6 * HALF;            // floats per patch row
  static constexpr int ROWS = 2 * (NR - 1) + KS;   // input rows of one step
  static constexpr int BUF = ROWS * ROWF;          // floats per patch buffer
  static constexpr int SW = (PX * 3 + 6) / 4;      // uint8 staging: words per row, any alignment
};

struct ConvPoolParams {
  const float* x;       // [B,H,W,3]
  const float* w;       // [k,k,3,Cout]
  const float* bias;    // [Cout] or null
  const float* scale;   // [Cout] or null
  const float* shift;
  float* y;             // [B,Hp,Wp,Cout]
  int B, H, W, Cout;
  int Hc, Wc;           // conv output size
  int Hp, Wp;           // pooled output size
  int cpad_t, cpad_l;   // conv pad_before
  int ppad_t, ppad_l;   // pool pad_before
  int relu;
  int tiles_w, tiles_h;
  int strip_h;          // pooled rows per CTA (even)
};

// The uint8-input instances' parameters (x unused).
struct ConvPoolU8Params : ConvPoolParams {
  const uint8_t* x8;    // [B,H,W,3] BGR bytes, any byte alignment
  double mean[3];       // subtracted per channel
};

__device__ __forceinline__ void cp_async4(void* dst, const void* src, int nbytes) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(nbytes)
               : "memory");
}

// acc[j][c] = sum over K, in HWIO order from 0, of x * w for conv row j (patch rows 2j .. 2j+KS-1
// from x) and channel c of the thread's group.  x points at the thread's even pixel slot.
template <int KS, int ROWS>
__device__ __forceinline__ void conv_rows(const float* __restrict__ x, const float* __restrict__ wg,
                                          int Cout, float (&acc)[ROWS][16]) {
  using G = PatchGeom<KS>;
#pragma unroll
  for (int j = 0; j < ROWS; ++j)
#pragma unroll
    for (int c = 0; c < 16; ++c) acc[j][c] = 0.f;
  for (int a = 0; a < KS; ++a) {
    const float* xa = x + a * G::ROWF;
    const float* wa = wg + a * KS * 3 * Cout;
#pragma unroll
    for (int bc = 0; bc < KS * 3; ++bc) {          // (b, c) flattened: the HWIO order
      const int b = bc / 3, c = bc % 3;
      const int off = ((b & 1) * G::HALF + (b >> 1)) * 3 + c;   // pixel 2*col + b, channel c
      float xx[ROWS];
#pragma unroll
      for (int j = 0; j < ROWS; ++j) xx[j] = xa[2 * j * G::ROWF + off];
#pragma unroll
      for (int q = 0; q < 4; ++q) {                // 4 channels at a time: fewer live weights
        const float4 w4 = *reinterpret_cast<const float4*>(wa + bc * Cout + q * 4);
        const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
        for (int j = 0; j < ROWS; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[j][q * 4 + e] = fmaf(xx[j], wv[e], acc[j][q * 4 + e]);
      }
    }
  }
}

// U8: the input is uint8 BGR (p.x8) and the patch cell of an in-image byte b of channel c is
// float32(double(b) - mean[c]), exactly what the engine's conversion launch writes for the fp32
// path to read; a padding cell is 0 either way.  Only the patch staging differs, so the outputs
// are bitwise those of the fp32 instance on the converted images.
template <int KS, int NT, int MINB, bool U8 = false>
__global__ void __launch_bounds__(NT, MINB)
conv_pool_simt_kernel(const std::conditional_t<U8, ConvPoolU8Params, ConvPoolParams> p) {
  using G = PatchGeom<KS>;
  constexpr int K = KS * KS * 3;
  const int Cout = p.Cout;
  extern __shared__ __align__(16) float sm[];
  float* s_w = sm;                                  // [K][Cout]
  float* s_bias = s_w + K * Cout;                   // [Cout]
  float* s_scale = s_bias + Cout;                   // [Cout]
  float* s_shift = s_scale + Cout;                  // [Cout]
  float* s_patch = s_shift + Cout;                  // [2][ROWS][ROWF]
  float* s_vert = s_patch + ((2 * G::BUF + 3) & ~3);   // [Cout/16][VGS] (swizzled chunks)
  unsigned* s_stage = reinterpret_cast<unsigned*>(s_vert + (Cout / 16) * VGS);  // U8: [ROWS][SW]

  const int tid = threadIdx.x;
  const int nthreads = blockDim.x;
  const int wid = tid >> 5, lane = tid & 31, nwarps = nthreads >> 5;
  int tile = blockIdx.x;
  const int tw = tile % p.tiles_w;
  tile /= p.tiles_w;
  const int th = tile % p.tiles_h;
  const int img = tile / p.tiles_h;
  const int ph0 = th * p.strip_h, pw0 = tw * PT_W;               // pooled origin
  const int ph_end = min(p.Hp, ph0 + p.strip_h);
  const int nsteps = (ph_end - ph0 + 1) / 2;
  const int ch0 = 2 * ph0 - p.ppad_t, cw0 = 2 * pw0 - p.ppad_l;   // conv origin
  const int iy0 = 2 * ch0 - p.cpad_t, ix0 = 2 * cw0 - p.cpad_l;   // input origin

  // ---- input rows iy0 + r0 .. + nrows -> one patch buffer (U8: -> s_stage, see convert) ----
  auto load_rows = [&](float* buf, int r0, int nrows) {
    if constexpr (U8) {
      // One warp per in-image row: the words from the one holding the row's first needed byte
      // to the one holding its last.  Each holds at least one byte of the row, so no load
      // touches a padding row, another image or (allocations being 4-byte aligned) past an end.
      const uint8_t* xin = p.x8 + (size_t)img * p.H * p.W * 3;
      const int b0 = max(ix0 * 3, 0), b1 = min((ix0 + G::PX) * 3, p.W * 3);
      for (int row = wid; row < nrows; row += nwarps) {
        const int iy = iy0 + r0 + row;
        if (iy < 0 || iy >= p.H || b0 >= b1) continue;
        const uintptr_t a0 = (uintptr_t)(xin + (size_t)iy * p.W * 3 + b0);
        const uintptr_t w0 = a0 & ~(uintptr_t)3;
        const int nw = (int)((a0 + (b1 - b0) + 3 - w0) >> 2);
        for (int j = lane; j < nw; j += 32)
          cp_async4(s_stage + row * G::SW + j, (const void*)(w0 + 4 * j), 4);
      }
    } else {
      const float* xin = p.x + (size_t)img * p.H * p.W * 3;
      for (int t = tid; t < nrows * G::PX; t += nthreads) {
        const int row = t / G::PX, px = t - row * G::PX;
        const int iy = iy0 + r0 + row, ix = ix0 + px;
        const bool ok = iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
        const float* src = xin + (ok ? ((size_t)iy * p.W + ix) * 3 : 0);
        float* dst = buf + row * G::ROWF + ((px & 1) * G::HALF + (px >> 1)) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) cp_async4(dst + c, src + c, ok ? 4 : 0);  // 0: zero-filled
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  // U8: once a warp's own copies have landed, it converts the rows it staged (no block barrier)
  auto convert_rows = [&](float* buf, int r0, int nrows) {
    if constexpr (U8) {
      asm volatile("cp.async.wait_all;" ::: "memory");
      __syncwarp();
      const uint8_t* xin = p.x8 + (size_t)img * p.H * p.W * 3;
      const uint8_t* s_bytes = reinterpret_cast<const uint8_t*>(s_stage);
      const int b0 = max(ix0 * 3, 0), b1 = min((ix0 + G::PX) * 3, p.W * 3);
      for (int row = wid; row < nrows; row += nwarps) {
        const int iy = iy0 + r0 + row;
        const bool row_ok = iy >= 0 && iy < p.H;
        // byte b of the row sits at (row start + b0) % 4 + b - b0 in the row's staged words
        const int skew = row_ok ? (int)((uintptr_t)(xin + (size_t)iy * p.W * 3 + b0) & 3) - b0 : 0;
        for (int col = lane; col < G::PX * 3; col += 32) {
          const int ixc = ix0 * 3 + col;
          const int px = col / 3, c = col - 3 * px;
          float v = 0.f;                             // TF pads the mean-subtracted image with 0
          if (row_ok && ixc >= b0 && ixc < b1)
            v = (float)((double)s_bytes[row * G::SW * 4 + skew + ixc] -
                        (c == 0 ? p.mean[0] : c == 1 ? p.mean[1] : p.mean[2]));
          buf[row * G::ROWF + ((px & 1) * G::HALF + (px >> 1)) * 3 + c] = v;
        }
      }
    }
  };

  // ---- prologue: weights, bias/BN, the rows of conv row 0 and of step 0 ----
  for (int i = tid; i < K * Cout / 4; i += nthreads) {
    const unsigned dst = (unsigned)__cvta_generic_to_shared(s_w + i * 4);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(p.w + i * 4) : "memory");
  }
  if (tid < Cout) {
    s_bias[tid] = p.bias ? __ldg(p.bias + tid) : 0.f;
    s_scale[tid] = p.scale ? __ldg(p.scale + tid) : 1.f;
    s_shift[tid] = p.scale ? __ldg(p.shift + tid) : 0.f;
  }
  load_rows(s_patch, 0, KS);
  convert_rows(s_patch, 0, KS);
  load_rows(s_patch + G::BUF, 2, G::ROWS);
  convert_rows(s_patch + G::BUF, 2, G::ROWS);
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();

  const int cg = tid >> 6;                 // channel group (warp-uniform)
  const int col = tid & 63;                // conv column within the CTA
  const float* wg = s_w + cg * 16;
  const bool col_ok = cw0 + col >= 0 && cw0 + col < p.Wc;
  // +bias [, affine], relu; -inf outside the conv output (tf.nn.max_pool ignores padded cells)
  auto finish = [&](float (&v)[16], int crow) {
    const int oh = ch0 + crow;
    const bool ok = col_ok && oh >= 0 && oh < p.Hc;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float f = v[c] + s_bias[cg * 16 + c];
      if (p.scale) f = f * s_scale[cg * 16 + c] + s_shift[cg * 16 + c];
      if (p.relu) f = fmaxf(f, 0.f);
      v[c] = ok ? f : -CUDART_INF_F;
    }
  };

  float carry[16];                         // conv row 4s of the strip, finished
  {
    float acc[1][16];
    conv_rows<KS, 1>(s_patch + col * 3, wg, Cout, acc);
    finish(acc[0], 0);
#pragma unroll
    for (int c = 0; c < 16; ++c) carry[c] = acc[0][c];
  }

  const int chunks = Cout / 4;             // 16-byte chunks per pooled pixel; nthreads = 16 * chunks
  const int chunk = tid % chunks, pg = chunk >> 2, pj = chunk & 3;
  const float* vsrc = s_vert + pg * VGS;
  float* vdst = s_vert + cg * VGS;
  for (int s = 0; s < nsteps; ++s) {
    float* cur = s_patch + ((s + 1) & 1) * G::BUF;
    float* nxt = s_patch + (s & 1) * G::BUF;
    __syncthreads();                       // nxt and s_vert are free again
    const bool more = s + 1 < nsteps;
    if (more) load_rows(nxt, 8 * (s + 1) + 2, G::ROWS);

    float acc[NR][16];
    conv_rows<KS, NR>(cur + col * 3, wg, Cout, acc);
#pragma unroll
    for (int j = 0; j < NR; ++j) finish(acc[j], 4 * s + 1 + j);
    // vertical max: pooled row 2s over conv rows 4s .. 4s+2, row 2s+1 over 4s+2 .. 4s+4
    const int sw = (col >> 1) & 3;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float o0[4], o1[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = q * 4 + e;
        o0[e] = fmaxf(fmaxf(carry[c], acc[0][c]), acc[1][c]);
        o1[e] = fmaxf(fmaxf(acc[1][c], acc[2][c]), acc[3][c]);
        carry[c] = acc[3][c];
      }
      *reinterpret_cast<float4*>(vdst + col * 16 + ((q ^ sw) << 2)) =
          make_float4(o0[0], o0[1], o0[2], o0[3]);
      *reinterpret_cast<float4*>(vdst + (CT_C + col) * 16 + ((q ^ sw) << 2)) =
          make_float4(o1[0], o1[1], o1[2], o1[3]);
    }
    if (more) {
      convert_rows(nxt, 8 * (s + 1) + 2, G::ROWS);
      asm volatile("cp.async.wait_all;" ::: "memory");
    }
    __syncthreads();                       // s_vert written; nxt landed

    // ---- horizontal 3-wide max of the two rows, coalesced 128-bit stores ----
    for (int pp = tid / chunks; pp < 2 * PT_W; pp += 16) {
      const int prow = pp >= PT_W, pc = pp - prow * PT_W;
      const int ph = ph0 + 2 * s + prow, pw = pw0 + pc;
      if (ph >= ph_end || pw >= p.Wp) continue;
      float4 m = make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F);
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const int cc = prow * CT_C + 2 * pc + b;
        const float4 q = *reinterpret_cast<const float4*>(vsrc + cc * 16 + ((pj ^ ((cc >> 1) & 3)) << 2));
        m.x = fmaxf(m.x, q.x); m.y = fmaxf(m.y, q.y);
        m.z = fmaxf(m.z, q.z); m.w = fmaxf(m.w, q.w);
      }
      *reinterpret_cast<float4*>(p.y + (((size_t)img * p.Hp + ph) * p.Wp + pw) * Cout + chunk * 4) = m;
    }
  }
}

template <int KS>
size_t smem_bytes_for(int Cout, bool u8) {
  using G = PatchGeom<KS>;
  return sizeof(float) * ((size_t)KS * KS * 3 * Cout + 3 * (size_t)Cout +
                          (size_t)((2 * G::BUF + 3) & ~3) + (size_t)(Cout / 16) * VGS +
                          (u8 ? (size_t)G::ROWS * G::SW : 0));
}

// The <KS, NT, MINB> instantiations, indexed by conv_pool_instance.
void (*const kConvPoolU8Kernels[4])(ConvPoolU8Params) = {
    conv_pool_simt_kernel<3, 256, 2, true>, conv_pool_simt_kernel<3, 384, 1, true>,
    conv_pool_simt_kernel<7, 256, 1, true>, conv_pool_simt_kernel<7, 384, 1, true>};
void (*const kConvPoolKernels[4])(ConvPoolParams) = {
    conv_pool_simt_kernel<3, 256, 2>, conv_pool_simt_kernel<3, 384, 1>,
    conv_pool_simt_kernel<7, 256, 1>, conv_pool_simt_kernel<7, 384, 1>};

// Index of the kernel for a ksize x ksize conv on `threads` threads: the narrowest NT that holds them.
int conv_pool_instance(int ksize, int threads) { return (ksize == 7 ? 2 : 0) + (threads > 256); }

}  // namespace
bool conv_pool_simt_eligible(int Cin, int Cout, int ksize, int stride, int pool_size,
                             int pool_stride) {
  return Cin == 3 && (ksize == 3 || ksize == 7) && stride == 2 && pool_size == 3 &&
         pool_stride == 2 && Cout % 16 == 0 && Cout >= 16 && Cout <= 96;
}

int launch_conv_pool_simt(const float* x, const uint8_t* x8, const double* bgr_means,
                          const float* w, const float* bias, const float* scale,
                          const float* shift, float* y, int B, int H, int W, int Cout, int ksize,
                          int conv_padding, int relu, int pool_padding, cudaStream_t stream) {
  if (!conv_pool_simt_eligible(3, Cout, ksize, 2, 3, 2))
    return fail(SQDET_ERR_UNSUPPORTED, "conv+pool fusion: unsupported shape");
  const Geom ch = tf_geometry(H, ksize, 2, conv_padding), cw = tf_geometry(W, ksize, 2, conv_padding);
  if (ch.out <= 0 || cw.out <= 0) return fail(SQDET_ERR_INVALID_ARG, "conv+pool: empty conv output");
  const Geom ph = tf_geometry(ch.out, 3, 2, pool_padding), pw = tf_geometry(cw.out, 3, 2, pool_padding);
  if (ph.out <= 0 || pw.out <= 0) return fail(SQDET_ERR_INVALID_ARG, "conv+pool: empty pooled output");
  ConvPoolParams p;
  p.x = x; p.w = w; p.bias = bias; p.scale = scale; p.shift = shift; p.y = y;
  p.B = B; p.H = H; p.W = W; p.Cout = Cout;
  p.Hc = ch.out; p.Wc = cw.out; p.Hp = ph.out; p.Wp = pw.out;
  p.cpad_t = ch.pad_before; p.cpad_l = cw.pad_before;
  p.ppad_t = ph.pad_before; p.ppad_l = pw.pad_before;
  p.relu = relu;
  p.tiles_w = (p.Wp + PT_W - 1) / PT_W;
  const int threads = 64 * (Cout / 16);
  const int u8 = x8 != nullptr;
  const size_t smem = ksize == 3 ? smem_bytes_for<3>(Cout, u8) : smem_bytes_for<7>(Cout, u8);
  if (smem > 232448) return fail(SQDET_ERR_UNSUPPORTED, "conv+pool: tile does not fit in smem");
  // Exactly `threads` threads: each 64 of them own one 16-channel group (cg = tid >> 6), and
  // s_vert / bias hold Cout / 16 groups.  The instance's NT is only the __launch_bounds__ ceiling.
  const int inst = conv_pool_instance(ksize, threads);
  const void* fn = u8 ? (const void*)kConvPoolU8Kernels[inst] : (const void*)kConvPoolKernels[inst];
  // the opt-in is per device: remember which devices of this process already have it
  static unsigned long long attr_devs[2][4] = {};
  int dev = 0;
  SQ_CUDA(cudaGetDevice(&dev));
  if (dev >= 64 || !((attr_devs[u8][inst] >> dev) & 1ull)) {
    SQ_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    if (dev < 64) attr_devs[u8][inst] |= 1ull << dev;
  }
  // Strip height: a CTA costs about one step per two pooled rows plus one for its prologue and
  // pipeline fill, and the launch about that times its waves over the resident CTAs.  Taller
  // strips compute fewer rows twice; shorter ones leave a smaller last wave.
  int sms = 0, per_sm = 0;
  SQ_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  SQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, threads, smem));
  const long long slots = (long long)std::max(1, sms * per_sm);
  long long best = -1;
  for (int sh = 2; sh <= MAX_STRIP; sh += 2) {
    const long long ctas = (long long)B * ((p.Hp + sh - 1) / sh) * p.tiles_w;
    const long long cost = (ctas + slots - 1) / slots * (sh / 2 + 1);
    if (best < 0 || cost <= best) best = cost, p.strip_h = sh;
  }
  p.tiles_h = (p.Hp + p.strip_h - 1) / p.strip_h;
  const unsigned grid = (unsigned)(B * p.tiles_h * p.tiles_w);
  if (u8) {
    ConvPoolU8Params q;
    static_cast<ConvPoolParams&>(q) = p;
    q.x8 = x8;
    for (int c = 0; c < 3; ++c) q.mean[c] = bgr_means[c];
    kConvPoolU8Kernels[inst]<<<grid, threads, smem, stream>>>(q);
  } else {
    kConvPoolKernels[inst]<<<grid, threads, smem, stream>>>(p);
  }
  SQ_CHECK_LAUNCH("conv_pool_simt_kernel");
  return SQDET_OK;
}

}  // namespace sqdet
