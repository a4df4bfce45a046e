// Fused first layer: conv (Cin = 3, k x k, stride 2) + bias [+ frozen BN] + ReLU + 3x3/2
// max-pool in ONE kernel, fp32 FFMA.
//
// Replaces conv1 -> pool1 of every net (reference src/nets/squeezeDet.py:40-44,
// squeezeDetPlus.py:40-44, resnet50_convDet.py:41-46; layer code src/nn_skeleton.py:471-586).
// conv1's output is the largest tensor of the whole network (20 x 188 x 621 x 64 fp32 = 598 MB
// at the benchmark size); unfused it is written once and read once by pool1 (1.2 GB of the
// 4.7 GB a forward pass moves).  Here it never leaves shared memory.
//
// K = 27 (or 147) with Cin = 3 is too thin for a tensor-core tile and the layer is
// HBM-bound after fusion (reads 112 MB, writes 150 MB), so it stays on the FFMA pipe:
// exact fp32, same arithmetic as the reference's fp32 conv.
//
// CTA = one pooled tile of 4 x 16 pixels of one image:
//   input patch  (2*8+k) x (2*32+k) x 3 floats        -> smem (coalesced row loads, 0 = pad)
//                 (uint8 input: the 4-byte words holding each row's bytes -> smem, then
//                 float32(double(byte) - mean[c]) per cell, 0 = pad)
//   conv tile    9 x 33 conv pixels x Cout             -> registers (5 px x 16 ch per thread)
//                 -> +bias [*scale+shift], ReLU, -inf outside the image -> smem
//   pooled tile  4 x 16 x Cout, max over 3x3 windows   -> 128-bit coalesced global stores
// Threads: 64 per 16-channel group (Cout/16 groups).  Weights [k*k*3][Cout] live in smem.
#include <math_constants.h>

#include <type_traits>

#include "common.cuh"

namespace sqdet {
namespace {

constexpr int PT_H = 4, PT_W = 16;                 // pooled tile
constexpr int CT_H = 2 * PT_H + 1, CT_W = 2 * PT_W + 1;   // 9 x 33 conv pixels (3x3/2 pool)
constexpr int CT_PIX = CT_H * CT_W;               // 297
constexpr int PIX_PER_THREAD = (CT_PIX + 63) / 64;  // 5

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
};

// The uint8-input instances' parameters (x unused).  A type of their own: a larger block in the
// fp32 instances would change their code.
struct ConvPoolU8Params : ConvPoolParams {
  const uint8_t* x8;    // [B,H,W,3] BGR bytes, any byte alignment
  double mean[3];       // subtracted per channel
};

// U8: the input is uint8 BGR (p.x8) and the patch cell of an in-image byte b of channel c is
// float32(double(b) - mean[c]), exactly what the engine's conversion launch writes for the fp32
// path to read; a padding cell is 0 either way.  Only the patch staging differs, so the outputs
// are bitwise those of the fp32 instance on the converted images.
template <int KS, int NT, int MINB, bool U8 = false>
__global__ void __launch_bounds__(NT, MINB)
conv_pool_simt_kernel(const std::conditional_t<U8, ConvPoolU8Params, ConvPoolParams> p) {
  constexpr int PH = 2 * (CT_H - 1) + KS;          // input patch rows
  constexpr int PW = 2 * (CT_W - 1) + KS;          // input patch cols (pixels)
  constexpr int K = KS * KS * 3;
  // U8 staging: the aligned 4-byte words covering a row's PW*3 bytes at any alignment, one row of
  // SW words per patch row, in s_conv's space (free until epilogue 1)
  constexpr int SW = (PW * 3 + 6) / 4;
  static_assert(PH * SW <= CT_PIX * 16, "uint8 staging must fit in one channel group of s_conv");
  extern __shared__ __align__(16) float sm[];
  float* s_patch = sm;                             // [PH][PW*3]
  float* s_w = s_patch + ((PH * PW * 3 + 3) & ~3); // [K][Cout]
  float* s_conv = s_w + K * p.Cout;                // [Cout/16][CT_PIX][16] (swizzled chunks)

  const int tid = threadIdx.x;
  const int nthreads = blockDim.x;
  int tile = blockIdx.x;
  const int tw = tile % p.tiles_w;
  tile /= p.tiles_w;
  const int th = tile % p.tiles_h;
  const int img = tile / p.tiles_h;
  const int ph0 = th * PT_H, pw0 = tw * PT_W;            // pooled origin
  const int ch0 = 2 * ph0 - p.ppad_t, cw0 = 2 * pw0 - p.ppad_l;   // conv origin
  const int iy0 = 2 * ch0 - p.cpad_t, ix0 = 2 * cw0 - p.cpad_l;   // input origin

  // ---- stage weights and the input patch with cp.async (fire-and-forget, so the ~20
  // row-segment loads per thread overlap instead of paying one L2 round trip each) ----
  for (int i = tid; i < K * p.Cout / 4; i += nthreads) {
    const unsigned dst = (unsigned)__cvta_generic_to_shared(s_w + i * 4);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(p.w + i * 4) : "memory");
  }
  if constexpr (U8) {
    // One warp per in-image patch row: the words from the one holding the row's first needed
    // byte to the one holding its last.  Each holds at least one byte of the row, so no load
    // touches a padding row, another image or (allocations being 4-byte aligned) past an end.
    const uint8_t* xin = p.x8 + (size_t)img * p.H * p.W * 3;
    unsigned* s_stage = reinterpret_cast<unsigned*>(s_conv);
    const int wid = tid >> 5, lane = tid & 31, nwarps = nthreads >> 5;
    const int b0 = max(ix0 * 3, 0), b1 = min((ix0 + PW) * 3, p.W * 3);   // needed bytes of a row
    for (int row = wid; row < PH; row += nwarps) {
      const int iy = iy0 + row;
      if (iy < 0 || iy >= p.H || b0 >= b1) continue;
      const uintptr_t a0 = (uintptr_t)(xin + (size_t)iy * p.W * 3 + b0);
      const uintptr_t w0 = a0 & ~(uintptr_t)3;
      const int nw = (int)((a0 + (b1 - b0) + 3 - w0) >> 2);
      for (int j = lane; j < nw; j += 32) {
        const unsigned dst = (unsigned)__cvta_generic_to_shared(s_stage + row * SW + j);
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(w0 + 4 * j)
                     : "memory");
      }
    }
    // each warp converts the rows it staged once its own copies have landed: no block barrier
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncwarp();
    const uint8_t* s_bytes = reinterpret_cast<const uint8_t*>(s_stage);
    for (int row = wid; row < PH; row += nwarps) {
      const int iy = iy0 + row;
      const bool row_ok = iy >= 0 && iy < p.H;
      // byte b of the row sits at (row start + b0) % 4 + b - b0 in the row's staged words
      const int skew = row_ok ? (int)((uintptr_t)(xin + (size_t)iy * p.W * 3 + b0) & 3) - b0 : 0;
#pragma unroll
      for (int it = 0; it < (PW * 3 + 31) / 32; ++it) {
        const int col = lane + it * 32;
        if (col < PW * 3) {
          const int ixc = ix0 * 3 + col;
          float v = 0.f;                             // TF pads the mean-subtracted image with 0
          if (row_ok && ixc >= b0 && ixc < b1) {
            const int c = col % 3;
            v = (float)((double)s_bytes[row * SW * 4 + skew + ixc] -
                        (c == 0 ? p.mean[0] : c == 1 ? p.mean[1] : p.mean[2]));
          }
          s_patch[row * (PW * 3) + col] = v;
        }
      }
    }
  } else {
    const float* xin = p.x + (size_t)img * p.H * p.W * 3;
    const int wid = tid >> 5, lane = tid & 31, nwarps = nthreads >> 5;
    for (int row = wid; row < PH; row += nwarps) {       // one warp per patch row: coalesced
      const int iy = iy0 + row;
      const bool row_ok = iy >= 0 && iy < p.H;
      const float* src = xin + (size_t)(row_ok ? iy : 0) * p.W * 3;
#pragma unroll
      for (int it = 0; it < (PW * 3 + 31) / 32; ++it) {  // col counts floats (pixel*3 + c)
        const int col = lane + it * 32;
        if (col < PW * 3) {
          const int ixc = ix0 * 3 + col;
          const bool ok = row_ok && ixc >= 0 && ixc < p.W * 3;
          const unsigned dst = (unsigned)__cvta_generic_to_shared(s_patch + row * (PW * 3) + col);
          const int nbytes = ok ? 4 : 0;                 // 0 -> the 4 bytes are zero-filled
          asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst),
                       "l"(src + (ok ? ixc : 0)), "r"(nbytes)
                       : "memory");
        }
      }
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  // ---- conv: 5 pixels x 16 channels per thread ----
  const int cg = tid >> 6;                 // channel group (warp-uniform)
  const int l64 = tid & 63;
  float acc[PIX_PER_THREAD][16];
#pragma unroll
  for (int i = 0; i < PIX_PER_THREAD; ++i)
#pragma unroll
    for (int c = 0; c < 16; ++c) acc[i][c] = 0.f;
  int pbase[PIX_PER_THREAD];
#pragma unroll
  for (int i = 0; i < PIX_PER_THREAD; ++i) {
    int px = l64 + 64 * i;
    if (px >= CT_PIX) px = CT_PIX - 1;     // clamp (result discarded)
    const int cr = px / CT_W, cc = px - cr * CT_W;
    pbase[i] = (2 * cr * PW + 2 * cc) * 3;
  }
  const float* wg = s_w + cg * 16;
  for (int a = 0; a < KS; ++a) {
#pragma unroll
    for (int bc = 0; bc < KS * 3; ++bc) {          // (b, c) flattened: contiguous in the patch
      const int k = a * KS * 3 + bc;
      float xx[PIX_PER_THREAD];
#pragma unroll
      for (int i = 0; i < PIX_PER_THREAD; ++i) xx[i] = s_patch[pbase[i] + a * PW * 3 + bc];
#pragma unroll
      for (int q = 0; q < 4; ++q) {                // 4 channels at a time: fewer live weights
        const float4 w4 = *reinterpret_cast<const float4*>(wg + k * p.Cout + q * 4);
        const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
        for (int i = 0; i < PIX_PER_THREAD; ++i)
#pragma unroll
          for (int c = 0; c < 4; ++c) acc[i][q * 4 + c] = fmaf(xx[i], wv[c], acc[i][q * 4 + c]);
      }
    }
  }

  // ---- epilogue 1: bias [, affine], relu, mask, conv tile -> smem ----
  {
    float bv[16], sv[16], hv[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      bv[c] = p.bias ? __ldg(p.bias + cg * 16 + c) : 0.f;
      sv[c] = p.scale ? __ldg(p.scale + cg * 16 + c) : 1.f;
      hv[c] = p.scale ? __ldg(p.shift + cg * 16 + c) : 0.f;
    }
    float* tile_c = s_conv + (size_t)cg * CT_PIX * 16;
#pragma unroll
    for (int i = 0; i < PIX_PER_THREAD; ++i) {
      const int px = l64 + 64 * i;
      if (px < CT_PIX) {
        const int cr = px / CT_W, cc = px - cr * CT_W;
        const int oh = ch0 + cr, ow = cw0 + cc;
        const bool ok = oh >= 0 && oh < p.Hc && ow >= 0 && ow < p.Wc;
        const int sw = (px >> 1) & 3;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float o[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float f = acc[i][j * 4 + e] + bv[j * 4 + e];
            if (p.scale) f = f * sv[j * 4 + e] + hv[j * 4 + e];
            if (p.relu) f = fmaxf(f, 0.f);
            o[e] = ok ? f : -CUDART_INF_F;      // tf.nn.max_pool ignores padded cells
          }
          *reinterpret_cast<float4*>(tile_c + px * 16 + ((j ^ sw) << 2)) =
              make_float4(o[0], o[1], o[2], o[3]);
        }
      }
    }
  }
  __syncthreads();

  // ---- epilogue 2: 3x3/2 max-pool from smem, coalesced 128-bit stores ----
  const int chunks = p.Cout / 4;                   // 16-byte chunks per pooled pixel
  for (int u = tid; u < PT_H * PT_W * chunks; u += nthreads) {
    const int chunk = u % chunks, pp = u / chunks;
    const int py = pp / PT_W, pxp = pp - py * PT_W;
    const int ph = ph0 + py, pw = pw0 + pxp;
    if (ph >= p.Hp || pw >= p.Wp) continue;
    const int g = chunk >> 2, j = chunk & 3;
    const float* tile_c = s_conv + (size_t)g * CT_PIX * 16;
    float4 m = make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F);
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const int px = (2 * py + a) * CT_W + 2 * pxp + b;
        const float4 q = *reinterpret_cast<const float4*>(tile_c + px * 16 + ((j ^ ((px >> 1) & 3)) << 2));
        m.x = fmaxf(m.x, q.x); m.y = fmaxf(m.y, q.y);
        m.z = fmaxf(m.z, q.z); m.w = fmaxf(m.w, q.w);
      }
    *reinterpret_cast<float4*>(p.y + (((size_t)img * p.Hp + ph) * p.Wp + pw) * p.Cout + chunk * 4) = m;
  }
}

template <int KS>
size_t smem_bytes_for(int Cout) {
  constexpr int PH = 2 * (CT_H - 1) + KS, PW = 2 * (CT_W - 1) + KS;
  return sizeof(float) * ((size_t)((PH * PW * 3 + 3) & ~3) + (size_t)KS * KS * 3 * Cout +
                          (size_t)(Cout / 16) * CT_PIX * 16);
}

// The <KS, NT, MINB> instantiations, indexed by conv_pool_instance.  The uint8 ones come first:
// ptxas compiles a module's kernels last to first, and so compiles the fp32 ones as it did
// before they existed (their SASS is unchanged).
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
  p.tiles_h = (p.Hp + PT_H - 1) / PT_H;
  p.tiles_w = (p.Wp + PT_W - 1) / PT_W;
  const unsigned grid = (unsigned)(B * p.tiles_h * p.tiles_w);
  const int threads = 64 * (Cout / 16);
  const size_t smem = ksize == 3 ? smem_bytes_for<3>(Cout) : smem_bytes_for<7>(Cout);
  if (smem > 232448) return fail(SQDET_ERR_UNSUPPORTED, "conv+pool: tile does not fit in smem");
  // Exactly `threads` threads: each 64 of them own one 16-channel group (cg = tid >> 6), and
  // s_conv / bias hold Cout / 16 groups.  The instance's NT is only the __launch_bounds__ ceiling.
  const int u8 = x8 != nullptr, inst = conv_pool_instance(ksize, threads);
  const void* fn = u8 ? (const void*)kConvPoolU8Kernels[inst] : (const void*)kConvPoolKernels[inst];
  // the opt-in is per device: remember which devices of this process already have it
  static unsigned long long attr_devs[2][4] = {};
  int dev = 0;
  SQ_CUDA(cudaGetDevice(&dev));
  if (dev >= 64 || !((attr_devs[u8][inst] >> dev) & 1ull)) {
    SQ_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    if (dev < 64) attr_devs[u8][inst] |= 1ull << dev;
  }
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
