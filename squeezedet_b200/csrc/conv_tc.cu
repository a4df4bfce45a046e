// Hopper (sm_90a) wgmma implicit-GEMM convolution with the 3xTF32 split (SQDET_MATH_TF32X3_TC).
//
// Replaces tf.nn.conv2d + bias_add [+ batch_normalization] + relu of the reference
// (src/nn_skeleton.py:539-547, :441-449) for every stride-1 SAME 1x1 / 3x3 conv whose Cin is a
// multiple of 16 (all fire squeeze/expand convs, the ConvDet head, the VGG/ResNet body) and for
// 3x3 convs over 3-channel images ("gather mode"), and runs a fire module's expand1x1 ||
// expand3x3 + channel concat (src/nets/squeezeDet.py:96-106) as one launch.
//
// GEMM view per CTA:  D[128 pixels, NT] += A[128 pixels, K] * W[K, NT]
//   M tile : 128 output pixels; two warpgroups, each owning 64 rows (one wgmma m64 row block).
//            Halo mode (every launch with a 3x3 conv over a Cin % 16 == 0 input): an 8-row x
//            16-column tile of one image, warp 4 wg + wq owning tile row 4 wg + wq.  Row mode
//            (1x1-only launches) and gather mode: 128 consecutive pixels of the flattened
//            B*Ho*Wo output list.
//   N      : one chunk of NT output channels (16, 32, 64, or 72 for the ConvDet head) of one
//            conv; blockIdx.y walks the chunks of every conv of the launch (the fire expand pair
//            is two convs).
//   K      : walked in KC-channel chunks (KC = 32 or 16).  Halo mode walks a 3x3 conv channel
//            chunk by channel chunk with the nine taps inner; a 1x1 conv is its channel chunks.
//            Gather mode flattens (dy, dx, c) and pads it to a multiple of 32.
//   A      : TMA tensor-map loads (out-of-bounds zero fill = TF SAME padding) into a row-major
//            [pixel][KC] tile stored with the 128-byte (KC = 32) or 64-byte (KC = 16) swizzle,
//            then into registers in the wgmma A-fragment layout (the swizzle keeps the reads
//            conflict-free).  In halo mode a 3x3 conv loads the 10 x 18 halo of its tile once per
//            channel chunk and reads tap (dy, dx) at a row offset into it, so each input value
//            crosses from L2 once per channel chunk instead of once per tap.  Gather mode (a
//            12-byte pixel is below TMA's 16-byte granule) gathers with cp.async into the same
//            swizzled layout.
//   W      : host-packed per (chunk, K chunk) in the no-swizzle K-major core-matrix layout
//            [NT/8][KC/4][8 rows][4 floats], hi then lo half; one bulk copy per K chunk, read by
//            wgmma through a shared-memory descriptor.
// Precision: fp32 operands are split a = a_hi + a_lo with a_hi = rn_tf32(a), a_lo = rn_tf32(a - a_hi)
//   (rounding a_lo here keeps the tensor core's truncation of its inputs from biasing the sum);
//   D += a_lo*b_hi + a_hi*b_lo + a_hi*b_hi (the dropped lo*lo term is ~2^-22 of a product): fp32-
//   grade results, which the 1e-4 parity bar against the fp32 reference needs through ~25
//   stacked convs (plain TF32 misses it by 1-2 orders of magnitude).  Weights are pre-split on the
//   host, activations in registers after the A-fragment load.
// Accumulation: each 8-wide K step (the three split MMAs) accumulates from zero in the wgmma
//   accumulator and is then added into fp32 running sums with round-to-nearest FADDs, so the
//   tensor core's truncating accumulation never compounds over a long K (longer chains in the
//   accumulator left a one-signed error that fails the 1e-4 box parity of SqueezeDet+).
// Pipeline: 3-stage ring tracked by mbarriers.  A stage's `full` barrier completes on the bytes
//   of its copies; its `empty` barrier on one arrival per consumer warp once the warp has retired
//   the MMAs that read it.  One thread waits for a stage to be empty and issues its copies, so the
//   K loop has no block barrier.  A halo tile travels with the first K chunk that reads it, and
//   two halo buffers alternate between channel chunks.  Within a K chunk the steps alternate
//   between two accumulator sets: step k + 1's MMAs are issued before step k is waited for
//   (wait_group 1) and added in, and the next A fragment is loaded and split while they run.
//   Each chunk ends with wait_group 0 before its warp releases the stage.
//   The 72-wide tile runs its steps one at a time in one accumulator set instead, which lets two
//   of its CTAs share an SM.
// K split (the 72-wide halo-mode tile only): a cluster of S CTAs along blockIdx.z shares one
//   output tile; rank r walks a contiguous range of the conv's channel chunks, all nine taps of
//   each, through its own ring.  The ranks then reduce their partial tiles through distributed
//   shared memory in rank order 0, 1, ..., S - 1, each rank finishing 1/S of the tile.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "common.cuh"
#include "conv_tc.cuh"

namespace sqdet {
namespace {

constexpr int TILE_M = 128;
constexpr int NUM_THREADS = 256;   // 2 warpgroups x 64 rows
constexpr int STAGES = 3;
constexpr int MAX_CHUNKS = 32;
// output tiles of the halo-mode convolution and the fire kernel: 8 rows x FT_W columns, read
// through a (8 + 2) x FQ_W halo of FQ_P pixels
constexpr int FT_W = 16, FQ_W = FT_W + 2, FQ_P = 10 * FQ_W;

// conv_tc_kernel's operand tiling (see the file comment), or a plan of fire_tc_kernel
enum TcMode { TC_ROWS, TC_GATHER, TC_HALO, TC_FIRE };

struct TcChunk {
  int ksize, pad_t, pad_l;  // this conv's filter size and top / left zero padding (gather mode)
  int nk;                   // K chunks of KC channels
  int ncount;               // valid output channels of this chunk (<= NT)
  int y_off;                // first output channel in y
  int p_off;                // first entry of bias / scale / shift
  long long w_off;          // float offset of the chunk's packed weights
};

struct TcParams {
  // tensor maps over x (encoded per launch input): row mode (C, B*H*W) boxes of (KC, 128); halo
  // mode (C, W, H, B) boxes of (KC, 18, 10, 1) for 3x3 halos in `amap`, (KC, 16, 8, 1) for the
  // tile of a 1x1 conv in `amap1`
  CUtensorMap amap, amap1;
  const float* x;
  float* y;
  const float* w;
  const float* bias;   // may be null
  const float* scale;  // null unless a frozen-BN affine follows the bias
  const float* shift;
  int B, H, W, Cin, Ho, Wo, stride, relu, y_cstride;
  long long M;         // B * Ho * Wo
  int tiles_w, tiles_h;   // halo mode: output tiles per image row / column
  int nchunks;
  TcChunk chunks[MAX_CHUNKS];
};

// ---------------------------------------------------------------------------------------------
// PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src),
               "r"(valid ? 4 : 0)
               : "memory");
}
// makes cp.async operations this thread issued so far arrive on `bar` when they complete (the
// barrier's count includes the arrival)
__device__ __forceinline__ void cp_async_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// mbarriers
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// orders the initialisations before the barriers' use by other threads and the async proxy
__device__ __forceinline__ void mbar_init_fence() {
  asm volatile("fence.mbarrier_init.release.cluster;\n\tfence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrives and adds `bytes` to the transaction count the current phase waits for
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
// waits for the completion of the phase of parity `parity`
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred done;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 done, [%0], %1;\n\t"
      "@!done bra WAIT_%=;\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// The operand ring: K chunk j of a kernel's sequence goes through stage j % STAGES.  A stage's
// full barrier completes once its copies (and in gather mode every thread's cp.async arrival)
// have landed; its empty barrier once each warp has released the stage's K chunk.
__device__ __forceinline__ void ring_init(uint64_t* full, uint64_t* empty, int full_count) {
  for (int s = 0; s < STAGES; ++s) {
    mbar_init(&full[s], full_count);
    mbar_init(&empty[s], NUM_THREADS / 32);
  }
  mbar_init_fence();
}
// Loader: waits until the warps have released K chunk j - STAGES, the last one in j's stage, and
// returns the stage.
__device__ __forceinline__ int ring_acquire(uint64_t* empty, int j) {
  const int s = j % STAGES;
  if (j >= STAGES) mbar_wait(&empty[s], (j / STAGES & 1) ^ 1);
  return s;
}
// Consumer: waits for K chunk j's copies and returns its stage.
__device__ __forceinline__ int ring_wait_full(uint64_t* full, int j) {
  const int s = j % STAGES;
  mbar_wait(&full[s], j / STAGES & 1);
  return s;
}
// Consumer warp: releases K chunk j's stage once every lane is done with it (its MMAs retired).
__device__ __forceinline__ void ring_release(uint64_t* empty, int j) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[j % STAGES]);
}

// `bytes` contiguous bytes from global memory into shared memory, completing on `bar`
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// one box of a 2-D / 4-D tensor map at the given coordinates (innermost first), completing on `bar`
__device__ __forceinline__ void tma_load(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2,
                                         int c3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
      : "memory");
}
// every thread of every CTA of the cluster; orders each thread's shared-memory writes before the
// other CTAs' reads after it
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the four floats at this CTA's shared address `addr` as seen in the shared memory of cluster rank `rank`
__device__ __forceinline__ float4 ld_cluster_f4(uint32_t addr, int rank) {
  float4 v;
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %4, %5;\n\t"
      "ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [ra];\n\t}"
      : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
      : "r"(addr), "r"(rank)
      : "memory");
  return v;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
// waits until at most N committed wgmma groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator / A-fragment reads and writes across the
// asynchronous MMAs
__device__ __forceinline__ void fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }
__device__ __forceinline__ void fence_operand(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }

// No-swizzle K-major descriptor: core matrices of 8 rows x 16 bytes, K-adjacent ones 128 B apart
// (LBO), 8-row groups `sbo` bytes apart (SBO).
__device__ __forceinline__ uint64_t make_desc(uint32_t addr, uint32_t sbo) {
  return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)(128 >> 4) << 16) |
         ((uint64_t)(sbo >> 4) << 32);
}

__device__ __forceinline__ float rn_tf32(float x) {
  // round-to-nearest (ties away) onto the 10-bit TF32 mantissa; the low 13 bits end up zero so
  // the value is exact whatever the tensor core does with the low bits of its fp32 inputs
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}

// D[64 x N] (+)= A[64 x 8] (registers) * B[8 x N] (shared-memory descriptor), tf32 -> fp32
template <int N>
struct Mma;
template <>
struct Mma<16> {
  static __device__ __forceinline__ void run(float (&d)[8], const uint32_t (&a)[4], uint64_t b,
                                             int acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
};
template <>
struct Mma<32> {
  static __device__ __forceinline__ void run(float (&d)[16], const uint32_t (&a)[4], uint64_t b,
                                             int acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),
          "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
};
template <>
struct Mma<64> {
  static __device__ __forceinline__ void run(float (&d)[32], const uint32_t (&a)[4], uint64_t b,
                                             int acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),
          "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
          "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]),
          "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
};
// the ConvDet head's 72 = 9 anchors x (classes + 1 + 4) channels as one tile
template <>
struct Mma<72> {
  static __device__ __forceinline__ void run(float (&d)[36], const uint32_t (&a)[4], uint64_t b,
                                             int acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %41, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n72k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35}, "
        "{%36, %37, %38, %39}, %40, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),
          "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
          "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]),
          "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
  }
};

// conv_tc_kernel's shared memory, from a 1024-byte aligned base (the swizzle pattern repeats
// every 1024 bytes): the weight ring, STAGES x [2 NT KC]; the A tiles, STAGES x [TILE_M][KC] (one
// per stage), or in halo mode for a 3x3 conv two halo tiles of halo_rows(KC) rows in the same
// space; then the full and empty barrier of each stage.
__host__ __device__ constexpr int halo_rows(int KC) {   // FQ_P rows rounded up to a multiple of 1024 bytes
  return (FQ_P * KC * 4 + 1023) / 1024 * 1024 / (KC * 4);
}
static_assert(2 * halo_rows(16) <= STAGES * TILE_M && 2 * halo_rows(32) <= STAGES * TILE_M,
              "two halo tiles fit in the A ring");
constexpr size_t conv_smem_bytes(int NT, int KC) {
  return 1024 + (size_t)STAGES * (2 * NT * KC + TILE_M * KC) * sizeof(float) + 2 * STAGES * sizeof(uint64_t);
}

// Splits four fp32 A values into their TF32 hi parts and rounded lo remainders.
__device__ __forceinline__ void split(const float (&v)[4], uint32_t (&ahi)[4], uint32_t (&alo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float hi = rn_tf32(v[i]);
    ahi[i] = __float_as_uint(hi);
    alo[i] = __float_as_uint(rn_tf32(v[i] - hi));   // rounded, not truncated by the MMA
  }
}

// A fragment of 8-wide K step `ks` for this thread's rows g (a0) and g + 8 (a1) of a padded tile.
__device__ __forceinline__ void load_split(const float* a0, const float* a1, int ks, int t,
                                           uint32_t (&ahi)[4], uint32_t (&alo)[4]) {
  split({a0[ks * 8 + t], a1[ks * 8 + t], a0[ks * 8 + t + 4], a1[ks * 8 + t + 4]}, ahi, alo);
}

// The swizzled [pixel][KC] tiles: 16-byte column chunk j of row p is stored at chunk j ^ swz(p),
// TMA's 128-byte swizzle for KC = 32 (128-byte rows), its 64-byte swizzle for KC = 16.  Rows
// p .. p + 7 then cover every bank once, at any p (so at every halo tap offset too).
template <int KC>
__device__ __forceinline__ int swz(int p) {
  return KC == 32 ? (p & 7) : ((p >> 1) & 3);
}
// A fragment of K step `ks` for rows p and p + 8 (which share the swizzle) of a swizzled tile
template <int KC>
__device__ __forceinline__ void load_split_swz(const float* tile, int p, int ks, int t,
                                               uint32_t (&ahi)[4], uint32_t (&alo)[4]) {
  const float* a0 = tile + p * KC + t;
  const float* a1 = a0 + 8 * KC;
  const int j0 = (2 * ks ^ swz<KC>(p)) * 4, j1 = ((2 * ks + 1) ^ swz<KC>(p)) * 4;
  split({a0[j0], a1[j0], a0[j1], a1[j1]}, ahi, alo);
}

// Issues K step `ks` of a KC-channel chunk as one wgmma group: the three split MMAs into `acc`,
// the first from zero.  B = hi tile at shared address `bhi`, lo tile right after it.
template <int NT, int KC>
__device__ __forceinline__ void mma_step(float (&acc)[NT / 2], const uint32_t (&ahi)[4],
                                         const uint32_t (&alo)[4], uint32_t bhi, int ks) {
  constexpr uint32_t SBO = (KC / 4) * 128;
  const uint32_t blo = bhi + NT * KC * 4;
  const uint64_t dhi = make_desc(bhi + ks * 256, SBO), dlo = make_desc(blo + ks * 256, SBO);
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) fence_operand(acc[i]);
  wgmma_fence();
  Mma<NT>::run(acc, alo, dhi, 0);
  Mma<NT>::run(acc, ahi, dlo, 1);
  Mma<NT>::run(acc, ahi, dhi, 1);
  wgmma_commit();
}

// Adds the accumulator of a retired K step into the fp32 running sums; its A fragment is free.
template <int N>
__device__ __forceinline__ void flush(float (&acc)[N], float (&sum)[N], uint32_t (&ahi)[4],
                                      uint32_t (&alo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) fence_operand(ahi[i]), fence_operand(alo[i]);
#pragma unroll
  for (int i = 0; i < N; ++i) {
    fence_operand(acc[i]);
    sum[i] += acc[i];
  }
}

// One K chunk of KC channels; `load_a(ks, ahi, alo)` loads and splits this thread's A fragment
// of step ks, B is at `bhi`.  Software-pipelined over two accumulator sets: step ks runs into
// acc[ks & 1], and while its MMAs are in flight the previous step is retired
// (wgmma.wait_group 1) and added into the fp32 running sums, and the next step's A fragment is
// loaded and split.  Every step still runs from a zeroed accumulator and is added in K order, as
// in an unpipelined loop.
//
// The chunk ends with every group retired (wait_group 0).  That drain leaves one MMA latency
// exposed per chunk, but after it no wgmma of this warpgroup reads the chunk's stage, so the
// caller may release it.  (ptxas also serialises every wgmma of a kernel whose accumulators are
// read in a loop that a group stays in flight across.)
//
// PIPE = false runs one step at a time in acc[0] (wait_group 0 after each): the 72-wide tile's
// registers then allow two CTAs per SM, and the other CTA fills the exposed MMA latency.
template <int NT, int KC, bool PIPE = true, typename LoadA>
__device__ __forceinline__ void mma_chunk(LoadA load_a, uint32_t bhi, float (&acc)[2][NT / 2],
                                          float (&sum)[NT / 2]) {
  constexpr int KSTEPS = KC / 8;
  uint32_t ahi[2][4], alo[2][4];
  if constexpr (!PIPE) {
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
      load_a(ks, ahi[0], alo[0]);
      mma_step<NT, KC>(acc[0], ahi[0], alo[0], bhi, ks);
      wgmma_wait<0>();
      flush(acc[0], sum, ahi[0], alo[0]);
    }
  } else {
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
      const int cur = ks & 1;
      load_a(ks, ahi[cur], alo[cur]);
      mma_step<NT, KC>(acc[cur], ahi[cur], alo[cur], bhi, ks);
      if (ks > 0) {
        wgmma_wait<1>();
        flush(acc[cur ^ 1], sum, ahi[cur ^ 1], alo[cur ^ 1]);
      }
    }
    constexpr int last = (KSTEPS - 1) & 1;
    wgmma_wait<0>();
    flush(acc[last], sum, ahi[last], alo[last]);
  }
}

// Halo mode and the fire kernel: the CTA's 8 x FT_W output tile, of image n at (oy0, ox0)
struct HaloTile {
  int n, oy0, ox0;
};
__device__ __forceinline__ HaloTile halo_tile(int tiles_w, int tiles_h) {
  const int tx = blockIdx.x % tiles_w, rest = blockIdx.x / tiles_w;
  return {rest / tiles_h, rest % tiles_h * 8, tx * FT_W};
}

// Output channel c of chunk ch from its sum: bias, frozen-BN affine, ReLU.
__device__ __forceinline__ float finish(const TcParams& p, const TcChunk& ch, int c, float v) {
  if (p.bias) v += p.bias[ch.p_off + c];
  if (p.scale) v = v * p.scale[ch.p_off + c] + p.shift[ch.p_off + c];
  if (p.relu) v = fmaxf(v, 0.f);
  return v;
}

// Stores channels c and c + 1 (c even) of an output row whose first `ncount` channels are valid,
// value(c) giving each: one 8-byte store when `pair` (every row of the chunk starts 8-byte
// aligned) and both are valid, else one 4-byte store per valid channel.
template <typename Value>
__device__ __forceinline__ void store_pair(float* yrow, int c, int ncount, bool pair, Value value) {
  if (pair && c + 1 < ncount) {
    *reinterpret_cast<float2*>(yrow + c) = make_float2(value(c), value(c + 1));
  } else {
    if (c < ncount) yrow[c] = value(c);
    if (c + 1 < ncount) yrow[c + 1] = value(c + 1);
  }
}
// Whether every output row of chunk ch starts 8-byte aligned.
__device__ __forceinline__ bool rows_pair_aligned(const TcParams& p, const TcChunk& ch) {
  return ((p.y_cstride | ch.y_off) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.y) & 7) == 0;
}

// ---------------------------------------------------------------------------------------------
// Two CTAs per SM (the shared memory of 3 stages allows it up to NT = 72, KC = 32): at most 128
// registers a thread.  The 72-wide tile fits them only with one accumulator set (mma_chunk's
// PIPE = false: 72 accumulator and sum registers instead of 108).
//
// KSPLIT (halo mode): launched in clusters of gridDim.z CTAs along z; rank blockIdx.z sums the
// channel chunks [z nc / S, (z + 1) nc / S) of the conv's nc (see the file comment).
template <int NT, int KC, int MODE, bool KSPLIT = false>
__global__ void __launch_bounds__(NUM_THREADS, 2)
conv_tc_kernel(const __grid_constant__ TcParams p) {
  static_assert(!KSPLIT || MODE == TC_HALO, "the K split walks halo-mode channel chunks");
  constexpr int NACC = NT / 2;
  constexpr int WST = 2 * NT * KC;   // floats of one stage's hi + lo weight tiles
  constexpr uint32_t W_BYTES = WST * 4, TILE_BYTES = TILE_M * KC * 4, HALO_BYTES = FQ_P * KC * 4;
  constexpr int HROWS = halo_rows(KC);
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float* const smem = reinterpret_cast<float*>(smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023));
  float* const sa = smem + STAGES * WST;   // A tiles
  uint64_t* const full = reinterpret_cast<uint64_t*>(sa + STAGES * TILE_M * KC);
  uint64_t* const empty = full + STAGES;

  const TcChunk& ch = p.chunks[blockIdx.y];
  const int tid = threadIdx.x;
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const float* wch = p.w + ch.w_off;
  // this CTA's K chunks [k0, k0 + nk) of the conv's ch.nk; the loop below counts them from 0
  int k0 = 0, nk = ch.nk;
  const int taps = ch.ksize * ch.ksize;   // 1 or 9
  if (KSPLIT) {
    const int nc = ch.nk / taps, S = gridDim.z, z = blockIdx.z;
    k0 = z * nc / S * taps;
    nk = (z + 1) * nc / S * taps - k0;
    wch += (size_t)k0 * WST;
  }

  // gather mode: every thread's cp.async arrival besides the weight copy's
  if (tid == 0) ring_init(full, empty, MODE == TC_GATHER ? NUM_THREADS + 1 : 1);
  __syncthreads();

  // ---- row and gather mode: 128 consecutive output pixels from m0
  const long long m0 = (long long)blockIdx.x * TILE_M;

  // Gather mode, every thread: pixel `lp`, half `lh` of the 32 K values of K chunk kk into stage s
  auto gather_stage = [&](int kk, int s) {
    const int lp = tid >> 1, lh = tid & 1;
    const long long lm = m0 + lp;
    const bool lvalid = lm < p.M;
    int ln = 0, liy0 = 0, lix0 = 0;
    if (lvalid) {
      const int hw = p.Ho * p.Wo;
      ln = (int)(lm / hw);
      const int r = (int)(lm - (long long)ln * hw);
      liy0 = (r / p.Wo) * p.stride - ch.pad_t;
      lix0 = (r % p.Wo) * p.stride - ch.pad_l;
    }
    const float* xn = p.x + (size_t)ln * p.H * p.W * p.Cin;
    float* const arow = sa + (s * TILE_M + lp) * KC;
#pragma unroll
    for (int j = 0; j < KC / 2; ++j) {
      const int col = lh * (KC / 2) + j, k = kk * KC + col;
      const int tap = k / p.Cin, c = k - tap * p.Cin;
      const int iy = liy0 + tap / ch.ksize, ix = lix0 + tap % ch.ksize;
      const bool ok = lvalid && tap < taps && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
      // 32-bit offset: one image of a 3-channel input is far below 2^31 floats
      cp_async4(smem_u32(arow + ((col >> 2 ^ swz<KC>(lp)) << 2) + (col & 3)),
                ok ? xn + ((iy * p.W + ix) * p.Cin + c) : p.x, ok);
    }
    cp_async_arrive(&full[s]);
  };

  // K chunk j into stage s once the warps have released the stage's previous K chunk: its
  // weights and the A values it is the first to read.  Thread 0 issues the bulk and tensor copies.
  auto load_stage = [&](int j) {
    if (MODE != TC_GATHER && tid != 0) return;
    const int s = ring_acquire(empty, j);
    if (MODE == TC_GATHER) gather_stage(j, s);
    if (tid != 0) return;
    uint32_t bytes = W_BYTES;
    if (MODE == TC_ROWS) {
      // 1x1, stride 1: output pixel m reads input pixel m
      bytes += TILE_BYTES;
      mbar_expect_tx(&full[s], bytes);
      tma_load(smem_u32(sa + s * TILE_M * KC), &p.amap, j * KC, (int)m0, &full[s]);
    } else if (MODE == TC_HALO) {
      const HaloTile tl = halo_tile(p.tiles_w, p.tiles_h);
      if (taps == 1) {
        bytes += TILE_BYTES;
        mbar_expect_tx(&full[s], bytes);
        tma_load(smem_u32(sa + s * TILE_M * KC), &p.amap1, (k0 + j) * KC, tl.ox0, tl.oy0, tl.n, &full[s]);
      } else if (j % 9 == 0) {
        // channel chunk c = j / 9: its halo, into buffer c & 1, whose last reader (K chunk j - 10)
        // was released before K chunk j - STAGES was
        bytes += HALO_BYTES;
        mbar_expect_tx(&full[s], bytes);
        tma_load(smem_u32(sa + (j / 9 & 1) * HROWS * KC), &p.amap, (k0 + j) / 9 * KC, tl.ox0 - 1,
                 tl.oy0 - 1, tl.n, &full[s]);
      } else {
        mbar_expect_tx(&full[s], bytes);
      }
    } else {
      mbar_expect_tx(&full[s], bytes);
    }
    bulk_load(smem_u32(smem + s * WST), wch + (size_t)j * WST, W_BYTES, &full[s]);
  };

#pragma unroll 1
  for (int j = 0; j < STAGES - 1 && j < nk; ++j) load_stage(j);

  // ---- MMA role: warpgroup `wg` owns rows [64 wg, 64 wg + 64); A-fragment row g / g + 8 of
  // warp `wq`'s 16-row slice, columns t / t + 4 of each 8-wide K step.  In halo mode the slice
  // is tile row r = 4 wg + wq and rows g / g + 8 are its columns g / g + 8.
  const int arow0 = wg * 64 + wq * 16 + g;
  const int r = wg * 4 + wq;
  float acc[2][NACC], sum[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[0][i] = acc[1][i] = sum[i] = 0.f;

  for (int kk = 0; kk < nk; ++kk) {
    if (kk + STAGES - 1 < nk) load_stage(kk + STAGES - 1);
    const int s = ring_wait_full(full, kk);

    // (in halo mode row arow0 of an 8 x FT_W tile is pixel (r, g), as a 1x1 conv loads it)
    const float* tile = sa + s * TILE_M * KC;
    int prow = arow0;
    if (MODE == TC_HALO && taps > 1) {
      const int c = kk / 9, tap = kk - c * 9;
      tile = sa + (c & 1) * HROWS * KC;
      prow = (r + tap / 3) * FQ_W + g + tap % 3;
    }
    mma_chunk<NT, KC, NT != 72>(
        [&](int ks, uint32_t(&ahi)[4], uint32_t(&alo)[4]) { load_split_swz<KC>(tile, prow, ks, t, ahi, alo); },
        smem_u32(smem + s * WST), acc, sum);
    ring_release(empty, kk);
  }

  // ---- epilogue: accumulator element 4j + 2h + e is (row g + 8h, column 8j + 2t + e)
  if constexpr (KSPLIT) {
    // this rank's partial tile, [TILE_M][NT] over the ring once every warp is done with the ring
    static_assert(TILE_M * NT <= STAGES * (WST + TILE_M * KC), "the partial tile fits in the ring");
    float* const part = smem;
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < NT / 8; ++j)
        *reinterpret_cast<float2*>(part + (arow0 + 8 * h) * NT + 8 * j + 2 * t) =
            make_float2(sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
    cluster_sync();
    // rank z finishes the 4-channel groups [z G / S, (z + 1) G / S) of the tile's G, adding the
    // ranks' partials in rank order
    constexpr int G = TILE_M * NT / 4;
    const int S = gridDim.z, z = blockIdx.z;
    const HaloTile tl = halo_tile(p.tiles_w, p.tiles_h);
    for (int i = z * G / S + tid; i < (z + 1) * G / S; i += NUM_THREADS) {
      const uint32_t at = smem_u32(part + 4 * i);
      float4 v = ld_cluster_f4(at, 0);
      for (int q = 1; q < S; ++q) {
        const float4 u = ld_cluster_f4(at, q);
        v.x += u.x, v.y += u.y, v.z += u.z, v.w += u.w;
      }
      const int px = 4 * i / NT, c0 = 4 * i % NT;   // tile pixel, first channel
      const int oy = tl.oy0 + px / FT_W, ox = tl.ox0 + px % FT_W;
      if (oy >= p.Ho || ox >= p.Wo) continue;
      float* yrow = p.y + (((size_t)tl.n * p.Ho + oy) * p.Wo + ox) * p.y_cstride + ch.y_off;
      const float vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (c0 + e < ch.ncount) yrow[c0 + e] = finish(p, ch, c0 + e, vs[e]);
    }
    cluster_sync();   // no CTA exits while another may still read its partial tile
  } else {
    const bool pair = rows_pair_aligned(p, ch);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      long long m = m0 + arow0 + 8 * h;   // output pixel
      if (MODE == TC_HALO) {
        const HaloTile tl = halo_tile(p.tiles_w, p.tiles_h);
        const int oy = tl.oy0 + r, ox = tl.ox0 + g + 8 * h;
        if (oy >= p.Ho || ox >= p.Wo) continue;
        m = ((long long)tl.n * p.Ho + oy) * p.Wo + ox;
      } else if (m >= p.M) {
        continue;
      }
      float* yrow = p.y + (size_t)m * p.y_cstride + ch.y_off;
#pragma unroll
      for (int j = 0; j < NT / 8; ++j)
        store_pair(yrow, 8 * j + 2 * t, ch.ncount, pair,
                   [&](int c) { return finish(p, ch, c, sum[4 * j + 2 * h + (c & 1)]); });
    }
  }
}

// ---------------------------------------------------------------------------------------------
// The fire module with a 16-channel squeeze as ONE kernel: a CTA owns an 8 x 16 tile of output
// pixels of one image.
//   squeeze: 1x1 conv over the 10 x 18 halo of the tile (192 rows = three m64 blocks; warpgroup 0
//            takes blocks 0 and 2, warpgroup 1 block 1), bias + ReLU, zero outside the image (SAME
//            padding of the 3x3 expand pads the post-ReLU squeeze output), kept in shared memory
//            as Q[halo pixel][FS + 4] fp32.  Each K chunk of KCI channels brings its halo by TMA
//            through the halo-mode tensor map of conv_tc_kernel and its weight tile by one bulk copy;
//   expand:  1x1 and 3x3 convs over Q in chunks of 64 output channels; K chunk kk of a 3x3 chunk
//            is tap kk = (dy, dx), whose A fragments are read from Q at the tap-shifted halo row,
//            so the squeeze tensor never leaves the SM; one bulk copy of weights per K chunk.
// Squeeze and expand K chunks are one sequence through the mbarrier ring (squeeze chunk kk, then
// expand K chunk it as nks + it), so thread 0 prefetches the expand's first weight tiles while the
// squeeze runs; the block barrier that publishes Q is the only one after the ring is set up.
//
// The kernel reads the TcParams of a fire plan (tc_fire_plan): chunk 0 is the squeeze (Cin / KCI
// K chunks, FS output channels), chunks 1.. the 64-wide expand chunks, each with one K chunk of
// FS channels per tap; w holds the squeeze tiles [Cin / KCI][2][FS][KCI], then the expand tiles
// [taps][2][64][FS] chunk after chunk; bias is [b_sq | b_e1 | b_e3]; amap is the halo-mode map.
constexpr int FS = 16;         // squeeze channels
constexpr int FQ_ROWS = 192;   // FQ_P halo pixels padded to three m64 blocks

// fire_tc_kernel's shared memory, from a 1024-byte aligned base: STAGES x [squeeze weight tile
// 2 FS KCI][A tile FQ_ROWS x KCI] (an expand weight tile reuses the stage's first 8 KiB), then Q
// and the full and empty barrier of each stage.
__host__ __device__ constexpr int fire_stage_floats(int KCI) { return 2 * FS * KCI + FQ_ROWS * KCI; }
constexpr size_t fire_smem_bytes(int KCI) {
  return 1024 + ((size_t)STAGES * fire_stage_floats(KCI) + FQ_ROWS * (FS + 4)) * sizeof(float) +
         2 * STAGES * sizeof(uint64_t);
}

// Two CTAs per SM: at most 128 registers a thread, and 102.4 KB of shared memory at KCI = 32.
template <int KCI>
__global__ void __launch_bounds__(NUM_THREADS, 2)
fire_tc_kernel(const __grid_constant__ TcParams p) {
  constexpr int QP = FS + 4;
  constexpr int SQW = 2 * FS * KCI;   // floats of a squeeze weight tile, hi + lo
  constexpr int STAGE = fire_stage_floats(KCI);
  constexpr uint32_t SQW_BYTES = SQW * 4, HALO_BYTES = FQ_P * KCI * 4, EX_BYTES = 2 * 64 * FS * 4;
  // the expand's weight tiles leave the A tiles' rows FQ_P.. zeroed below alone
  static_assert(EX_BYTES <= (SQW + FQ_P * KCI) * 4, "expand tile fits before the zeroed rows");
  static_assert(SQW_BYTES % 1024 == 0 && STAGE * 4 % 1024 == 0, "A tiles keep the swizzle's alignment");
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float* const smem = reinterpret_cast<float*>(smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023));
  float* const q = smem + STAGES * STAGE;
  uint64_t* const full = reinterpret_cast<uint64_t*>(q + FQ_ROWS * QP);
  uint64_t* const empty = full + STAGES;

  const int tid = threadIdx.x;
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int nks = p.Cin / KCI;
  int total = 0;   // K chunks of the squeeze and every expand chunk
#pragma unroll 1
  for (int c = 0; c < p.nchunks; ++c) total += p.chunks[c].nk;
  if (tid == 0) ring_init(full, empty, 1);
  // A-tile rows FQ_P.. feed only the discarded squeeze rows; the halo box never writes them
  for (int i = tid; i < STAGES * (FQ_ROWS - FQ_P) * KCI; i += NUM_THREADS) {
    const int s = i / ((FQ_ROWS - FQ_P) * KCI);
    smem[s * STAGE + SQW + FQ_P * KCI + i % ((FQ_ROWS - FQ_P) * KCI)] = 0.f;
  }
  __syncthreads();

  // K chunk j of the sequence into its stage (thread 0): for j < nks the squeeze's halo of
  // channels [j KCI, j KCI + KCI) and weight tile, then expand K chunk j - nks's weight tile
  auto load_stage = [&](int j) {
    const int s = ring_acquire(empty, j);
    float* const st = smem + s * STAGE;
    if (j < nks) {
      const HaloTile tl = halo_tile(p.tiles_w, p.tiles_h);
      mbar_expect_tx(&full[s], SQW_BYTES + HALO_BYTES);
      tma_load(smem_u32(st + SQW), &p.amap, j * KCI, tl.ox0 - 1, tl.oy0 - 1, tl.n, &full[s]);
      bulk_load(smem_u32(st), p.w + (size_t)j * SQW, SQW_BYTES, &full[s]);
    } else {
      mbar_expect_tx(&full[s], EX_BYTES);
      bulk_load(smem_u32(st), p.w + (size_t)nks * SQW + (size_t)(j - nks) * 2 * 64 * FS, EX_BYTES,
                &full[s]);
    }
  };
  if (tid == 0) {
#pragma unroll 1
    for (int j = 0; j < STAGES - 1 && j < total; ++j) load_stage(j);
  }

  // ---- squeeze
  float accq[2][FS / 2], sq[2][FS / 2];
#pragma unroll
  for (int i = 0; i < FS / 2; ++i) accq[0][i] = accq[1][i] = sq[0][i] = sq[1][i] = 0.f;
  const int rb = wq * 16 + g;
  for (int kk = 0; kk < nks; ++kk) {
    if (tid == 0 && kk + STAGES - 1 < total) load_stage(kk + STAGES - 1);
    const float* st = smem + ring_wait_full(full, kk) * STAGE;
    const float* sa = st + SQW;
    if (wg == 0) {
      // blocks 0 and 2 interleaved, block 2 * bi in accumulator set bi: one block's step is in
      // flight while the other block's previous step is added in; drained like mma_chunk
      uint32_t qhi[2][4], qlo[2][4];
#pragma unroll
      for (int j = 0; j < 2 * (KCI / 8); ++j) {
        const int bi = j & 1, ks = j >> 1;
        load_split_swz<KCI>(sa, 128 * bi + rb, ks, t, qhi[bi], qlo[bi]);
        mma_step<FS, KCI>(accq[bi], qhi[bi], qlo[bi], smem_u32(st), ks);
        if (j > 0) {
          wgmma_wait<1>();
          flush(accq[bi ^ 1], sq[bi ^ 1], qhi[bi ^ 1], qlo[bi ^ 1]);
        }
      }
      wgmma_wait<0>();
      flush(accq[1], sq[1], qhi[1], qlo[1]);
    } else {
      mma_chunk<FS, KCI>(
          [&](int ks, uint32_t(&ahi)[4], uint32_t(&alo)[4]) {
            load_split_swz<KCI>(sa, 64 + rb, ks, t, ahi, alo);
          },
          smem_u32(st), accq, sq[0]);
    }
    ring_release(empty, kk);
  }
  {
    const HaloTile tl = halo_tile(p.tiles_w, p.tiles_h);
#pragma unroll
    for (int bi = 0; bi < 2; ++bi) {
      const int b = wg + 2 * bi;
      if (b >= 3) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = b * 64 + wq * 16 + g + 8 * h;
        const int iy = tl.oy0 - 1 + row / FQ_W, ix = tl.ox0 - 1 + row % FQ_W;
        const bool ok = row < FQ_P && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
#pragma unroll
        for (int j = 0; j < FS / 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 8 * j + 2 * t + e;
            q[row * QP + c] = ok ? fmaxf(sq[bi][4 * j + 2 * h + e] + p.bias[c], 0.f) : 0.f;
          }
      }
    }
  }
  __syncthreads();   // Q complete

  // ---- expand: pixel rows g / g + 8 of this warp are tile row (4 wg + wq), columns g / g + 8
  const int r = wg * 4 + wq;
  float acc[2][32], sum[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[0][i] = acc[1][i] = sum[i] = 0.f;
  int c = 1, kk = 0;
  for (int j = nks; j < total; ++j) {
    if (tid == 0 && j + STAGES - 1 < total) load_stage(j + STAGES - 1);
    const int s = ring_wait_full(full, j);
    const TcChunk& ch = p.chunks[c];   // nk: its taps, one K chunk of FS channels each
    const int dy = ch.nk == 1 ? 1 : kk / 3, dx = ch.nk == 1 ? 1 : kk % 3;
    const int qr = (r + dy) * FQ_W + g + dx;
    mma_chunk<64, FS>(
        [&](int ks, uint32_t(&ahi)[4], uint32_t(&alo)[4]) {
          load_split(q + qr * QP, q + (qr + 8) * QP, ks, t, ahi, alo);
        },
        smem_u32(smem + s * STAGE), acc, sum);
    ring_release(empty, j);
    if (++kk == ch.nk) {
      const HaloTile tl = halo_tile(p.tiles_w, p.tiles_h);
      const int oy = tl.oy0 + r;
      const size_t prow = ((size_t)tl.n * p.H + oy) * p.W;
      const bool pair = rows_pair_aligned(p, ch);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ox = tl.ox0 + g + 8 * h;
        if (oy >= p.H || ox >= p.W) continue;
        float* yrow = p.y + (prow + ox) * p.y_cstride + ch.y_off;
#pragma unroll
        for (int jn = 0; jn < 8; ++jn)
          store_pair(yrow, 8 * jn + 2 * t, ch.ncount, pair, [&](int col) {
            return fmaxf(sum[4 * jn + 2 * h + (col & 1)] + p.bias[ch.p_off + col], 0.f);
          });
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) sum[i] = 0.f;
      kk = 0;
      ++c;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Host side
using TcKernel = void (*)(TcParams);

template <int KC, int MODE>
TcKernel conv_tc_instance(int NT) {
  return NT == 64 ? conv_tc_kernel<64, KC, MODE>
         : NT == 32 ? conv_tc_kernel<32, KC, MODE> : conv_tc_kernel<16, KC, MODE>;
}

// The conv_tc_kernel instantiation of a plan (gather mode always walks K in chunks of 32; the
// 72-wide head tile only comes with KC = 32).
TcKernel conv_tc_instance(int NT, int KC, int mode) {
  if (NT == 72) return mode == TC_HALO ? conv_tc_kernel<72, 32, TC_HALO> : conv_tc_kernel<72, 32, TC_ROWS>;
  if (mode == TC_GATHER) return conv_tc_instance<32, TC_GATHER>(NT);
  if (mode == TC_HALO)
    return KC == 32 ? conv_tc_instance<32, TC_HALO>(NT) : conv_tc_instance<16, TC_HALO>(NT);
  return KC == 32 ? conv_tc_instance<32, TC_ROWS>(NT) : conv_tc_instance<16, TC_ROWS>(NT);
}

// One conv of a plan: its output channels in chunks [chunk0, chunk0 + ceil(Cout / NT)) of NT,
// its K over its cin input channels in chunks of KC.
struct PlanGroup {
  ConvGroup conv;
  int NT, KC, cin, chunk0;
};

}  // namespace

struct TcImpl {
  TcParams prm{};
  int KC = 0;          // channels of a box of the input's tensor maps
  int mode = TC_ROWS;
  TcKernel kernel = nullptr;
  int ksplit = 1;      // CTAs of a cluster that split K (kernel is then the KSPLIT instance)
  size_t smem_bytes = 0;
  std::vector<PlanGroup> groups;
  int cout_total = 0;
  float* d_w = nullptr;
  float* d_bias = nullptr;
  float* d_scale = nullptr;
  float* d_shift = nullptr;
  long long w_floats = 0;
  // the input and image count prm's tensor maps were encoded for (null: none yet)
  const float* map_x = nullptr;
  int map_n = 0;
};

static inline float host_rn_tf32(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  u = (u + 0x1000u) & 0xFFFFE000u;
  float r;
  memcpy(&r, &u, 4);
  return r;
}

// Output-channel tile: the narrowest of 16 / 32 / 64 that covers the launch's chunks with the
// least padded MMA work plus A-tile re-reads (each chunk reloads the pixels' K values).  A
// 72-wide tile is also a candidate for one conv of 65..72 output channels walked in 32-channel
// K chunks, the ConvDet head (9 anchors x 8 values), which it covers in one chunk instead of
// two 64-wide ones that are 44 % padding.
static int pick_nt(const std::vector<ConvGroup>& groups, int KC, bool gather) {
  int best = 0;
  long long best_cost = 0;
  const bool head = !gather && KC == 32 && groups.size() == 1 && groups[0].Cout > 64 &&
                    groups[0].Cout <= 72;
  for (int nt : {72, 64, 32, 16}) {
    if (nt == 72 && !head) continue;
    long long chunks = 0;
    for (const auto& g : groups) chunks += (g.Cout + nt - 1) / nt;
    if (chunks > MAX_CHUNKS) continue;
    const long long cost = chunks * (nt + 32);
    if (!best || cost < best_cost) best = nt, best_cost = cost;
  }
  return best;
}

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

// A tiled tensor map over the fp32 tensor at x: `rank` dims (innermost first, dims[0] the
// channels) of densely packed `dims`, boxes of `box`, stored with the swizzle the kernel reads
// KC-channel rows with; elements outside the tensor read as zero.
static int encode_map(CUtensorMap* map, const float* x, int rank, const cuuint64_t* dims,
                      const cuuint32_t* box, int KC) {
  static EncodeTiledFn encode = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      fn = nullptr;
    return reinterpret_cast<EncodeTiledFn>(fn);
  }();
  if (!encode) return fail(SQDET_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  cuuint64_t strides[3];
  cuuint64_t stride = sizeof(float);
  for (int i = 0; i + 1 < rank; ++i) strides[i] = stride *= dims[i];
  const cuuint32_t elem_strides[4] = {1, 1, 1, 1};
  const CUresult rc = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<float*>(x), dims, strides,
                             box, elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             KC == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS)
    return fail(SQDET_ERR_CUDA, "cuTensorMapEncodeTiled failed (error " + std::to_string((int)rc) + ")");
  return SQDET_OK;
}

// A (C, W, H, n) map over n NHWC images of H x W x C at x, with (KC, box_w, box_h, 1) boxes.
static int encode_nhwc_map(CUtensorMap* map, const float* x, int n, int H, int W, int C, int KC,
                           int box_w, int box_h) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)n};
  const cuuint32_t box[4] = {(cuuint32_t)KC, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  return encode_map(map, x, 4, dims, box, KC);
}

// Encodes the plan's tensor maps for input x of n images, unless they already are: row mode its
// row map; halo mode and the fire the halo map, halo mode also the map of a 1x1 conv's tile.
static int update_maps(TcImpl* im, const float* x, int n) {
  if (im->mode == TC_GATHER || (im->map_x == x && im->map_n == n)) return SQDET_OK;
  TcParams& p = im->prm;
  im->map_x = nullptr;
  int rc;
  if (im->mode == TC_ROWS) {
    const cuuint64_t dims[2] = {(cuuint64_t)p.Cin, (cuuint64_t)n * p.H * p.W};
    const cuuint32_t box[2] = {(cuuint32_t)im->KC, TILE_M};
    rc = encode_map(&p.amap, x, 2, dims, box, im->KC);
  } else {
    rc = encode_nhwc_map(&p.amap, x, n, p.H, p.W, p.Cin, im->KC, FQ_W, 10);
    if (!rc && im->mode == TC_HALO) rc = encode_nhwc_map(&p.amap1, x, n, p.H, p.W, p.Cin, im->KC, FT_W, 8);
  }
  if (rc) return rc;
  im->map_x = x;
  im->map_n = n;
  return SQDET_OK;
}

// The grid's CTAs over n images: one per 8 x FT_W output tile in halo mode and the fire, one per
// TILE_M output pixels otherwise.
static long long grid_blocks(const TcImpl* im, int n) {
  const TcParams& p = im->prm;
  if (im->mode == TC_HALO || im->mode == TC_FIRE) return (long long)n * p.tiles_h * p.tiles_w;
  return ((long long)n * p.Ho * p.Wo + TILE_M - 1) / TILE_M;
}

// Plans the convs of im->groups over one [B, H, W, Cin] input into a [B, Ho, Wo, y_cstride]
// output, for the mode, kernel and group tiling already in im: their chunks, the kernel's shared
// memory, and the weight, bias and affine buffers.  Returns 1 (planned), 0 (declined) or a
// negative status.
//
// The chunks follow group order, except that halo mode numbers its 3x3 convs' chunks first.  The
// block scheduler starts a grid's CTAs in blockIdx order, so an expand pair's long 3x3 CTAs (9x
// the K chunks of its 1x1 CTAs) start first and the short 1x1 CTAs fill the last wave, instead of
// a last wave of 3x3 CTAs running on a partly idle GPU.
static int plan_common(TcImpl* im, int B, int H, int W, int Cin, int Ho, int Wo, int stride,
                       int pad_t, int pad_l, int relu, bool has_affine, int y_cstride) {
  const bool gather = im->mode == TC_GATHER;
  TcParams& p = im->prm;
  p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Ho = Ho; p.Wo = Wo; p.stride = stride;
  p.relu = relu; p.y_cstride = y_cstride; p.M = (long long)B * Ho * Wo;
  p.tiles_w = (Wo + FT_W - 1) / FT_W; p.tiles_h = (Ho + 7) / 8;
  if (p.M <= 0 || grid_blocks(im, B) > 0x7fffffffLL) return 0;
  // each group's first bias / scale / shift entry, in group order (tc_conv_pack_weights)
  std::vector<int> poffs;
  int poff = 0;
  for (const auto& g : im->groups) poffs.push_back(poff), poff += g.conv.Cout;
  std::vector<size_t> order;
  for (int pass = 0; pass < 2; ++pass)
    for (size_t gi = 0; gi < im->groups.size(); ++gi)
      if ((im->mode == TC_HALO && im->groups[gi].conv.ksize == 3) == (pass == 0)) order.push_back(gi);
  int nch = 0;
  long long woff = 0;
  for (const size_t gi : order) {
    PlanGroup& g = im->groups[gi];
    g.chunk0 = nch;
    const int taps = g.conv.ksize * g.conv.ksize;
    const int nk = gather ? (taps * g.cin + g.KC - 1) / g.KC : taps * (g.cin / g.KC);
    for (int cb = 0; cb < g.conv.Cout; cb += g.NT, ++nch) {
      TcChunk& c = p.chunks[nch];
      c.ksize = g.conv.ksize;
      c.pad_t = gather ? pad_t : g.conv.ksize / 2;
      c.pad_l = gather ? pad_l : g.conv.ksize / 2;
      c.nk = nk;
      c.ncount = g.conv.Cout - cb < g.NT ? g.conv.Cout - cb : g.NT;
      c.y_off = g.conv.y_off + cb;
      c.p_off = poffs[gi] + cb;
      c.w_off = woff;
      woff += (long long)nk * 2 * g.NT * g.KC;
    }
  }
  p.nchunks = nch;
  im->cout_total = poff;
  im->w_floats = woff;
  cudaError_t ce = cudaFuncSetAttribute(im->kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)im->smem_bytes);
  if (ce != cudaSuccess) return cuda_fail(ce, "cudaFuncSetAttribute(tensor-core kernel)");
  SQ_CUDA(cudaMalloc(&im->d_w, sizeof(float) * (size_t)woff));
  SQ_CUDA(cudaMalloc(&im->d_bias, sizeof(float) * poff));
  SQ_CUDA(cudaMemset(im->d_bias, 0, sizeof(float) * poff));
  if (has_affine) {
    SQ_CUDA(cudaMalloc(&im->d_scale, sizeof(float) * poff));
    SQ_CUDA(cudaMalloc(&im->d_shift, sizeof(float) * poff));
  }
  p.w = im->d_w;
  p.bias = im->d_bias;
  p.scale = im->d_scale;
  p.shift = im->d_shift;
  return 1;
}

// Packs K chunks [0, nk) of one output-channel chunk [n0, n0 + NT) of a weight matrix whose rows
// are the flattened HWIO K index (tap * Cin + channel, `kreal` of them) into the tiles the
// kernels read: per K chunk [NT/8 row groups][KC/4 K core matrices][8 rows][4 floats], hi tile
// then lo tile.  Rows past `kreal` and channels past `cout` are zero.  With taps == 1 K chunk kk
// holds rows [kk * KC, kk * KC + KC); otherwise the chunks walk channel chunk c with the taps
// inner (the halo-mode order): K chunk c * taps + tap holds rows tap * cin + c * KC + [0, KC).
static void pack_tiles(const float* w, long long kreal, int cout, int n0, int NT, int KC, int nk,
                       int taps, int cin, float* dst) {
  for (int kk = 0; kk < nk; ++kk) {
    float* hi_t = dst + (size_t)kk * 2 * NT * KC;
    float* lo_t = hi_t + NT * KC;
    const long long k0 = (long long)(kk % taps) * cin + (long long)(kk / taps) * KC;
    for (int n = 0; n < NT; ++n)
      for (int k = 0; k < KC; ++k) {
        const long long kg = k0 + k;
        const float v = (n0 + n < cout && kg < kreal) ? w[kg * cout + n0 + n] : 0.f;
        const float hi = host_rn_tf32(v);
        const size_t at = ((size_t)(n / 8) * (KC / 4) + k / 4) * 32 + (n % 8) * 4 + k % 4;
        hi_t[at] = hi;
        lo_t[at] = host_rn_tf32(v - hi);
      }
  }
}

// Packs group g's weights (HWIO [k, k, cin, Cout]) into each of its chunks' tiles: a 3x3 conv
// channel chunk by channel chunk with the taps inner (in the fire's expand, whose K chunks are
// the squeeze's FS channels, that is the flat HWIO order), a 1x1 conv and gather mode the
// flattened K rows in order.
static void pack_group(const TcImpl* im, const PlanGroup& g, const float* w_hwio, std::vector<float>& packed) {
  const int taps = im->mode == TC_GATHER ? 1 : g.conv.ksize * g.conv.ksize;
  int ci = g.chunk0;
  for (int cb = 0; cb < g.conv.Cout; cb += g.NT, ++ci) {
    const TcChunk& c = im->prm.chunks[ci];
    pack_tiles(w_hwio, (long long)g.conv.ksize * g.conv.ksize * g.cin, g.conv.Cout, cb, g.NT, g.KC,
               c.nk, taps, g.cin, packed.data() + c.w_off);
  }
}

// A launch of `grid` whose clusters are the S CTAs along z that split K (S = 1: no cluster).
struct ClusterLaunch {
  cudaLaunchAttribute attr;
  cudaLaunchConfig_t cfg;
  ClusterLaunch(dim3 grid, size_t smem, int S, cudaStream_t stream) : attr{}, cfg{} {
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = (unsigned)S;
    cfg.gridDim = dim3(grid.x, grid.y, grid.z * S);
    cfg.blockDim = dim3(NUM_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
  }
};

constexpr int MAX_KSPLIT = 4;
constexpr int MIN_RANK_CHUNKS = 4;   // channel chunks a rank walks at the least when S is chosen

// The K split of a 72-wide halo-mode plan (the ConvDet head, whose few long tiles leave a short
// last wave: 300 tiles on 264 CTA slots at b = 20, 120 on 264 at b = 8).  forced == 0 picks, for the planned B,
// the S in 1..MAX_KSPLIT with the fewest waves of S-CTA clusters over the device's resident
// clusters, counting a wave of split CTAs as 1/S of a whole one and keeping the smaller S on a
// tie, among the S that leave every rank MIN_RANK_CHUNKS channel chunks.  forced > 0 takes that
// S, at most one rank per channel chunk.
static int plan_ksplit(TcImpl* im, int forced) {
  const TcKernel split = conv_tc_kernel<72, 32, TC_HALO, true>;
  const int nc = im->prm.chunks[0].nk / 9;
  if (forced < 0 || forced > MAX_KSPLIT || forced > nc)
    return fail(SQDET_ERR_INVALID_ARG, "K split outside [1, min(4, channel chunks)]");
  SQ_CUDA(cudaFuncSetAttribute(split, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)im->smem_bytes));
  int S = forced;
  if (!forced) {
    int dev = 0, sms = 0, per_sm = 0;
    SQ_CUDA(cudaGetDevice(&dev));
    SQ_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    SQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, im->kernel, NUM_THREADS, im->smem_bytes));
    const long long ctas = grid_blocks(im, im->prm.B) * im->prm.nchunks;
    S = 1;
    long long best_waves = (ctas + per_sm * sms - 1) / (per_sm * sms);
    for (int s = 2; s <= MAX_KSPLIT && s * MIN_RANK_CHUNKS <= nc; ++s) {
      // clusters of s resident at once: a cluster's CTAs share one GPC, whose SM count need not
      // be a multiple of s
      int clusters = 0;
      const ClusterLaunch l(dim3(1), im->smem_bytes, s, nullptr);
      SQ_CUDA(cudaOccupancyMaxActiveClusters(&clusters, split, &l.cfg));
      if (clusters < 1) continue;
      const long long waves = (ctas + clusters - 1) / clusters;
      if (waves * S < best_waves * s) S = s, best_waves = waves;   // waves / s < best_waves / S
    }
  }
  if (S > 1) im->kernel = split;
  im->ksplit = S;
  return 1;
}

// ---------------------------------------------------------------------------------------------
bool tc_conv_eligible(int Cin, int Cout, int size, int stride, int padding) {
  // shapes this path takes: stride-1 SAME, 1x1 or 3x3, Cin a multiple of 16
  if (stride != 1 || padding != SQDET_PAD_SAME || (size != 1 && size != 3)) return false;
  return Cin % 16 == 0 && Cin >= 16 && Cout > 0;
}

int tc_conv_plan(TcConvPlan* plan, int B, int H, int W, int Cin, const std::vector<ConvGroup>& convs,
                 int stride, int padding, int relu, bool has_affine, int y_cstride, int k_split) {
  plan->impl = nullptr;
  const int size = convs[0].ksize;
  const bool gather = convs.size() == 1 && Cin == 3 && size == 3 && (stride == 1 || stride == 2) &&
                      convs[0].Cout > 0;
  if (!gather)
    for (const auto& g : convs)
      if (!tc_conv_eligible(Cin, g.Cout, g.ksize, stride, padding)) return 0;
  const Geom gh = tf_geometry(H, size, stride, padding);
  const Geom gw = tf_geometry(W, size, stride, padding);
  if (gh.out <= 0 || gw.out <= 0) return 0;
  const int KC = (gather || Cin % 32 == 0) ? 32 : 16;
  const int NT = pick_nt(convs, KC, gather);
  if (!NT) return 0;
  int mode = gather ? TC_GATHER : TC_ROWS;
  for (const auto& g : convs)
    if (!gather && g.ksize == 3) mode = TC_HALO;   // stride-1 SAME (tc_conv_eligible)
  TcImpl* im = plan->impl = new TcImpl();
  im->KC = KC;
  im->mode = mode;
  im->kernel = conv_tc_instance(NT, KC, mode);
  im->smem_bytes = conv_smem_bytes(NT, KC);
  for (const auto& g : convs) im->groups.push_back({g, NT, KC, Cin, 0});
  int rc = plan_common(im, B, H, W, Cin, gh.out, gw.out, stride, gh.pad_before, gw.pad_before,
                       relu, has_affine, y_cstride);
  if (rc > 0 && NT == 72 && mode == TC_HALO) {
    rc = plan_ksplit(im, k_split);
  } else if (rc > 0 && k_split > 1) {
    rc = fail(SQDET_ERR_INVALID_ARG, "a K split needs a 72-wide 3x3 tensor-core plan");
  }
  if (rc <= 0) tc_conv_release(plan);
  return rc;
}

int tc_conv_k_split(const TcConvPlan& plan) { return plan.impl ? plan.impl->ksplit : 1; }

int tc_fire_plan(TcConvPlan* plan, int B, int H, int W, int Cin, int S, int E1, int E3) {
  plan->impl = nullptr;
  if (Cin % 16 || Cin < 16 || S != FS || E1 <= 0 || E3 <= 0) return 0;
  if ((E1 + 63) / 64 + (E3 + 63) / 64 > 16) return 0;   // expand chunks of 64 channels
  const int KCI = Cin % 32 == 0 ? 32 : 16;
  TcImpl* im = plan->impl = new TcImpl();
  im->KC = KCI;
  im->mode = TC_FIRE;
  im->kernel = KCI == 32 ? fire_tc_kernel<32> : fire_tc_kernel<16>;
  im->smem_bytes = fire_smem_bytes(KCI);
  // chunk 0 the squeeze, then the 64-wide expand chunks, expand1x1's before expand3x3's
  im->groups = {{{1, FS, 0}, FS, KCI, Cin, 0}, {{1, E1, 0}, 64, FS, FS, 0}, {{3, E3, E1}, 64, FS, FS, 0}};
  const int rc = plan_common(im, B, H, W, Cin, H, W, 1, 0, 0, 1, false, E1 + E3);
  if (rc <= 0) tc_conv_release(plan);
  return rc;
}

int tc_conv_pack_weights(TcConvPlan* plan, const std::vector<const float*>& w_hwio,
                         const std::vector<const float*>& bias) {
  TcImpl* im = plan->impl;
  std::vector<float> packed((size_t)im->w_floats, 0.f);
  for (size_t gi = 0; gi < im->groups.size(); ++gi) pack_group(im, im->groups[gi], w_hwio[gi], packed);
  SQ_CUDA(cudaMemcpy(im->d_w, packed.data(), packed.size() * sizeof(float), cudaMemcpyHostToDevice));
  int off = 0;
  for (size_t gi = 0; gi < im->groups.size(); ++gi) {
    const int n = im->groups[gi].conv.Cout;
    if (bias[gi]) SQ_CUDA(cudaMemcpy(im->d_bias + off, bias[gi], sizeof(float) * n, cudaMemcpyHostToDevice));
    off += n;
  }
  return SQDET_OK;
}

int tc_conv_set_affine(TcConvPlan* plan, const float* scale, const float* shift) {
  TcImpl* im = plan->impl;
  if (!im->d_scale) return fail(SQDET_ERR_STATE, "tc conv planned without an affine epilogue");
  SQ_CUDA(cudaMemcpy(im->d_scale, scale, sizeof(float) * im->cout_total, cudaMemcpyHostToDevice));
  SQ_CUDA(cudaMemcpy(im->d_shift, shift, sizeof(float) * im->cout_total, cudaMemcpyHostToDevice));
  return SQDET_OK;
}

int launch_conv_tc(const TcConvPlan& plan, const float* x_dev, float* y_dev, int n,
                   cudaStream_t stream) {
  TcImpl* im = plan.impl;
  if (n < 1 || n > im->prm.B) return fail(SQDET_ERR_INVALID_ARG, "launch_conv_tc: image count outside [1, B]");
  const int rc = update_maps(im, x_dev, n);
  if (rc) return rc;
  TcParams prm = im->prm;
  prm.x = x_dev;
  prm.y = y_dev;
  prm.B = n;
  prm.M = (long long)n * prm.Ho * prm.Wo;
  // a fire CTA walks every chunk of its tile
  const dim3 grid((unsigned)grid_blocks(im, n), im->mode == TC_FIRE ? 1u : (unsigned)prm.nchunks);
  if (im->ksplit > 1) {
    const ClusterLaunch l(grid, im->smem_bytes, im->ksplit, stream);
    SQ_CUDA(cudaLaunchKernelEx(&l.cfg, im->kernel, prm));
  } else {
    im->kernel<<<grid, NUM_THREADS, im->smem_bytes, stream>>>(prm);
  }
  SQ_CHECK_LAUNCH(im->mode == TC_FIRE ? "fire_tc_kernel" : "conv_tc_kernel");
  return SQDET_OK;
}

void tc_conv_release(TcConvPlan* plan) {
  TcImpl* im = plan->impl;
  if (!im) return;
  cudaFree(im->d_w);
  cudaFree(im->d_bias);
  cudaFree(im->d_scale);
  cudaFree(im->d_shift);
  delete im;
  plan->impl = nullptr;
}

int tc_conv_oneshot(TcConvPlan* plan, const std::vector<const float*>& w_hwio_dev,
                    const std::vector<const float*>& bias_dev, const float* scale_dev,
                    const float* shift_dev, const float* x_dev, float* y_dev, cudaStream_t stream) {
  TcImpl* im = plan->impl;
  if (!im) return 1;
  const size_t ng = im->groups.size();
  std::vector<std::vector<float>> w(ng), b(ng);
  std::vector<float> sc, sh;
  std::vector<const float*> w_host(ng), b_host(ng);
  cudaError_t ce = cudaSuccess;
  auto download = [&ce](std::vector<float>& dst, const float* src, size_t n) {
    dst.resize(n);
    if (ce == cudaSuccess) ce = cudaMemcpy(dst.data(), src, n * sizeof(float), cudaMemcpyDeviceToHost);
    return dst.data();
  };
  for (size_t gi = 0; gi < ng; ++gi) {
    const ConvGroup& g = im->groups[gi].conv;
    w_host[gi] = download(w[gi], w_hwio_dev[gi], (size_t)g.ksize * g.ksize * im->groups[gi].cin * g.Cout);
    b_host[gi] = bias_dev[gi] ? download(b[gi], bias_dev[gi], g.Cout) : nullptr;
  }
  if (scale_dev) download(sc, scale_dev, im->cout_total), download(sh, shift_dev, im->cout_total);
  int rc = ce == cudaSuccess ? tc_conv_pack_weights(plan, w_host, b_host)
                             : cuda_fail(ce, "tc_conv_oneshot: parameter download");
  if (!rc && scale_dev) rc = tc_conv_set_affine(plan, sc.data(), sh.data());
  if (!rc) rc = launch_conv_tc(*plan, x_dev, y_dev, im->prm.B, stream);
  ce = cudaStreamSynchronize(stream);
  tc_conv_release(plan);
  if (rc) return rc;
  if (ce != cudaSuccess) return cuda_fail(ce, "tc_conv_oneshot sync");
  return SQDET_OK;
}

}  // namespace sqdet
