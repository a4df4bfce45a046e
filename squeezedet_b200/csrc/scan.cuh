// Block-wide exclusive scan shared by the entropy coders (jpeg.cu, png.cu).
#pragma once
#include "common.cuh"

namespace sqdet {

struct ScanSum {
  static constexpr int64_t kIdentity = 0;
  __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a + b; }
};
struct ScanMax {
  static constexpr int64_t kIdentity = INT64_MIN;
  __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a > b ? a : b; }
};

// Exclusive scan of v under Op over the CTA's threads (blockDim.x a multiple of 32, at most 1024);
// *total gets the reduction of all of them.  Ends with a barrier, so `warp` may be reused right
// after.
template <class Op = ScanSum>
__device__ int64_t block_exclusive_scan(int64_t v, int64_t* warp, int64_t* total, Op op = Op()) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int64_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x = op(x, y);
  }
  if (lane == 31) warp[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int64_t w = lane < nw ? warp[lane] : Op::kIdentity;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w = op(w, y);
    }
    if (lane < nw) warp[lane] = w;
  }
  __syncthreads();
  // the inclusive value of the lanes before this one, then the warps before this one's
  int64_t before = __shfl_up_sync(0xffffffffu, x, 1);
  if (lane == 0) before = Op::kIdentity;
  if (wid) before = op(warp[wid - 1], before);
  *total = warp[nw - 1];
  __syncthreads();
  return before;
}

}  // namespace sqdet
