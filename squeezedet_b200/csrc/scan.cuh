// Block-wide exclusive scan shared by the entropy coders (jpeg.cu, png.cu), the JPEG decoder
// (jpeg_decode.cu) and the KITTI evaluation (kitti_eval.cu).
#pragma once
#include <type_traits>

#include "common.cuh"

namespace sqdet {

struct ScanSum {
  static constexpr int64_t kIdentity = 0;
  template <class T>
  __device__ __forceinline__ T operator()(T a, T b) const { return a + b; }
};
struct ScanMax {                       // int64_t scans only
  static constexpr int64_t kIdentity = INT64_MIN;
  __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a > b ? a : b; }
};

// Exclusive scan of v under Op over the CTA's threads (blockDim.x a multiple of 32, at most 1024);
// *total gets the reduction of all of them.  T (int32_t or int64_t) is the type of `warp` and
// `total`; v converts to it.  Ends with a barrier, so `warp` may be reused right after.
template <class T, class Op = ScanSum>
__device__ T block_exclusive_scan(std::common_type_t<T> v, T* warp, T* total, Op op = Op()) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x = op(x, y);
  }
  if (lane == 31) warp[wid] = x;
  __syncthreads();
  if (wid == 0) {
    T w = lane < nw ? warp[lane] : T(Op::kIdentity);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w = op(w, y);
    }
    if (lane < nw) warp[lane] = w;
  }
  __syncthreads();
  // the inclusive value of the lanes before this one, then the warps before this one's
  T before = __shfl_up_sync(0xffffffffu, x, 1);
  if (lane == 0) before = T(Op::kIdentity);
  if (wid) before = op(warp[wid - 1], before);
  *total = warp[nw - 1];
  __syncthreads();
  return before;
}

}  // namespace sqdet
