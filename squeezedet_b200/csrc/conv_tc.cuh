// wgmma (Hopper tensor core) convolution path: plans, weight packing, launchers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

namespace sqdet {

// One conv of an implicit-GEMM launch: all convs of a launch read the same input and write
// channels [y_off, y_off + Cout) of the same output.
struct ConvGroup {
  int ksize, Cout, y_off;
};

// Convs over one input executed as one implicit GEMM on wgmma with the 3xTF32 split: a single
// conv, or a fire module's expand pair (1x1 || 3x3 on the squeeze tensor) writing the
// channel-concatenated output.  A null impl means "not planned".
struct TcConvPlan {
  void* impl = nullptr;          // opaque device/host state (packed weights, launch parameters)
};

bool tc_conv_eligible(int Cin, int Cout, int size, int stride, int padding);

// Returns 1 when the tensor-core path takes the convs (plan->impl set), 0 when they are left to
// the fp32 SIMT kernel, negative on error.  Gather mode (3-channel input) takes a single conv.
int tc_conv_plan(TcConvPlan* plan, int B, int H, int W, int Cin, const std::vector<ConvGroup>& convs,
                 int stride, int padding, int relu, bool has_affine, int y_cstride);
// HWIO weights and bias (or null) of each planned conv, in plan order.
int tc_conv_pack_weights(TcConvPlan* plan, const std::vector<const float*>& w_hwio,
                         const std::vector<const float*>& bias);
int tc_conv_set_affine(TcConvPlan* plan, const float* scale, const float* shift);
// Runs the plan over images [0, n) of its batch, 1 <= n <= the planned B: the same kernel and
// chunks, with M = n * Ho * Wo and the grid sized to it.
int launch_conv_tc(const TcConvPlan& plan, const float* x_dev, float* y_dev, int n,
                   cudaStream_t stream);
void tc_conv_release(TcConvPlan* plan);

// The whole fire module (squeeze 1x1 -> expand 1x1 || 3x3 + concat) as ONE kernel: the squeeze
// tile of each 8 x 16 output tile stays in shared memory.  Cin % 16 == 0, S == 16, at most 16
// expand chunks of 64 channels.  The plan caches the tensor map of its last (input, image count).
struct TcFusedFirePlan {
  void* impl = nullptr;
};
int tc_fused_fire_plan(TcFusedFirePlan* plan, int B, int H, int W, int Cin, int S, int E1, int E3);
int tc_fused_fire_pack_weights(TcFusedFirePlan* plan, const float* w_sq, const float* b_sq,
                               const float* w_e1, const float* b_e1, const float* w_e3,
                               const float* b_e3);
// Runs the plan over images [0, n) of its batch, 1 <= n <= the planned B: n * tiles blocks.
int launch_fused_fire_tc(const TcFusedFirePlan& plan, const float* x_dev, float* y_dev, int n,
                         cudaStream_t stream);
void tc_fused_fire_release(TcFusedFirePlan* plan);
// Stage-isolated one-kernel fire from device weights; synchronises.  Returns 1 when the shape is
// not taken by the kernel.
int fire_fused_oneshot(const float* x_dev, const float* w_sq_dev, const float* b_sq_dev,
                       const float* w_e1_dev, const float* b_e1_dev, const float* w_e3_dev,
                       const float* b_e3_dev, float* y_dev, int B, int H, int W, int Cin, int S,
                       int E1, int E3, cudaStream_t stream);

// Stage-isolated entry (sqdet_conv2d with SQDET_MATH_TF32X3_TC): plans, packs from device
// weights, launches, and releases; synchronises the stream (test/debug path, not the hot path).
int conv2d_tc_oneshot(const float* x_dev, const float* w_hwio_dev, const float* bias_dev,
                      const float* scale_dev, const float* shift_dev, float* y_dev, int B, int H,
                      int W, int Cin, int Cout, int size, int stride, int padding, int relu,
                      int y_cstride, int y_coff, cudaStream_t stream);

}  // namespace sqdet
