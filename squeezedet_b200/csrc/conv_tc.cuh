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

struct TcImpl;   // a plan's device and host state (packed weights, launch parameters)

// Convs over one input executed as one wgmma launch with the 3xTF32 split: a single conv, a fire
// module's expand pair (1x1 || 3x3 on the squeeze tensor) writing the channel-concatenated
// output, or a whole fire module (tc_fire_plan).  A null impl means "not planned".
struct TcConvPlan {
  TcImpl* impl = nullptr;
};

bool tc_conv_eligible(int Cin, int Cout, int size, int stride, int padding);

// Returns 1 when the tensor-core path takes the convs (plan->impl set), 0 when they are left to
// the fp32 SIMT kernel, negative on error.  Gather mode (3-channel input) takes a single conv.
// A single 3x3 conv of 65..72 output channels (the ConvDet head) may split its K over a cluster
// of S CTAs: k_split 0 chooses S from B and the device's resident clusters, 1..4 forces it (an
// error for any other plan when above 1).  S stays fixed for every image count the plan runs.
int tc_conv_plan(TcConvPlan* plan, int B, int H, int W, int Cin, const std::vector<ConvGroup>& convs,
                 int stride, int padding, int relu, bool has_affine, int y_cstride, int k_split = 0);
// The plan's K split S (1 when unsplit or not planned).
int tc_conv_k_split(const TcConvPlan& plan);
// The whole fire module (squeeze 1x1 -> expand 1x1 || 3x3 + concat into E1 + E3 channels) as ONE
// kernel: the squeeze tile of each 8 x 16 output tile stays in shared memory.  Takes Cin % 16 ==
// 0, S == 16 and at most 16 expand chunks of 64 channels; returns as tc_conv_plan.  Its convs, in
// plan order, are the squeeze, expand1x1 and expand3x3.
int tc_fire_plan(TcConvPlan* plan, int B, int H, int W, int Cin, int S, int E1, int E3);
// HWIO weights and bias (or null) of each planned conv, in plan order.
int tc_conv_pack_weights(TcConvPlan* plan, const std::vector<const float*>& w_hwio,
                         const std::vector<const float*>& bias);
int tc_conv_set_affine(TcConvPlan* plan, const float* scale, const float* shift);
// Runs the plan over images [0, n) of its batch, 1 <= n <= the planned B: the same kernel and
// chunks on a grid sized to n.  The plan caches the tensor maps of its last (input, image count).
int launch_conv_tc(const TcConvPlan& plan, const float* x_dev, float* y_dev, int n,
                   cudaStream_t stream);
void tc_conv_release(TcConvPlan* plan);

// Stage-isolated run of a plan over its whole batch (test / debug path, not the hot path):
// downloads the device HWIO weights and biases (or null) of each conv in plan order and the
// affine scale / shift (or null), packs them, launches, synchronises the stream and releases the
// plan.  Returns 1, running nothing, when the plan was declined (null impl).
int tc_conv_oneshot(TcConvPlan* plan, const std::vector<const float*>& w_hwio_dev,
                    const std::vector<const float*>& bias_dev, const float* scale_dev,
                    const float* shift_dev, const float* x_dev, float* y_dev, cudaStream_t stream);

}  // namespace sqdet
