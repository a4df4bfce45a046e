// libsqdet_b200 engine: graph builder, parameter store, executor and the C ABI.
//
// The reference's "framework" for this path is the TF-1.0 graph that the nets build
// through ModelSkeleton's layer constructors and run through sess.run
// (src/nn_skeleton.py:74-135, 374-586; src/nets/*.py; src/demo.py:193-199).  Here the
// Python facade records the same constructor calls into a plan (sqdet_add_*), and this
// file owns everything behind it: shape inference with TF geometry, activation and
// weight storage in HBM, BN folding to (scale, shift), kernel selection per op
// (wgmma 3xTF32 implicit GEMM or fp32 SIMT), CUDA-graph capture of the whole forward,
// and the fused post-processing.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"
#include "conv_tc.cuh"

namespace sqdet {

// ---------------------------------------------------------------------------------------
static thread_local std::string g_last_error;

void set_error(const std::string& msg) { g_last_error = msg; }

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
int cuda_fail(cudaError_t err, const char* what) {
  g_last_error = std::string("CUDA error: ") + cudaGetErrorString(err) + " in " + what;
  return SQDET_ERR_CUDA;
}

// ---------------------------------------------------------------------------------------
struct Tensor {
  std::string name;
  int B = 0, H = 0, W = 0, C = 0;
  float* dev = nullptr;         // owned (except tensor 0 when the caller feeds its own)
  bool external = false;
  bool materialized = true;     // false: produced and consumed inside a fused kernel only
  int64_t numel() const { return (int64_t)B * H * W * C; }
};

struct Param {
  std::string name;
  std::vector<int64_t> shape;
  std::vector<float> host;
  float* dev = nullptr;
  int64_t numel() const {
    int64_t n = 1;
    for (auto s : shape) n *= s;
    return n;
  }
};

enum OpKind { OP_CONV, OP_POOL, OP_FIRE, OP_ADD_RELU };

struct ConvSpec {
  std::string name;
  int src = -1, dst = -1;
  int Cin = 0, Cout = 0, size = 1, stride = 1, padding = SQDET_PAD_SAME, relu = 1;
  int y_coff = 0;
  int p_kernel = -1, p_bias = -1, p_gamma = -1, p_beta = -1, p_mean = -1, p_var = -1;
  float* scale = nullptr;      // device, BN only
  float* shift = nullptr;
};

enum LaunchKind { L_CONV_SIMT, L_CONV_TC, L_CONV_POOL, L_MAXPOOL, L_ADD_RELU };

// One kernel launch of an op.
struct Launch {
  LaunchKind kind;
  int src = -1, dst = -1;        // tensor read (add+ReLU also reads the op's src2) and written
  int conv = 0, nconv = 0;       // computes the op's convs [conv, conv + nconv)
  int pool_padding = 0;          // L_CONV_POOL: padding of the absorbed 3x3/2 max-pool
  TcConvPlan tc;                 // L_CONV_TC: a conv, an expand pair or a whole fire module
};

struct Op {
  OpKind kind;
  std::string name;
  std::vector<ConvSpec> convs;   // 1 for conv, 3 for fire (squeeze, expand1x1, expand3x3)
  int src = -1, src2 = -1, dst = -1;
  int size = 0, stride = 0, padding = 0;
  int64_t flops = 0, params = 0, min_bytes = 0;
  std::vector<Launch> launches;  // what the op runs, in order; empty for a pool its producer absorbed
};

// One of the two pipeline slots of the host path (sqdet_submit, sqdet_submit_frames_n).
struct Slot {
  float* input = nullptr;        // fp32 network input
  uint8_t* staging = nullptr;    // uint8 images or frames as uploaded; grow-only
  size_t staging_cap = 0;
  float* scales = nullptr;       // B (x_scale, y_scale) pairs of a rescaled frames submission
  cudaEvent_t h2d = nullptr, done = nullptr;   // the upload; the forward and its copies back
  bool used = false;
};

}  // namespace sqdet

using namespace sqdet;

struct sqdet_engine {
  sqdet_config cfg;
  int device = 0;
  int sms = 0;                    // the device's SM count
  bool finalized = false;
  bool params_dirty = true;
  std::vector<Tensor> tensors;
  std::vector<Param> params;
  std::map<std::string, int> param_index;
  std::vector<Op> ops;
  int preds = -1;
  int grid_h = 0, grid_w = 0;
  int64_t num_anchors = 0;
  std::vector<double> anchors_f64;
  float* d_anchors = nullptr;
  float* d_boxes = nullptr;
  float* d_probs = nullptr;
  int64_t* d_cls = nullptr;
  sqdet_det* d_dets = nullptr;
  int32_t* d_counts = nullptr;
  int max_dets = 0;
  // sqdet_forward_tiles' merged records [B, max_dets] and counts [B] (one allocation), and the
  // scratch of its per-tile top-N stage (null when TOP_N_DETECTION is off or above 1024)
  sqdet_det* d_tile_dets = nullptr;
  int32_t* d_tile_counts = nullptr;
  void* d_tile_cand = nullptr;
  // CUDA graphs of one forward, keyed by (input, input type, stream, image count, scales); small
  // LRU-less cache
  struct GraphEntry {
    cudaGraphExec_t exec = nullptr;
    const void* input = nullptr;
    bool u8 = false;              // input is uint8 BGR (sqdet_forward_u8)
    cudaStream_t stream = nullptr;
    int n = 0;
    const float* scales = nullptr;
  };
  GraphEntry graphs[4];
  int graph_next = 0;
  bool use_graph = true;
  // sqdet_forward_u8 hands its uint8 images to the first layer: the plan's only reader of tensor 0
  // is a conv+pool launch.  Otherwise they are converted into tensor 0 first.
  bool u8_fused = false;
  // pipelined host path (sqdet_submit / sqdet_wait), depth 2
  cudaStream_t copy_stream = nullptr;
  Slot slots[2];
  long long n_submitted = 0, n_waited = 0;
  double bgr_means[3] = {103.939, 116.779, 123.68};   // config.py:72
  cudaStream_t own_stream = nullptr;
  // recorded behind every forward: a reload, sqdet_read_tensor and sqdet_set_box_scale wait for it
  // rather than for the device, which is invalid while another thread captures a graph
  cudaEvent_t last_forward = nullptr;
  std::vector<cudaEvent_t> prof_events;
  float* box_scale = nullptr;     // sqdet_set_box_scale's B (x_scale, y_scale) pairs, or null
  // sqdet_forward_frames_{u8,nv12}'s B (x_scale, y_scale) pairs, written by their resize launch; one
  // address for the engine's life, so the forward graphs keyed on it stay valid
  float* frame_scales = nullptr;
  // multi-GPU: the ONE collective of the path, ncclAllGather of the result blob
  void* comm = nullptr;           // ncclComm_t
  bool comm_owned = false;
  int comm_nranks = 0, comm_rank = 0;
  uint8_t* d_gathered = nullptr;  // [nranks][blob_bytes]
  size_t blob_bytes = 0;
  bool gather_in_forward = false;
};

namespace sqdet {

static int add_param(sqdet_engine* e, const std::string& name, std::vector<int64_t> shape) {
  auto it = e->param_index.find(name);
  if (it != e->param_index.end()) return it->second;
  Param p;
  p.name = name;
  p.shape = std::move(shape);
  p.host.assign((size_t)p.numel(), 0.f);
  e->params.push_back(std::move(p));
  const int idx = (int)e->params.size() - 1;
  e->param_index[name] = idx;
  return idx;
}

// True when an op other than `self` reads tensor `t`.
static bool read_by_other_op(const sqdet_engine* e, int t, const Op* self) {
  for (const auto& o : e->ops) {
    if (&o == self) continue;
    if (o.src == t || o.src2 == t) return true;
    for (const auto& c : o.convs)
      if (c.src == t) return true;
  }
  return false;
}

static int new_tensor(sqdet_engine* e, const std::string& name, int B, int H, int W, int C) {
  Tensor t;
  t.name = name;
  t.B = B; t.H = H; t.W = W; t.C = C;
  e->tensors.push_back(t);
  return (int)e->tensors.size() - 1;
}

static int check_build(sqdet_engine* e, int src) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  if (e->finalized) return fail(SQDET_ERR_STATE, "graph is frozen (already finalized)");
  if (src < 0 || src >= (int)e->tensors.size())
    return fail(SQDET_ERR_INVALID_ARG, "unknown source tensor id");
  return SQDET_OK;
}

// Describe one convolution reading tensor `src`; output geometry by TF rules.
static int make_conv(sqdet_engine* e, const std::string& name, int src, int filters, int size,
                     int stride, int padding, int relu, bool bn, bool with_bias,
                     ConvSpec* cs, int* Ho, int* Wo) {
  if (filters <= 0 || size <= 0 || stride <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "conv '" + name + "': non-positive filters/size/stride");
  if (padding != SQDET_PAD_SAME && padding != SQDET_PAD_VALID)
    return fail(SQDET_ERR_INVALID_ARG, "conv '" + name + "': padding must be SAME(0) or VALID(1)");
  const Tensor& in = e->tensors[src];
  const Geom gh = tf_geometry(in.H, size, stride, padding);
  const Geom gw = tf_geometry(in.W, size, stride, padding);
  if (gh.out <= 0 || gw.out <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "conv '" + name + "': kernel larger than input");
  cs->name = name;
  cs->src = src;
  cs->Cin = in.C;
  cs->Cout = filters;
  cs->size = size;
  cs->stride = stride;
  cs->padding = padding;
  cs->relu = relu;
  cs->p_kernel = add_param(e, name + "/kernels", {size, size, in.C, filters});
  if (!bn || with_bias) cs->p_bias = add_param(e, name + "/biases", {filters});
  if (bn) {
    // reference order of model_params: kernels, [biases], gamma, beta, mean, var
    cs->p_gamma = add_param(e, name + "/gamma", {filters});
    cs->p_beta = add_param(e, name + "/beta", {filters});
    cs->p_mean = add_param(e, name + "/mean", {filters});
    cs->p_var = add_param(e, name + "/var", {filters});
  }
  *Ho = gh.out;
  *Wo = gw.out;
  return SQDET_OK;
}

static void conv_cost(const sqdet_engine* e, const ConvSpec& c, int Ho, int Wo, Op* op) {
  const Tensor& in = e->tensors[c.src];
  const int64_t px = (int64_t)in.B * Ho * Wo;
  op->flops += 2LL * c.size * c.size * c.Cin * c.Cout * px;
  op->params += (int64_t)(1 + c.size * c.size * c.Cin) * c.Cout;
}

// sqdet_add_conv / sqdet_add_conv_bn: one conv op and its output tensor.
static int add_conv_op(sqdet_engine* e, const char* what, const char* name, int src, int filters,
                       int size, int stride, int padding, int relu, bool bn, bool with_bias,
                       int* out) {
  int rc = check_build(e, src);
  if (rc) return rc;
  if (!name || !out) return fail(SQDET_ERR_INVALID_ARG, std::string(what) + ": null argument");
  Op op;
  op.kind = OP_CONV;
  op.name = name;
  ConvSpec cs;
  int Ho, Wo;
  rc = make_conv(e, name, src, filters, size, stride, padding, relu, bn, with_bias, &cs, &Ho, &Wo);
  if (rc) return rc;
  cs.dst = new_tensor(e, name, e->tensors[src].B, Ho, Wo, filters);
  conv_cost(e, cs, Ho, Wo, &op);
  op.src = src;
  op.dst = cs.dst;
  op.convs.push_back(cs);
  e->ops.push_back(op);
  *out = cs.dst;
  return SQDET_OK;
}

// Tensor `t` as the forward reads it: the caller's images stand in for tensor 0.
static const float* input_ptr(const sqdet_engine* e, int t, const float* images) {
  return (t == 0 && images) ? images : e->tensors[t].dev;
}

// One launch over images [0, n): every kernel takes the image count as a launch argument, so a
// forward of n < B images runs the kernels planned for B on smaller grids.  `u8`, when non-null,
// is uint8 BGR images the conv+pool launch reads in place of tensor 0 (e->u8_fused).
static int run_launch(sqdet_engine* e, const Op& op, const Launch& l, const float* images,
                      const uint8_t* u8, int n, cudaStream_t stream) {
  const Tensor& in = e->tensors[l.src];
  const float* x = input_ptr(e, l.src, images);
  float* y = e->tensors[l.dst].dev;
  switch (l.kind) {
    case L_CONV_SIMT: {
      const ConvSpec& c = op.convs[l.conv];
      ConvArgs a;
      a.x = x;
      a.w = e->params[c.p_kernel].dev;
      a.bias = c.p_bias >= 0 ? e->params[c.p_bias].dev : nullptr;
      a.scale = c.scale;
      a.shift = c.shift;
      a.y = y;
      a.B = n; a.H = in.H; a.W = in.W; a.Cin = c.Cin; a.Cout = c.Cout;
      a.size = c.size; a.stride = c.stride; a.padding = c.padding; a.relu = c.relu;
      a.y_cstride = e->tensors[l.dst].C;
      a.y_coff = c.y_coff;
      return launch_conv_simt(a, stream);
    }
    case L_CONV_TC:
      return launch_conv_tc(l.tc, x, y, n, stream);
    case L_CONV_POOL: {
      const ConvSpec& c = op.convs[0];
      const uint8_t* x8 = l.src == 0 ? u8 : nullptr;
      return launch_conv_pool_simt(x8 ? nullptr : x, x8, e->bgr_means, e->params[c.p_kernel].dev,
                                   c.p_bias >= 0 ? e->params[c.p_bias].dev : nullptr, c.scale,
                                   c.shift, y, n, in.H, in.W, c.Cout, c.size, c.padding, c.relu,
                                   l.pool_padding, stream);
    }
    case L_MAXPOOL:
      return launch_maxpool(x, y, n, in.H, in.W, in.C, op.size, op.stride, op.padding, stream);
    case L_ADD_RELU:
      return launch_add_relu(x, input_ptr(e, op.src2, images), y, (int64_t)n * in.H * in.W * in.C,
                             stream);
  }
  return fail(SQDET_ERR_STATE, "unknown launch kind");
}

static int run_op(sqdet_engine* e, const Op& op, const float* images, const uint8_t* u8, int n,
                  cudaStream_t stream) {
  for (const Launch& l : op.launches) {
    int rc = run_launch(e, op, l, images, u8, n, stream);
    if (rc) return rc;
  }
  return SQDET_OK;
}

static void release_launches(Op& op) {
  for (auto& l : op.launches) tc_conv_release(&l.tc);
  op.launches.clear();
}

// ---- NCCL, bound at run time (dlopen): the library must load on boxes without NCCL ----------
// Prototypes restated from nccl.h (stable since NCCL 2.0); ncclUniqueId is passed BY VALUE.
struct NcclId { char internal[128]; };
struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(NcclId*) = nullptr;
  int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static int nccl_load() {
  if (g_nccl.handle) return SQDET_OK;
  const char* env = getenv("SQDET_NCCL_LIB");
  const char* cands[] = {env, "libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* c : cands) {
    if (!c || !*c) continue;
    h = dlopen(c, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) return fail(SQDET_ERR_UNSUPPORTED, "NCCL not found (set SQDET_NCCL_LIB to libnccl.so.2)");
  NcclApi a;
  a.handle = h;
  a.GetUniqueId = (int (*)(NcclId*))dlsym(h, "ncclGetUniqueId");
  a.CommInitRank = (int (*)(void**, int, NcclId, int))dlsym(h, "ncclCommInitRank");
  a.CommDestroy = (int (*)(void*))dlsym(h, "ncclCommDestroy");
  a.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(h, "ncclAllGather");
  a.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
  if (!a.GetUniqueId || !a.CommInitRank || !a.CommDestroy || !a.AllGather)
    return fail(SQDET_ERR_UNSUPPORTED, "NCCL library lacks the expected entry points");
  g_nccl = a;
  return SQDET_OK;
}
static int nccl_fail(int r, const char* what) {
  std::string m = std::string("NCCL error in ") + what + ": ";
  m += g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "unknown";
  return fail(SQDET_ERR_CUDA, m);
}

static int run_allgather(sqdet_engine* e, void* comm, cudaStream_t stream) {
  if (!comm) return fail(SQDET_ERR_STATE, "sqdet_allgather: no communicator attached");
  if (!e->d_gathered) return fail(SQDET_ERR_STATE, "sqdet_allgather: gather buffer missing");
  // records and counts are ONE contiguous blob (sqdet_finalize): one collective per step
  const int r = g_nccl.AllGather(e->d_dets, e->d_gathered, e->blob_bytes, /*ncclUint8*/ 1, comm,
                                 stream);
  if (r != 0) return nccl_fail(r, "ncclAllGather");
  return SQDET_OK;
}

// interpret_output of images [0, n), then the eval-order rescale by `scales` unless it is null
static int run_interpret(sqdet_engine* e, int n, const float* scales, cudaStream_t stream) {
  const sqdet_config& c = e->cfg;
  int rc = launch_interpret(e->tensors[e->preds].dev, e->d_anchors, e->d_boxes, e->d_probs,
                            e->d_cls, n, e->grid_h, e->grid_w, c.anchors_per_grid,
                            c.classes, c.image_width, c.image_height, c.exp_thresh, stream);
  if (rc || !scales) return rc;
  return launch_rescale_boxes(e->d_boxes, scales, n, (int)e->num_anchors, stream);
}

// filter_prediction of images [0, n); the counts of images [n, B) are set to 0, so the result blob
// (records + counts) stays fully defined for the all-gather
static int run_filter(sqdet_engine* e, int n, cudaStream_t stream) {
  const sqdet_config& c = e->cfg;
  int rc = launch_topk_nms(e->d_boxes, e->d_probs, e->d_cls, n, (int)e->num_anchors,
                           c.classes, c.top_n_detection, c.prob_thresh, c.nms_thresh, e->d_dets,
                           e->d_counts, e->max_dets, stream);
  if (rc || n == c.batch_size) return rc;
  SQ_CUDA(cudaMemsetAsync(e->d_counts + n, 0, sizeof(int32_t) * (size_t)(c.batch_size - n), stream));
  return SQDET_OK;
}

static int run_postproc(sqdet_engine* e, int n, const float* scales, cudaStream_t stream) {
  int rc = run_interpret(e, n, scales, stream);
  if (!rc) rc = run_filter(e, n, stream);
  if (rc) return rc;
  if (e->gather_in_forward && e->comm) return run_allgather(e, e->comm, stream);
  return SQDET_OK;
}

// Upload parameters and derive what the kernels consume (BN scale/shift, TC packs).  The uploads
// are synchronous copies on the legacy stream, which is not ordered with the engine's own stream
// or a caller's non-blocking one.  So the forwards already enqueued are waited for first, or they
// would read the new weights part-way through, and the legacy stream after the uploads, because a
// copy from pageable memory can return before its DMA lands and this forward must not read ahead.
static int prepare_params(sqdet_engine* e) {
  if (!e->params_dirty) return SQDET_OK;
  SQ_CUDA(cudaEventSynchronize(e->last_forward));
  for (auto& p : e->params) {
    if (!p.dev) SQ_CUDA(cudaMalloc(&p.dev, sizeof(float) * (size_t)p.numel()));
    SQ_CUDA(cudaMemcpy(p.dev, p.host.data(), sizeof(float) * (size_t)p.numel(),
                       cudaMemcpyHostToDevice));
  }
  auto host = [e](int p) { return p >= 0 ? e->params[p].host.data() : nullptr; };
  for (auto& op : e->ops) {
    std::vector<std::vector<float>> scale(op.convs.size()), shift(op.convs.size());
    for (size_t k = 0; k < op.convs.size(); ++k) {
      ConvSpec& c = op.convs[k];
      if (c.p_gamma < 0) continue;
      // tf.nn.batch_normalization: inv = rsqrt(var+eps)*gamma; y = x*inv + (beta - mean*inv)
      const int n = c.Cout;
      std::vector<float>& sc = scale[k];
      std::vector<float>& sh = shift[k];
      sc.resize(n);
      sh.resize(n);
      const auto& g = e->params[c.p_gamma].host;
      const auto& b = e->params[c.p_beta].host;
      const auto& m = e->params[c.p_mean].host;
      const auto& v = e->params[c.p_var].host;
      for (int i = 0; i < n; ++i) {
        const float inv = (1.0f / sqrtf(v[i] + e->cfg.batch_norm_epsilon)) * g[i];
        sc[i] = inv;
        sh[i] = b[i] - m[i] * inv;
      }
      if (!c.scale) SQ_CUDA(cudaMalloc(&c.scale, sizeof(float) * n));
      if (!c.shift) SQ_CUDA(cudaMalloc(&c.shift, sizeof(float) * n));
      SQ_CUDA(cudaMemcpy(c.scale, sc.data(), sizeof(float) * n, cudaMemcpyHostToDevice));
      SQ_CUDA(cudaMemcpy(c.shift, sh.data(), sizeof(float) * n, cudaMemcpyHostToDevice));
    }
    // tensor-core weight packs
    for (auto& l : op.launches) {
      if (l.kind != L_CONV_TC) continue;
      std::vector<const float*> w, b;
      for (int k = l.conv; k < l.conv + l.nconv; ++k) {
        w.push_back(host(op.convs[k].p_kernel));
        b.push_back(host(op.convs[k].p_bias));
      }
      int rc = tc_conv_pack_weights(&l.tc, w, b);
      if (!rc && !scale[l.conv].empty())
        rc = tc_conv_set_affine(&l.tc, scale[l.conv].data(), shift[l.conv].data());
      if (rc) return rc;
    }
  }
  SQ_CUDA(cudaStreamSynchronize(nullptr));
  e->params_dirty = false;
  // weights changed -> any captured graph still points at the same buffers, so it stays valid
  return SQDET_OK;
}

// Destroys the cached graphs, or only those of uint8 inputs.  A graph still running finishes first.
static void drop_graph(sqdet_engine* e, bool only_u8 = false) {
  for (auto& g : e->graphs) {
    if (only_u8 && !g.u8) continue;
    if (g.exec) cudaGraphExecDestroy(g.exec);
    g = sqdet_engine::GraphEntry();
  }
}

// The forward of fp32 images, or of uint8 BGR images (`u8`): handed to the first layer when the
// plan fuses it, else converted into tensor 0 by one launch: the byte-wise same-size path of the
// resize kernel on one frame of n*H rows, which reads images starting at any byte.
static int enqueue_all(sqdet_engine* e, const void* images, bool u8, int n, const float* scales,
                       cudaStream_t stream) {
  const float* x = u8 ? nullptr : static_cast<const float*>(images);
  const uint8_t* x8 = u8 ? static_cast<const uint8_t*>(images) : nullptr;
  if (x8 && !e->u8_fused) {
    const Tensor& t = e->tensors[0];
    const FrameSource f = {{x8}, {3 * (int64_t)t.W}, 0, 0, n * t.H, t.W};
    const int rc = launch_resize_meansub_frames(SQDET_FMT_BGR, &f, 1, t.dev, n * t.H, t.W,
                                                e->bgr_means, 0, nullptr, stream);
    if (rc) return rc;
    x8 = nullptr;
  }
  for (const auto& op : e->ops) {
    int rc = run_op(e, op, x, x8, n, stream);
    if (rc) return rc;
  }
  return run_postproc(e, n, scales, stream);
}

// The forward over images [0, n) of `images` (uint8 BGR when `u8`, else fp32), 1 <= n <= B,
// rescaled by `scales` unless null.
static int forward_impl(sqdet_engine* e, const void* images, bool u8, int n, const float* scales,
                        cudaStream_t stream) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  if (!e->finalized)
    return fail(SQDET_ERR_STATE, u8 ? "sqdet_forward_u8 before sqdet_finalize"
                                    : "sqdet_forward before sqdet_finalize");
  if (!images) return fail(SQDET_ERR_INVALID_ARG, "null images pointer");
  if (n < 1 || n > e->cfg.batch_size)
    return fail(SQDET_ERR_INVALID_ARG, u8 ? "sqdet_forward_u8: n must be in [1, batch_size]"
                                          : "sqdet_forward_n: n must be in [1, batch_size]");
  DeviceGuard guard(e->device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select the engine's device");
  int rc = prepare_params(e);
  if (rc) return rc;
  const bool can_graph = e->use_graph && stream != nullptr;   // legacy stream cannot capture
  if (!can_graph) {
    rc = enqueue_all(e, images, u8, n, scales, stream);
    if (!rc) SQ_CUDA(cudaEventRecord(e->last_forward, stream));
    return rc;
  }
  sqdet_engine::GraphEntry* hit = nullptr;
  for (auto& g : e->graphs)
    if (g.exec && g.input == images && g.u8 == u8 && g.stream == stream && g.n == n &&
        g.scales == scales)
      hit = &g;
  if (!hit) {
    sqdet_engine::GraphEntry& slot = e->graphs[e->graph_next];
    e->graph_next = (e->graph_next + 1) % 4;
    if (slot.exec) cudaGraphExecDestroy(slot.exec);
    slot = sqdet_engine::GraphEntry();
    cudaGraph_t graph = nullptr;
    SQ_CUDA(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
    rc = enqueue_all(e, images, u8, n, scales, stream);
    cudaError_t ce = cudaStreamEndCapture(stream, &graph);
    if (rc) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    if (ce != cudaSuccess) return cuda_fail(ce, "cudaStreamEndCapture");
    ce = cudaGraphInstantiate(&slot.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) return cuda_fail(ce, "cudaGraphInstantiate");
    slot.input = images;
    slot.u8 = u8;
    slot.stream = stream;
    slot.n = n;
    slot.scales = scales;
    hit = &slot;
  }
  SQ_CUDA(cudaGraphLaunch(hit->exec, stream));
  SQ_CUDA(cudaEventRecord(e->last_forward, stream));
  return SQDET_OK;
}

// Pipelined host path (sqdet_submit, sqdet_submit_frames): refuses a third batch in flight, sets
// the pipeline up on first use and picks the slot of this submission.
static int begin_submit(sqdet_engine* e, const char* what, Slot** slot) {
  if (e->n_submitted - e->n_waited >= 2)
    return fail(SQDET_ERR_STATE, std::string(what) + ": two batches already in flight; call sqdet_wait");
  if (!e->copy_stream) {
    SQ_CUDA(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
    for (Slot& s : e->slots) {
      SQ_CUDA(cudaMalloc(&s.input, sizeof(float) * (size_t)e->tensors[0].numel()));
      SQ_CUDA(cudaEventCreateWithFlags(&s.h2d, cudaEventDisableTiming));
      SQ_CUDA(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    }
  }
  *slot = &e->slots[e->n_submitted & 1];
  return SQDET_OK;
}

// One submission's host-to-device copies on the copy stream, behind the slot's previous forward:
// host buffer i (bytes[i] long) goes to offset off[i] of the slot's fp32 input when `to_input`, else
// of its uint8 staging buffer, grown when too small.  The compute stream then waits for them.
static int upload(sqdet_engine* e, Slot& s, bool to_input, int count, const uint8_t* const* src,
                  const size_t* bytes, const size_t* off) {
  cudaStream_t cs = e->copy_stream;
  // the slot's buffers are free once the forward that last read them has finished
  if (s.used) SQ_CUDA(cudaStreamWaitEvent(cs, s.done, 0));
  const size_t total = off[count - 1] + bytes[count - 1];
  if (!to_input && s.staging_cap < total) {
    // growing the staging buffer: the slot's previous forward must be done with it
    if (s.used) SQ_CUDA(cudaEventSynchronize(s.done));
    cudaFree(s.staging);
    s.staging = nullptr;
    SQ_CUDA(cudaMalloc(&s.staging, total));
    s.staging_cap = total;
  }
  uint8_t* dst = to_input ? reinterpret_cast<uint8_t*>(s.input) : s.staging;
  for (int i = 0; i < count; ++i)
    SQ_CUDA(cudaMemcpyAsync(dst + off[i], src[i], bytes[i], cudaMemcpyHostToDevice, cs));
  SQ_CUDA(cudaEventRecord(s.h2d, cs));
  SQ_CUDA(cudaStreamWaitEvent(e->own_stream, s.h2d, 0));
  return SQDET_OK;
}

// The forward over images [0, n) of `input`, one of the slot's buffers (uint8 BGR when `u8`, else
// fp32), on the compute stream, then their records and counts back to the caller's buffers;
// `done` marks the slot's buffers free again.
static int finish_submit(sqdet_engine* e, Slot& s, const void* input, bool u8, int n,
                         const float* scales, sqdet_det* dets, int32_t* counts) {
  cudaStream_t ks = e->own_stream;
  int rc = forward_impl(e, input, u8, n, scales, ks);
  if (rc) return rc;
  if (dets)
    SQ_CUDA(cudaMemcpyAsync(dets, e->d_dets, sizeof(sqdet_det) * (size_t)n * e->max_dets,
                            cudaMemcpyDeviceToHost, ks));
  if (counts)
    SQ_CUDA(cudaMemcpyAsync(counts, e->d_counts, sizeof(int32_t) * (size_t)n,
                            cudaMemcpyDeviceToHost, ks));
  SQ_CUDA(cudaEventRecord(s.done, ks));
  s.used = true;
  ++e->n_submitted;
  return SQDET_OK;
}

}  // namespace sqdet

// =========================================================================================
//                                        C ABI
// =========================================================================================
extern "C" {

const char* sqdet_last_error(void) { return g_last_error.c_str(); }
const char* sqdet_version(void) { return "sqdet_b200 0.1 (sm_90a)"; }

int sqdet_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int sqdet_create(const sqdet_config* cfg, int device, sqdet_engine** out) {
  if (!cfg || !out) return fail(SQDET_ERR_INVALID_ARG, "sqdet_create: null argument");
  if (cfg->batch_size <= 0 || cfg->image_height <= 0 || cfg->image_width <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_create: batch/image size must be positive");
  if (cfg->classes <= 0 || cfg->anchors_per_grid <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_create: classes/anchors_per_grid must be positive");
  if (cfg->math_mode != SQDET_MATH_FP32_SIMT && cfg->math_mode != SQDET_MATH_TF32X3_TC)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_create: unknown math_mode");
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess) return cuda_fail(ce, "cudaGetDeviceCount (no CUDA device: this "
                                              "library has no CPU fallback)");
  if (device < 0 || device >= ndev)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_create: device index out of range");
  cudaDeviceProp prop;
  SQ_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(SQDET_ERR_UNSUPPORTED, "sqdet_create: this build targets sm_90a (H100) only");
  std::unique_ptr<sqdet_engine> e(new sqdet_engine());
  e->cfg = *cfg;
  e->device = device;
  e->sms = prop.multiProcessorCount;
  new_tensor(e.get(), "image_input", cfg->batch_size, cfg->image_height, cfg->image_width, 3);
  *out = e.release();
  return SQDET_OK;
}

int sqdet_destroy(sqdet_engine* e) {
  if (!e) return SQDET_OK;
  DeviceGuard guard(e->device);
  drop_graph(e);
  for (auto& t : e->tensors)
    if (t.dev && !t.external) cudaFree(t.dev);
  for (auto& p : e->params)
    if (p.dev) cudaFree(p.dev);
  for (auto& op : e->ops) {
    for (auto& c : op.convs) {
      if (c.scale) cudaFree(c.scale);
      if (c.shift) cudaFree(c.shift);
    }
    release_launches(op);
  }
  cudaFree(e->d_anchors);
  cudaFree(e->d_boxes);
  cudaFree(e->d_probs);
  cudaFree(e->d_cls);
  cudaFree(e->d_dets);   // also owns d_counts (one blob)
  cudaFree(e->d_tile_dets);   // also owns d_tile_counts
  cudaFree(e->d_tile_cand);
  for (auto ev : e->prof_events) cudaEventDestroy(ev);
  for (Slot& s : e->slots) {
    cudaFree(s.input);
    cudaFree(s.staging);
    cudaFree(s.scales);
    if (s.h2d) cudaEventDestroy(s.h2d);
    if (s.done) cudaEventDestroy(s.done);
  }
  if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
  if (e->own_stream) cudaStreamDestroy(e->own_stream);
  if (e->last_forward) cudaEventDestroy(e->last_forward);
  cudaFree(e->box_scale);
  cudaFree(e->frame_scales);
  cudaFree(e->d_gathered);
  if (e->comm && e->comm_owned && g_nccl.CommDestroy) g_nccl.CommDestroy(e->comm);
  (void)cudaGetLastError();   // never leave a stale error for the next engine's launch checks
  delete e;
  return SQDET_OK;
}

int sqdet_add_conv(sqdet_engine* e, const char* layer_name, int src, int filters, int size,
                   int stride, int padding, int relu, int* out) {
  return add_conv_op(e, "sqdet_add_conv", layer_name, src, filters, size, stride, padding, relu,
                     false, true, out);
}

int sqdet_add_conv_bn(sqdet_engine* e, const char* scope_name, int src, int filters, int size,
                      int stride, int relu, int conv_with_bias, int* out) {
  return add_conv_op(e, "sqdet_add_conv_bn", scope_name, src, filters, size, stride,
                     SQDET_PAD_SAME, relu, true, conv_with_bias != 0, out);
}

int sqdet_add_pool(sqdet_engine* e, const char* layer_name, int src, int size, int stride,
                   int padding, int* out) {
  int rc = check_build(e, src);
  if (rc) return rc;
  if (!layer_name || !out) return fail(SQDET_ERR_INVALID_ARG, "sqdet_add_pool: null argument");
  if (size <= 0 || stride <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_add_pool: non-positive size/stride");
  if (padding != SQDET_PAD_SAME && padding != SQDET_PAD_VALID)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_add_pool: padding must be SAME(0) or VALID(1)");
  const Tensor in = e->tensors[src];
  const Geom gh = tf_geometry(in.H, size, stride, padding);
  const Geom gw = tf_geometry(in.W, size, stride, padding);
  if (gh.out <= 0 || gw.out <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_add_pool: window larger than input");
  Op op;
  op.kind = OP_POOL;
  op.name = layer_name;
  op.src = src;
  op.size = size;
  op.stride = stride;
  op.padding = padding;
  op.dst = new_tensor(e, layer_name, in.B, gh.out, gw.out, in.C);
  e->ops.push_back(op);
  *out = op.dst;
  return SQDET_OK;
}

int sqdet_add_fire(sqdet_engine* e, const char* layer_name, int src, int s1x1, int e1x1,
                   int e3x3, int* out) {
  int rc = check_build(e, src);
  if (rc) return rc;
  if (!layer_name || !out) return fail(SQDET_ERR_INVALID_ARG, "sqdet_add_fire: null argument");
  const std::string base(layer_name);
  Op op;
  op.kind = OP_FIRE;
  op.name = base;
  ConvSpec sq, x1, x3;
  int Ho, Wo;
  rc = make_conv(e, base + "/squeeze1x1", src, s1x1, 1, 1, SQDET_PAD_SAME, 1, false, true, &sq,
                 &Ho, &Wo);
  if (rc) return rc;
  sq.dst = new_tensor(e, base + "/squeeze1x1", e->tensors[src].B, Ho, Wo, s1x1);
  conv_cost(e, sq, Ho, Wo, &op);
  rc = make_conv(e, base + "/expand1x1", sq.dst, e1x1, 1, 1, SQDET_PAD_SAME, 1, false, true,
                 &x1, &Ho, &Wo);
  if (rc) return rc;
  rc = make_conv(e, base + "/expand3x3", sq.dst, e3x3, 3, 1, SQDET_PAD_SAME, 1, false, true,
                 &x3, &Ho, &Wo);
  if (rc) return rc;
  const int dst = new_tensor(e, base, e->tensors[src].B, Ho, Wo, e1x1 + e3x3);
  x1.dst = dst; x1.y_coff = 0;
  x3.dst = dst; x3.y_coff = e1x1;      // tf.concat([ex1x1, ex3x3], 3)  squeezeDet.py:106
  conv_cost(e, x1, Ho, Wo, &op);
  conv_cost(e, x3, Ho, Wo, &op);
  op.src = src;
  op.dst = dst;
  op.convs = {sq, x1, x3};
  e->ops.push_back(op);
  *out = dst;
  return SQDET_OK;
}

int sqdet_add_add_relu(sqdet_engine* e, const char* name, int a, int b, int* out) {
  int rc = check_build(e, a);
  if (rc) return rc;
  rc = check_build(e, b);
  if (rc) return rc;
  if (!name || !out) return fail(SQDET_ERR_INVALID_ARG, "sqdet_add_add_relu: null argument");
  const Tensor ta = e->tensors[a], tb = e->tensors[b];
  if (ta.B != tb.B || ta.H != tb.H || ta.W != tb.W || ta.C != tb.C)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_add_add_relu: operand shapes differ");
  Op op;
  op.kind = OP_ADD_RELU;
  op.name = name;
  op.src = a;
  op.src2 = b;
  op.dst = new_tensor(e, name, ta.B, ta.H, ta.W, ta.C);
  e->ops.push_back(op);
  *out = op.dst;
  return SQDET_OK;
}

int sqdet_set_preds(sqdet_engine* e, int preds, const double* anchor_box, int64_t num_anchors) {
  int rc = check_build(e, preds);
  if (rc) return rc;
  if (!anchor_box) return fail(SQDET_ERR_INVALID_ARG, "sqdet_set_preds: null anchors");
  const Tensor& t = e->tensors[preds];
  const int K = e->cfg.anchors_per_grid, C = e->cfg.classes;
  if (t.C != K * (C + 1 + 4))
    return fail(SQDET_ERR_INVALID_ARG,
                "sqdet_set_preds: preds must have ANCHOR_PER_GRID*(CLASSES+1+4) channels");
  if (num_anchors != (int64_t)t.H * t.W * K)
    return fail(SQDET_ERR_INVALID_ARG,
                "sqdet_set_preds: len(ANCHOR_BOX) != grid_h*grid_w*ANCHOR_PER_GRID");
  e->preds = preds;
  e->grid_h = t.H;
  e->grid_w = t.W;
  e->num_anchors = num_anchors;
  e->anchors_f64.assign(anchor_box, anchor_box + num_anchors * 4);
  return SQDET_OK;
}

static int plan_ops(sqdet_engine* e);

int sqdet_finalize(sqdet_engine* e) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  if (e->finalized) return fail(SQDET_ERR_STATE, "already finalized");
  if (e->preds < 0) return fail(SQDET_ERR_STATE, "sqdet_finalize before sqdet_set_preds");
  DeviceGuard guard(e->device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select the engine's device");
  const sqdet_config& c = e->cfg;
  // result capacity
  const bool topn = c.top_n_detection > 0 && c.top_n_detection < e->num_anchors;
  e->max_dets = c.max_dets > 0 ? c.max_dets : (topn ? c.top_n_detection : 1024);
  if (topn && e->max_dets < c.top_n_detection)
    return fail(SQDET_ERR_INVALID_ARG, "max_dets smaller than TOP_N_DETECTION");
  if (topn && c.top_n_detection > 1024)
    return fail(SQDET_ERR_UNSUPPORTED, "TOP_N_DETECTION above 1024 is not supported");
  int rc = plan_ops(e);
  if (rc) return rc;
  // activations
  for (size_t i = 0; i < e->tensors.size(); ++i) {
    Tensor& t = e->tensors[i];
    if (!t.materialized) continue;
    SQ_CUDA(cudaMalloc(&t.dev, sizeof(float) * (size_t)t.numel()));
  }
  const int64_t A = e->num_anchors, B = c.batch_size;
  std::vector<float> anc((size_t)A * 4);
  for (size_t i = 0; i < anc.size(); ++i) anc[i] = (float)e->anchors_f64[i];   // fp64 -> fp32 cast
  SQ_CUDA(cudaMalloc(&e->d_anchors, sizeof(float) * anc.size()));
  SQ_CUDA(cudaMemcpy(e->d_anchors, anc.data(), sizeof(float) * anc.size(), cudaMemcpyHostToDevice));
  SQ_CUDA(cudaMalloc(&e->d_boxes, sizeof(float) * (size_t)(B * A * 4)));
  SQ_CUDA(cudaMalloc(&e->d_probs, sizeof(float) * (size_t)(B * A)));
  SQ_CUDA(cudaMalloc(&e->d_cls, sizeof(int64_t) * (size_t)(B * A)));
  // records and counts share ONE allocation: [B*max_dets records][B int32 counts] is the
  // blob a rank contributes to the N-GPU all-gather (squeezedet_b200/shard.py).
  {
    const size_t rec_bytes = sizeof(sqdet_det) * (size_t)(B * e->max_dets);
    void* blob = nullptr;
    SQ_CUDA(cudaMalloc(&blob, rec_bytes + sizeof(int32_t) * (size_t)B));
    e->d_dets = reinterpret_cast<sqdet_det*>(blob);
    e->d_counts = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(blob) + rec_bytes);
    // the same layout for sqdet_forward_tiles' merged records, all counts 0 until its first call
    SQ_CUDA(cudaMalloc(&blob, rec_bytes + sizeof(int32_t) * (size_t)B));
    SQ_CUDA(cudaMemset(blob, 0, rec_bytes + sizeof(int32_t) * (size_t)B));
    e->d_tile_dets = reinterpret_cast<sqdet_det*>(blob);
    e->d_tile_counts = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(blob) + rec_bytes);
  }
  if (c.top_n_detection > 0 && c.top_n_detection <= 1024)
    SQ_CUDA(cudaMalloc(&e->d_tile_cand,
                       merge_tiles_scratch_bytes((int)B, (int)A, c.top_n_detection)));
  SQ_CUDA(cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking));
  SQ_CUDA(cudaEventCreateWithFlags(&e->last_forward, cudaEventDisableTiming));
  e->finalized = true;
  e->params_dirty = true;
  return SQDET_OK;
}

// One conv as one launch: the wgmma implicit GEMM where the tensor-core path takes the shape,
// else the FFMA kernel.
static int plan_conv(sqdet_engine* e, const ConvSpec& c, int index, bool tc, Launch* l) {
  *l = Launch{L_CONV_SIMT, c.src, c.dst, index, 1};
  if (!tc) return SQDET_OK;
  const Tensor& in = e->tensors[c.src];
  const int rc = tc_conv_plan(&l->tc, in.B, in.H, in.W, c.Cin, {{c.size, c.Cout, c.y_coff}},
                              c.stride, c.padding, c.relu, c.p_gamma >= 0, e->tensors[c.dst].C);
  if (rc > 0) l->kind = L_CONV_TC;
  return rc < 0 ? rc : SQDET_OK;
}

// A fire module on tensor cores runs as one kernel where the squeeze is 16 channels wide and the
// grid holds at least 4 tiles per SM (SqueezeDet fire2/3); otherwise as the squeeze conv, then
// the expand pair as one launch over the squeeze tensor.  What the wgmma kernels decline, and
// every fire in the SIMT math mode, runs as three FFMA convs.
static int plan_fire(sqdet_engine* e, Op& op, bool tc) {
  const ConvSpec& sq = op.convs[0];
  const ConvSpec& e1 = op.convs[1];
  const ConvSpec& e3 = op.convs[2];
  const Tensor& x = e->tensors[op.src];
  const long long tiles = (long long)x.B * ((x.H + 7) / 8) * ((x.W + 15) / 16);
  if (tc && sq.Cout <= 16 && tiles >= 4LL * e->sms && sq.dst != e->preds &&
      !read_by_other_op(e, sq.dst, &op)) {
    Launch l{L_CONV_TC, op.src, op.dst, 0, 3};
    const int rc = tc_fire_plan(&l.tc, x.B, x.H, x.W, x.C, sq.Cout, e1.Cout, e3.Cout);
    if (rc < 0) return rc;
    if (rc) {
      op.launches.push_back(l);
      e->tensors[sq.dst].materialized = false;
      return SQDET_OK;
    }
  }
  Launch l;
  int rc = plan_conv(e, sq, 0, tc, &l);
  op.launches.push_back(l);
  if (rc) return rc;
  if (tc) {
    const Tensor& q = e->tensors[sq.dst];
    Launch pair{L_CONV_TC, sq.dst, op.dst, 1, 2};
    rc = tc_conv_plan(&pair.tc, q.B, q.H, q.W, q.C,
                      {{e1.size, e1.Cout, e1.y_coff}, {e3.size, e3.Cout, e3.y_coff}}, 1,
                      SQDET_PAD_SAME, 1, false, e->tensors[op.dst].C);
    if (rc < 0) return rc;
    if (rc) {
      op.launches.push_back(pair);
      return SQDET_OK;
    }
  }
  op.launches.push_back(Launch{L_CONV_SIMT, sq.dst, op.dst, 1, 1});
  op.launches.push_back(Launch{L_CONV_SIMT, sq.dst, op.dst, 2, 1});
  return SQDET_OK;
}

// The bytes an op has to move at the least: its input, the tensor it finally writes (a fused
// pool's output) and its parameters; add+ReLU reads two tensors and writes one.
static int64_t min_bytes(const sqdet_engine* e, const Op& op) {
  auto bytes = [e](int t) { return 4 * e->tensors[t].numel(); };
  if (op.kind == OP_ADD_RELU) return 3 * bytes(op.dst);
  if (op.launches.empty()) return 0;
  return bytes(op.src) + bytes(op.launches.back().dst) + 4 * op.params;
}

// Every kernel choice of the forward: first-layer pool fusion, tensor-core plans, one-kernel fire
// or expand pair, and which tensors are never materialised.  Runs before the activations are
// allocated.
static int plan_ops(sqdet_engine* e) {
  const bool tc = e->cfg.math_mode == SQDET_MATH_TF32X3_TC;
  for (auto& op : e->ops) release_launches(op);
  for (size_t i = 0; i < e->ops.size(); ++i) {
    Op& op = e->ops[i];
    int rc = SQDET_OK;
    switch (op.kind) {
      case OP_CONV: {
        const ConvSpec& c = op.convs[0];
        Op* pool = i + 1 < e->ops.size() ? &e->ops[i + 1] : nullptr;
        Launch l;
        if (pool && pool->kind == OP_POOL && pool->src == op.dst && op.dst != e->preds &&
            conv_pool_simt_eligible(c.Cin, c.Cout, c.size, c.stride, pool->size, pool->stride) &&
            !read_by_other_op(e, op.dst, pool)) {
          // the first layer (Cin = 3, stride 2) and the 3x3/2 pool that alone reads it: one FFMA
          // kernel in both math modes.  The pool keeps no launch and the un-pooled tensor is never
          // materialised.
          l = Launch{L_CONV_POOL, op.src, pool->dst, 0, 1};
          l.pool_padding = pool->padding;
          e->tensors[op.dst].materialized = false;
          ++i;
        } else {
          rc = plan_conv(e, c, 0, tc, &l);
        }
        op.launches.push_back(l);
        break;
      }
      case OP_FIRE:
        rc = plan_fire(e, op, tc);
        break;
      case OP_POOL:
        op.launches.push_back(Launch{L_MAXPOOL, op.src, op.dst});
        break;
      case OP_ADD_RELU:
        op.launches.push_back(Launch{L_ADD_RELU, op.src, op.dst});
        break;
    }
    if (rc) return rc;
  }
  for (auto& op : e->ops) op.min_bytes = min_bytes(e, op);
  int readers = 0;
  bool pool_reads = false;
  for (const auto& op : e->ops)
    for (const auto& l : op.launches)
      if (l.src == 0 || (l.kind == L_ADD_RELU && op.src2 == 0)) {
        ++readers;
        pool_reads = pool_reads || l.kind == L_CONV_POOL;
      }
  e->u8_fused = readers == 1 && pool_reads;
  return SQDET_OK;
}

int sqdet_num_params(sqdet_engine* e) { return e ? (int)e->params.size() : SQDET_ERR_INVALID_ARG; }

int sqdet_param_info(sqdet_engine* e, int index, char* name_buf, int name_cap, int64_t shape[4],
                     int* ndim) {
  if (!e || index < 0 || index >= (int)e->params.size())
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_param_info: bad index");
  const Param& p = e->params[index];
  if (name_buf && name_cap > 0) {
    strncpy(name_buf, p.name.c_str(), (size_t)name_cap - 1);
    name_buf[name_cap - 1] = 0;
  }
  if (shape)
    for (int i = 0; i < 4; ++i) shape[i] = i < (int)p.shape.size() ? p.shape[i] : 1;
  if (ndim) *ndim = (int)p.shape.size();
  return SQDET_OK;
}

int sqdet_set_param(sqdet_engine* e, const char* name, const float* data, const int64_t* shape,
                    int ndim) {
  if (!e || !name || !data || !shape)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_set_param: null argument");
  auto it = e->param_index.find(name);
  if (it == e->param_index.end())
    return fail(SQDET_ERR_NOT_FOUND, std::string("sqdet_set_param: no parameter named '") + name + "'");
  Param& p = e->params[it->second];
  bool same = ndim == (int)p.shape.size();
  for (int i = 0; same && i < ndim; ++i) same = shape[i] == p.shape[i];
  if (!same)
    return fail(SQDET_ERR_INVALID_ARG,
                std::string("sqdet_set_param: shape mismatch for '") + name + "'");
  memcpy(p.host.data(), data, sizeof(float) * (size_t)p.numel());
  e->params_dirty = true;
  return SQDET_OK;
}

int sqdet_num_tensors(sqdet_engine* e) { return e ? (int)e->tensors.size() : SQDET_ERR_INVALID_ARG; }

int sqdet_tensor_info(sqdet_engine* e, int id, char* name_buf, int name_cap, int64_t shape[4]) {
  if (!e || id < 0 || id >= (int)e->tensors.size())
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_tensor_info: bad id");
  const Tensor& t = e->tensors[id];
  if (name_buf && name_cap > 0) {
    strncpy(name_buf, t.name.c_str(), (size_t)name_cap - 1);
    name_buf[name_cap - 1] = 0;
  }
  if (shape) { shape[0] = t.B; shape[1] = t.H; shape[2] = t.W; shape[3] = t.C; }
  return SQDET_OK;
}

int sqdet_read_tensor(sqdet_engine* e, int id, float* host_out) {
  if (!e || id < 0 || id >= (int)e->tensors.size() || !host_out)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_read_tensor: bad argument");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_read_tensor before sqdet_finalize");
  DeviceGuard guard(e->device);
  SQ_CUDA(cudaEventSynchronize(e->last_forward));
  const Tensor& t = e->tensors[id];
  if (!t.materialized)
    return fail(SQDET_ERR_NOT_FOUND, "tensor '" + t.name + "' is not materialised (fused into its consumer)");
  SQ_CUDA(cudaMemcpy(host_out, t.dev, sizeof(float) * (size_t)t.numel(), cudaMemcpyDeviceToHost));
  return SQDET_OK;
}

int sqdet_num_ops(sqdet_engine* e) { return e ? (int)e->ops.size() + 2 : SQDET_ERR_INVALID_ARG; }

int sqdet_op_info(sqdet_engine* e, int index, char* name_buf, int name_cap, int64_t* flops,
                  int64_t* params, int64_t* min_bytes) {
  if (!e || index < 0 || index >= (int)e->ops.size() + 2)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_op_info: bad index");
  std::string name;
  int64_t fl = 0, pa = 0, by = 0;
  const int nops = (int)e->ops.size();
  if (index < nops) {
    const Op& op = e->ops[index];
    name = op.name; fl = op.flops; pa = op.params; by = op.min_bytes;
  } else {
    const int64_t B = e->cfg.batch_size, A = e->num_anchors;
    if (index == nops) {
      name = "interpret_output";
      by = e->preds >= 0 ? 4 * e->tensors[e->preds].numel() + B * A * (16 + 4 + 8) : 0;
    } else {
      name = "filter_prediction";
      by = B * A * 4 + B * (int64_t)e->max_dets * (int64_t)sizeof(sqdet_det);
    }
  }
  if (name_buf && name_cap > 0) {
    strncpy(name_buf, name.c_str(), (size_t)name_cap - 1);
    name_buf[name_cap - 1] = 0;
  }
  if (flops) *flops = fl;
  if (params) *params = pa;
  if (min_bytes) *min_bytes = by;
  return SQDET_OK;
}

int sqdet_op_k_split(sqdet_engine* e, int index) {
  if (!e || index < 0 || index >= (int)e->ops.size() + 2)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_op_k_split: bad index");
  int s = 1;
  if (index < (int)e->ops.size())
    for (const auto& l : e->ops[index].launches)
      if (l.kind == L_CONV_TC) s = std::max(s, tc_conv_k_split(l.tc));
  return s;
}

int sqdet_forward(sqdet_engine* e, const float* images_dev, void* stream) {
  return sqdet_forward_n(e, images_dev, e ? e->cfg.batch_size : 0, stream);
}

int sqdet_forward_n(sqdet_engine* e, const float* images_dev, int n, void* stream) {
  return forward_impl(e, images_dev, false, n, e ? e->box_scale : nullptr, (cudaStream_t)stream);
}

int sqdet_forward_u8(sqdet_engine* e, const uint8_t* images_dev, int n, void* stream) {
  return forward_impl(e, images_dev, true, n, e ? e->box_scale : nullptr, (cudaStream_t)stream);
}

int sqdet_forward_profiled(sqdet_engine* e, const float* images_dev, void* stream_v,
                           float* op_ms) {
  if (!e || !op_ms) return fail(SQDET_ERR_INVALID_ARG, "sqdet_forward_profiled: null argument");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_forward_profiled before sqdet_finalize");
  if (!images_dev) return fail(SQDET_ERR_INVALID_ARG, "null images pointer");
  cudaStream_t stream = (cudaStream_t)stream_v;
  DeviceGuard guard(e->device);
  int rc = prepare_params(e);
  if (rc) return rc;
  const int n = (int)e->ops.size() + 2;
  while ((int)e->prof_events.size() < n + 1) {
    cudaEvent_t ev;
    SQ_CUDA(cudaEventCreate(&ev));
    e->prof_events.push_back(ev);
  }
  const int B = e->cfg.batch_size;
  SQ_CUDA(cudaEventRecord(e->prof_events[0], stream));
  for (int i = 0; i < (int)e->ops.size(); ++i) {
    rc = run_op(e, e->ops[i], images_dev, nullptr, B, stream);
    if (rc) return rc;
    SQ_CUDA(cudaEventRecord(e->prof_events[i + 1], stream));
  }
  rc = run_interpret(e, B, e->box_scale, stream);
  if (rc) return rc;
  SQ_CUDA(cudaEventRecord(e->prof_events[n - 1], stream));
  rc = run_filter(e, B, stream);
  if (rc) return rc;
  SQ_CUDA(cudaEventRecord(e->prof_events[n], stream));
  SQ_CUDA(cudaEventSynchronize(e->prof_events[n]));
  for (int i = 0; i < n; ++i)
    SQ_CUDA(cudaEventElapsedTime(&op_ms[i], e->prof_events[i], e->prof_events[i + 1]));
  return SQDET_OK;
}

int sqdet_results_dev(sqdet_engine* e, float** det_boxes, float** det_probs, int64_t** det_class,
                      sqdet_det** dets, int32_t** counts, int32_t* max_dets) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_results_dev before sqdet_finalize");
  if (det_boxes) *det_boxes = e->d_boxes;
  if (det_probs) *det_probs = e->d_probs;
  if (det_class) *det_class = e->d_cls;
  if (dets) *dets = e->d_dets;
  if (counts) *counts = e->d_counts;
  if (max_dets) *max_dets = e->max_dets;
  return SQDET_OK;
}

int sqdet_detect(sqdet_engine* e, const float* images, float* det_boxes, float* det_probs,
                 int64_t* det_class, sqdet_det* dets, int32_t* counts, void* stream_v) {
  if (!e || !images) return fail(SQDET_ERR_INVALID_ARG, "sqdet_detect: null argument");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_detect before sqdet_finalize");
  DeviceGuard guard(e->device);
  cudaStream_t stream = stream_v ? (cudaStream_t)stream_v : e->own_stream;
  const sqdet_config& c = e->cfg;
  const size_t in_bytes = sizeof(float) * (size_t)e->tensors[0].numel();
  SQ_CUDA(cudaMemcpyAsync(e->tensors[0].dev, images, in_bytes, cudaMemcpyHostToDevice, stream));
  int rc = forward_impl(e, e->tensors[0].dev, false, c.batch_size, e->box_scale, stream);
  if (rc) return rc;
  const size_t BA = (size_t)c.batch_size * (size_t)e->num_anchors;
  if (det_boxes)
    SQ_CUDA(cudaMemcpyAsync(det_boxes, e->d_boxes, sizeof(float) * BA * 4, cudaMemcpyDeviceToHost, stream));
  if (det_probs)
    SQ_CUDA(cudaMemcpyAsync(det_probs, e->d_probs, sizeof(float) * BA, cudaMemcpyDeviceToHost, stream));
  if (det_class)
    SQ_CUDA(cudaMemcpyAsync(det_class, e->d_cls, sizeof(int64_t) * BA, cudaMemcpyDeviceToHost, stream));
  if (dets)
    SQ_CUDA(cudaMemcpyAsync(dets, e->d_dets, sizeof(sqdet_det) * (size_t)c.batch_size * e->max_dets,
                            cudaMemcpyDeviceToHost, stream));
  if (counts)
    SQ_CUDA(cudaMemcpyAsync(counts, e->d_counts, sizeof(int32_t) * (size_t)c.batch_size,
                            cudaMemcpyDeviceToHost, stream));
  SQ_CUDA(cudaStreamSynchronize(stream));
  return SQDET_OK;
}

int sqdet_set_bgr_means(sqdet_engine* e, const double bgr_means[3]) {
  if (!e || !bgr_means) return fail(SQDET_ERR_INVALID_ARG, "sqdet_set_bgr_means: null argument");
  // a uint8 forward's graph holds the means it was captured with
  if (memcmp(e->bgr_means, bgr_means, sizeof(e->bgr_means)) != 0) {
    DeviceGuard guard(e->device);
    drop_graph(e, true);
  }
  for (int i = 0; i < 3; ++i) e->bgr_means[i] = bgr_means[i];
  return SQDET_OK;
}

int sqdet_submit(sqdet_engine* e, const void* images, int img_type, sqdet_det* dets,
                 int32_t* counts) {
  if (!e || !images) return fail(SQDET_ERR_INVALID_ARG, "sqdet_submit: null argument");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_submit before sqdet_finalize");
  if (img_type != SQDET_IMG_F32 && img_type != SQDET_IMG_U8)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_submit: unknown img_type");
  DeviceGuard guard(e->device);
  const sqdet_config& c = e->cfg;
  Slot* s;
  int rc = begin_submit(e, "sqdet_submit", &s);
  if (rc) return rc;
  const bool u8 = img_type == SQDET_IMG_U8;
  const int64_t n_pix = (int64_t)c.batch_size * c.image_height * c.image_width;
  const size_t bytes = (size_t)n_pix * 3 * (u8 ? 1 : sizeof(float));
  const uint8_t* src = static_cast<const uint8_t*>(images);
  const size_t off = 0;
  rc = upload(e, *s, !u8, 1, &src, &bytes, &off);
  if (rc) return rc;
  return finish_submit(e, *s, u8 ? (const void*)s->staging : s->input, u8, c.batch_size,
                       e->box_scale, dets, counts);
}

int sqdet_wait(sqdet_engine* e) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  if (e->n_waited >= e->n_submitted) return fail(SQDET_ERR_STATE, "sqdet_wait: nothing in flight");
  DeviceGuard guard(e->device);
  SQ_CUDA(cudaEventSynchronize(e->slots[e->n_waited & 1].done));
  ++e->n_waited;
  return SQDET_OK;
}

int sqdet_launches_per_forward(sqdet_engine* e) {
  if (!e) return SQDET_ERR_INVALID_ARG;
  int n = 2 + (e->box_scale ? 1 : 0);   // interpret [+ rescale] + filter (NCCL's own kernel not counted)
  for (const auto& op : e->ops) n += (int)op.launches.size();
  return n;
}


// ---- eval-order rescale ---------------------------------------------------------------------------
int sqdet_set_box_scale(sqdet_engine* e, const float* xy_scales) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_set_box_scale before sqdet_finalize");
  DeviceGuard guard(e->device);
  const size_t n = (size_t)e->cfg.batch_size * 2;
  for (size_t i = 0; xy_scales && i < n; ++i)
    if (!(xy_scales[i] > 0.f)) return fail(SQDET_ERR_INVALID_ARG, "sqdet_set_box_scale: scales must be positive");
  // synchronous: no forward may be in flight while the table changes or goes.  No graph is
  // dropped: a graph reads the table at its key's address, whichever table is allocated there.
  SQ_CUDA(cudaEventSynchronize(e->last_forward));
  if (!xy_scales) {
    cudaFree(e->box_scale);
    e->box_scale = nullptr;
    return SQDET_OK;
  }
  if (!e->box_scale) SQ_CUDA(cudaMalloc(&e->box_scale, sizeof(float) * n));
  SQ_CUDA(cudaMemcpy(e->box_scale, xy_scales, sizeof(float) * n, cudaMemcpyHostToDevice));
  // the copy from pageable memory may return before its DMA lands; the next forward must not
  SQ_CUDA(cudaStreamSynchronize(nullptr));
  return SQDET_OK;
}

// ---- variable-size uint8 frames in front of the path (SURVEY 8 f-1) --------------------------------
int sqdet_submit_frames(sqdet_engine* e, const uint8_t* const* frames, const int32_t* heights,
                        const int32_t* widths, int order, int rescale, sqdet_det* dets,
                        int32_t* counts) {
  return sqdet_submit_frames_n(e, e ? e->cfg.batch_size : 0, frames, heights, widths, order,
                               rescale, dets, counts);
}

int sqdet_submit_frames_n(sqdet_engine* e, int n, const uint8_t* const* frames,
                          const int32_t* heights, const int32_t* widths, int order, int rescale,
                          sqdet_det* dets, int32_t* counts) {
  if (!e || !frames || !heights || !widths)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_submit_frames: null argument");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_submit_frames before sqdet_finalize");
  if (order != SQDET_PRE_RESIZE_THEN_SUB && order != SQDET_PRE_SUB_THEN_RESIZE)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_submit_frames: order must be 0 (demo) or 1 (eval)");
  const sqdet_config& c = e->cfg;
  const int B = c.batch_size;
  if (n < 1 || n > B)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_submit_frames_n: n must be in [1, batch_size]");
  DeviceGuard guard(e->device);
  Slot* s;
  int rc = begin_submit(e, "sqdet_submit_frames", &s);
  if (rc) return rc;
  std::vector<size_t> bytes((size_t)n), off((size_t)n);
  size_t end = 0;
  for (int i = 0; i < n; ++i) {
    if (!frames[i] || heights[i] <= 0 || widths[i] <= 0)
      return fail(SQDET_ERR_INVALID_ARG, "sqdet_submit_frames: empty frame");
    bytes[(size_t)i] = (size_t)heights[i] * widths[i] * 3;
    off[(size_t)i] = end;                                   // 256-byte aligned staging offsets
    end += (bytes[(size_t)i] + 255) & ~(size_t)255;
  }
  // eval order: boxes go back to each frame's own pixel grid before the filter (eval.py:80-87).
  // The resize launch writes the slot's table in stream order behind the forward that last read it.
  if (rescale && !s->scales) SQ_CUDA(cudaMalloc(&s->scales, sizeof(float) * (size_t)B * 2));
  rc = upload(e, *s, false, n, frames, bytes.data(), off.data());
  if (rc) return rc;
  std::vector<FrameSource> fr((size_t)n);
  for (int i = 0; i < n; ++i)
    fr[(size_t)i] = {{s->staging + off[(size_t)i]}, {3 * (int64_t)widths[i]}, 0, 0, heights[i],
                     widths[i]};
  float* scales = rescale ? s->scales : nullptr;
  rc = launch_resize_meansub_frames(SQDET_FMT_BGR, fr.data(), n, s->input, c.image_height,
                                    c.image_width, e->bgr_means, order == SQDET_PRE_SUB_THEN_RESIZE,
                                    scales, e->own_stream);
  if (rc) return rc;
  return finish_submit(e, *s, s->input, false, n, scales, dets, counts);
}

// ---- variable-size uint8 frames already in device memory ----------------------------------------
// Before the resize launch of a device-frames forward: the weights first, since their upload waits
// for the forwards in flight and the resize must not be left behind a failed one; then, with
// rescale, the box-scale table the launch writes, at *scales (null without rescale).
static int prepare_frames(sqdet_engine* e, int rescale, float** scales) {
  const int rc = prepare_params(e);
  if (rc) return rc;
  if (rescale && !e->frame_scales)
    SQ_CUDA(cudaMalloc(&e->frame_scales, sizeof(float) * (size_t)e->cfg.batch_size * 2));
  *scales = rescale ? e->frame_scales : nullptr;
  return SQDET_OK;
}

// The refusals of a device-frames forward before it reads any per-frame entry; null_arg: the engine
// or an array the call needs is null.
static int check_frames_call(sqdet_engine* e, const std::string& name, bool null_arg, int n,
                             int order) {
  if (null_arg) return fail(SQDET_ERR_INVALID_ARG, name + ": null argument");
  if (!e->finalized) return fail(SQDET_ERR_STATE, name + " before sqdet_finalize");
  if (n < 1 || n > e->cfg.batch_size)
    return fail(SQDET_ERR_INVALID_ARG, name + ": n must be in [1, batch_size]");
  if (order != SQDET_PRE_RESIZE_THEN_SUB && order != SQDET_PRE_SUB_THEN_RESIZE)
    return fail(SQDET_ERR_INVALID_ARG, name + ": order must be 0 (demo) or 1 (eval)");
  return SQDET_OK;
}

// sqdet_forward_frames, whose refusals name the call `name` and image i as image(i) (by default
// "frame i").
static int forward_frames(sqdet_engine* e, const std::string& name, int n, int format,
                          const uint8_t* const* planes, const int64_t* pitches,
                          const int32_t* heights, const int32_t* widths, const int32_t* crops,
                          int order, int rescale, void* stream_v,
                          const std::function<std::string(int)>& image = nullptr) {
  const PixFormat* pf = pix_format(format);
  if (!pf) return fail(SQDET_ERR_INVALID_ARG, name + ": unknown format");
  int rc = check_frames_call(e, name, !e || !planes || !heights || !widths, n, order);
  if (rc) return rc;
  DeviceGuard guard(e->device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select the engine's device");
  std::vector<FrameSource> fr;
  int device = e->device;
  rc = accept_frames(name, *pf, n, planes, pitches, heights, widths, crops, image, &device, fr);
  if (rc) return rc;
  cudaStream_t stream = (cudaStream_t)stream_v;
  float* scales = nullptr;
  rc = prepare_frames(e, rescale, &scales);
  if (rc) return rc;
  const sqdet_config& c = e->cfg;
  Tensor& t0 = e->tensors[0];
  rc = launch_resize_meansub_frames(format, fr.data(), n, t0.dev, c.image_height, c.image_width,
                                    e->bgr_means, order == SQDET_PRE_SUB_THEN_RESIZE, scales,
                                    stream);
  if (rc) return rc;
  return forward_impl(e, t0.dev, false, n, scales, stream);
}

// sqdet_forward_frames_u8 and _nv12, which pass plane p of frame i at planes[p][i] and its row
// pitch at pitches[p][i] (tight rows when pitches[p] is null): once the arrays are known to hold n
// entries, they are laid out as sqdet_forward_frames takes them.
static int forward_plane_arrays(sqdet_engine* e, const std::string& name, int n, int format,
                                const uint8_t* const* const (&planes)[2],
                                const int64_t* const (&pitches)[2], const int32_t* heights,
                                const int32_t* widths, const int32_t* crops, int order,
                                int rescale, void* stream) {
  const PixFormat& pf = *pix_format(format);
  bool null_arg = !e || !heights || !widths;
  for (int p = 0; p < pf.planes; ++p) null_arg = null_arg || !planes[p];
  const int rc = check_frames_call(e, name, null_arg, n, order);
  if (rc) return rc;
  std::vector<const uint8_t*> fp(3 * (size_t)n);
  std::vector<int64_t> fq(3 * (size_t)n);
  for (int i = 0; i < n; ++i)
    for (int p = 0; p < pf.planes; ++p) {
      fp[3 * (size_t)i + p] = planes[p][i];
      fq[3 * (size_t)i + p] = pitches[p] ? pitches[p][i] : pf.plane[p].row_bytes(widths[i]);
    }
  return forward_frames(e, name, n, format, fp.data(), fq.data(), heights, widths, crops, order,
                        rescale, stream);
}

int sqdet_forward_frames(sqdet_engine* e, int n, int format, const uint8_t* const* planes,
                         const int64_t* pitches, const int32_t* heights, const int32_t* widths,
                         const int32_t* crops, int order, int rescale, void* stream) {
  return forward_frames(e, "sqdet_forward_frames", n, format, planes, pitches, heights, widths,
                        crops, order, rescale, stream);
}

int sqdet_forward_frames_u8(sqdet_engine* e, int n, const uint8_t* const* frames_dev,
                            const int32_t* heights, const int32_t* widths,
                            const int64_t* row_pitches, int order, int rescale, void* stream) {
  return forward_plane_arrays(e, "sqdet_forward_frames_u8", n, SQDET_FMT_BGR, {frames_dev, nullptr},
                              {row_pitches, nullptr}, heights, widths, nullptr, order, rescale,
                              stream);
}

int sqdet_forward_frames_nv12(sqdet_engine* e, int n, const uint8_t* const* luma_dev,
                              const int64_t* luma_pitches, const uint8_t* const* chroma_dev,
                              const int64_t* chroma_pitches, const int32_t* heights,
                              const int32_t* widths, const int32_t* crops, int order, int rescale,
                              void* stream) {
  return forward_plane_arrays(e, "sqdet_forward_frames_nv12", n, SQDET_FMT_NV12,
                              {luma_dev, chroma_dev}, {luma_pitches, chroma_pitches}, heights,
                              widths, crops, order, rescale, stream);
}

// ---- whole frames as overlapping tiles, merged per frame ---------------------------------------
int sqdet_forward_tiles(sqdet_engine* e, int n, int format, const uint8_t* const* planes,
                        const int64_t* pitches, const int32_t* heights, const int32_t* widths,
                        int t, const int32_t* tiles, int order, void* stream) {
  const std::string name = "sqdet_forward_tiles";
  if (!e || !planes || !heights || !widths || !tiles)
    return fail(SQDET_ERR_INVALID_ARG, name + ": null argument");
  if (!e->finalized) return fail(SQDET_ERR_STATE, name + " before sqdet_finalize");
  const sqdet_config& c = e->cfg;
  if (t < 1 || t > c.batch_size)
    return fail(SQDET_ERR_INVALID_ARG, name + ": t must be in [1, batch_size]");
  std::vector<int32_t> frame_of((size_t)t), xy((size_t)t * 2), crops((size_t)t * 4);
  std::vector<int32_t> hs((size_t)t), ws((size_t)t);
  for (int k = 0; k < t; ++k) frame_of[(size_t)k] = tiles[5 * k];
  int rc = check_merge_tiles(name.c_str(), (int)e->num_anchors, t, frame_of.data(), n,
                             c.top_n_detection, e->max_dets);
  if (rc) return rc;
  auto tile = [&](int k) {
    return "tile " + std::to_string(k) + " (frame " + std::to_string(frame_of[(size_t)k]) + ")";
  };
  for (int k = 0; k < t; ++k) {
    const int f = frame_of[(size_t)k];
    const int64_t x = tiles[5 * k + 1], y = tiles[5 * k + 2], w = tiles[5 * k + 3],
                  h = tiles[5 * k + 4];
    const std::string which = name + ": " + tile(k);
    if (w <= 0 || h <= 0) return fail(SQDET_ERR_INVALID_ARG, which + " is empty");
    if (x < 0 || y < 0 || x + w > widths[f] || y + h > heights[f])
      return fail(SQDET_ERR_INVALID_ARG, which + " is outside its frame");
    xy[2 * (size_t)k] = (int32_t)x;
    xy[2 * (size_t)k + 1] = (int32_t)y;
    for (int j = 0; j < 4; ++j) crops[4 * (size_t)k + j] = tiles[5 * k + 1 + j];
    hs[(size_t)k] = heights[f];
    ws[(size_t)k] = widths[f];
  }
  // image k of the forward is tile k: its frame's planes and pitches, cropped to the tile
  std::vector<const uint8_t*> tp((size_t)t * 3);
  std::vector<int64_t> tq(pitches ? (size_t)t * 3 : 0);
  for (int k = 0; k < t; ++k)
    for (int p = 0; p < 3; ++p) {
      const size_t src = 3 * (size_t)frame_of[(size_t)k] + p;
      tp[3 * (size_t)k + p] = planes[src];
      if (pitches) tq[3 * (size_t)k + p] = pitches[src];
    }
  rc = forward_frames(e, name, t, format, tp.data(), pitches ? tq.data() : nullptr, hs.data(),
                      ws.data(), crops.data(), order, 1, stream, tile);
  if (rc) return rc;
  DeviceGuard guard(e->device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select the engine's device");
  cudaStream_t s = (cudaStream_t)stream;
  rc = launch_merge_tiles("sqdet_forward_tiles", e->d_boxes, e->d_probs, e->d_cls,
                          (int)e->num_anchors, t, frame_of.data(), xy.data(), n, c.batch_size,
                          c.classes, c.top_n_detection, c.prob_thresh, c.nms_thresh,
                          e->d_tile_cand, e->d_tile_dets, e->d_tile_counts, e->max_dets, s);
  if (rc) return rc;
  // a weight reload or sqdet_set_box_scale waits for the merge too
  SQ_CUDA(cudaEventRecord(e->last_forward, s));
  return SQDET_OK;
}

int sqdet_tile_results_dev(sqdet_engine* e, sqdet_det** dets, int32_t** counts,
                           int32_t* max_dets) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "sqdet_tile_results_dev: null engine");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_tile_results_dev before sqdet_finalize");
  if (dets) *dets = e->d_tile_dets;
  if (counts) *counts = e->d_tile_counts;
  if (max_dets) *max_dets = e->max_dets;
  return SQDET_OK;
}

// ---- multi-GPU: ONE all-gather of the filtered records ---------------------------------------------
int sqdet_comm_unique_id(void* id128) {
  if (!id128) return fail(SQDET_ERR_INVALID_ARG, "sqdet_comm_unique_id: null buffer");
  int rc = nccl_load();
  if (rc) return rc;
  NcclId id;
  const int r = g_nccl.GetUniqueId(&id);
  if (r != 0) return nccl_fail(r, "ncclGetUniqueId");
  memcpy(id128, id.internal, 128);
  return SQDET_OK;
}

static int comm_buffers(sqdet_engine* e) {
  e->blob_bytes = sizeof(sqdet_det) * (size_t)e->cfg.batch_size * e->max_dets +
                  sizeof(int32_t) * (size_t)e->cfg.batch_size;
  cudaFree(e->d_gathered);
  e->d_gathered = nullptr;
  SQ_CUDA(cudaMalloc(&e->d_gathered, e->blob_bytes * (size_t)e->comm_nranks));
  SQ_CUDA(cudaMemset(e->d_gathered, 0, e->blob_bytes * (size_t)e->comm_nranks));
  return SQDET_OK;
}

int sqdet_comm_init(sqdet_engine* e, int nranks, int rank, const void* id128) {
  if (!e || !id128) return fail(SQDET_ERR_INVALID_ARG, "sqdet_comm_init: null argument");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_comm_init before sqdet_finalize");
  if (nranks <= 0 || rank < 0 || rank >= nranks)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_comm_init: bad nranks/rank");
  if (e->comm) return fail(SQDET_ERR_STATE, "sqdet_comm_init: a communicator is already attached");
  int rc = nccl_load();
  if (rc) return rc;
  DeviceGuard guard(e->device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select the engine's device");
  NcclId id;
  memcpy(id.internal, id128, 128);
  void* comm = nullptr;
  const int r = g_nccl.CommInitRank(&comm, nranks, id, rank);
  if (r != 0) return nccl_fail(r, "ncclCommInitRank");
  e->comm = comm;
  e->comm_owned = true;
  e->comm_nranks = nranks;
  e->comm_rank = rank;
  rc = comm_buffers(e);
  if (rc) return rc;
  // one eager collective so that channels / peer connections exist before any graph capture
  rc = run_allgather(e, e->comm, e->own_stream);
  if (rc) return rc;
  SQ_CUDA(cudaStreamSynchronize(e->own_stream));
  return SQDET_OK;
}

int sqdet_comm_attach(sqdet_engine* e, void* nccl_comm, int nranks, int rank) {
  if (!e || !nccl_comm) return fail(SQDET_ERR_INVALID_ARG, "sqdet_comm_attach: null argument");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_comm_attach before sqdet_finalize");
  if (nranks <= 0 || rank < 0 || rank >= nranks)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_comm_attach: bad nranks/rank");
  if (e->comm) return fail(SQDET_ERR_STATE, "sqdet_comm_attach: a communicator is already attached");
  int rc = nccl_load();
  if (rc) return rc;
  DeviceGuard guard(e->device);
  e->comm = nccl_comm;
  e->comm_owned = false;
  e->comm_nranks = nranks;
  e->comm_rank = rank;
  return comm_buffers(e);
}

int sqdet_comm_destroy(sqdet_engine* e) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  DeviceGuard guard(e->device);
  cudaDeviceSynchronize();
  drop_graph(e);
  if (e->comm && e->comm_owned && g_nccl.CommDestroy) g_nccl.CommDestroy(e->comm);
  e->comm = nullptr;
  e->comm_owned = false;
  e->gather_in_forward = false;
  cudaFree(e->d_gathered);
  e->d_gathered = nullptr;
  return SQDET_OK;
}

int sqdet_set_gather_in_forward(sqdet_engine* e, int on) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  if (on && !e->comm) return fail(SQDET_ERR_STATE, "sqdet_set_gather_in_forward: no communicator");
  if ((on != 0) != e->gather_in_forward) {
    e->gather_in_forward = on != 0;
    drop_graph(e);
  }
  return SQDET_OK;
}

int sqdet_allgather(sqdet_engine* e, void* nccl_comm, void* stream) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  if (!e->finalized) return fail(SQDET_ERR_STATE, "sqdet_allgather before sqdet_finalize");
  DeviceGuard guard(e->device);
  return run_allgather(e, nccl_comm ? nccl_comm : e->comm, (cudaStream_t)stream);
}

int sqdet_gathered_dev(sqdet_engine* e, void** gathered, int64_t* bytes_per_rank, int32_t* nranks) {
  if (!e) return fail(SQDET_ERR_INVALID_ARG, "null engine");
  if (!e->d_gathered) return fail(SQDET_ERR_STATE, "sqdet_gathered_dev: no communicator attached");
  if (gathered) *gathered = e->d_gathered;
  if (bytes_per_rank) *bytes_per_rank = (int64_t)e->blob_bytes;
  if (nranks) *nranks = e->comm_nranks;
  return SQDET_OK;
}

void* sqdet_engine_stream(sqdet_engine* e) { return e ? (void*)e->own_stream : nullptr; }

// ---- stage-isolated kernels ------------------------------------------------------------------
// The epilogue arguments every conv entry point checks before any device work, whichever kernel
// then runs: scale and shift come together, and the Cout output channels at y_coff lie inside
// each pixel's y_cstride channels.
static int check_conv_epilogue(const char* who, const float* scale_dev, const float* shift_dev,
                               int Cout, int y_cstride, int y_coff) {
  if ((scale_dev == nullptr) != (shift_dev == nullptr))
    return fail(SQDET_ERR_INVALID_ARG, std::string(who) + ": scale and shift must be given together");
  if (y_coff < 0 || (long long)y_coff + Cout > y_cstride)
    return fail(SQDET_ERR_INVALID_ARG, std::string(who) + ": output channel window out of range");
  return SQDET_OK;
}

int sqdet_conv2d(const float* x_dev, const float* w_hwio_dev, const float* bias_dev,
                 const float* scale_dev, const float* shift_dev, float* y_dev, int B, int H, int W,
                 int Cin, int Cout, int size, int stride, int padding, int relu, int y_cstride,
                 int y_coff, int math_mode, void* stream) {
  return sqdet_conv2d_k_split(x_dev, w_hwio_dev, bias_dev, scale_dev, shift_dev, y_dev, B, H, W, Cin,
                              Cout, size, stride, padding, relu, y_cstride, y_coff, math_mode, 0, stream);
}

int sqdet_conv2d_k_split(const float* x_dev, const float* w_hwio_dev, const float* bias_dev,
                         const float* scale_dev, const float* shift_dev, float* y_dev, int B, int H,
                         int W, int Cin, int Cout, int size, int stride, int padding, int relu,
                         int y_cstride, int y_coff, int math_mode, int k_split, void* stream) {
  if (!x_dev || !w_hwio_dev || !y_dev) return fail(SQDET_ERR_INVALID_ARG, "sqdet_conv2d: null pointer");
  if (k_split < 0 || k_split > 4) return fail(SQDET_ERR_INVALID_ARG, "sqdet_conv2d: k_split outside [0, 4]");
  if (k_split > 1 && math_mode != SQDET_MATH_TF32X3_TC)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_conv2d: a K split needs SQDET_MATH_TF32X3_TC");
  if (padding != SQDET_PAD_SAME && padding != SQDET_PAD_VALID)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_conv2d: padding must be SAME(0) or VALID(1)");
  if (int rc = check_conv_epilogue("sqdet_conv2d", scale_dev, shift_dev, Cout, y_cstride, y_coff))
    return rc;
  if (math_mode != SQDET_MATH_FP32_SIMT && math_mode != SQDET_MATH_TF32X3_TC)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_conv2d: unknown math_mode");
  if (math_mode == SQDET_MATH_TF32X3_TC) {
    TcConvPlan plan;
    int rc = tc_conv_plan(&plan, B, H, W, Cin, {{size, Cout, y_coff}}, stride, padding, relu,
                          scale_dev != nullptr, y_cstride, k_split);
    if (rc >= 0)
      rc = tc_conv_oneshot(&plan, {w_hwio_dev}, {bias_dev}, scale_dev, shift_dev, x_dev, y_dev,
                           (cudaStream_t)stream);
    if (rc == 1 && k_split > 1)
      return fail(SQDET_ERR_INVALID_ARG, "sqdet_conv2d: a K split needs a shape the tensor-core path takes");
    if (rc != 1) return rc;   // 1 = shape not taken by the tensor-core path (e.g. a strided conv)
  }
  // the fp32 SIMT kernel: the same dispatch as the engine
  ConvArgs a;
  a.x = x_dev; a.w = w_hwio_dev; a.bias = bias_dev; a.scale = scale_dev; a.shift = shift_dev;
  a.y = y_dev; a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.size = size;
  a.stride = stride; a.padding = padding; a.relu = relu; a.y_cstride = y_cstride; a.y_coff = y_coff;
  return launch_conv_simt(a, (cudaStream_t)stream);
}

/* SqueezeDet._fire_layer as ONE stage-isolated call (src/nets/squeezeDet.py:81-106). */
int sqdet_fire(const float* x_dev, const float* w_sq_dev, const float* b_sq_dev,
               const float* w_e1_dev, const float* b_e1_dev, const float* w_e3_dev,
               const float* b_e3_dev, float* y_dev, int B, int H, int W, int Cin, int S, int E1,
               int E3, int math_mode, void* stream_v) {
  if (!x_dev || !w_sq_dev || !b_sq_dev || !w_e1_dev || !b_e1_dev || !w_e3_dev || !b_e3_dev || !y_dev)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_fire: null pointer");
  if (B <= 0 || H <= 0 || W <= 0 || Cin <= 0 || S <= 0 || E1 <= 0 || E3 <= 0)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_fire: non-positive dimension");
  if (math_mode != SQDET_MATH_FP32_SIMT && math_mode != SQDET_MATH_TF32X3_TC)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_fire: unknown math_mode");
  cudaStream_t stream = (cudaStream_t)stream_v;
  if (math_mode == SQDET_MATH_TF32X3_TC) {
    TcConvPlan plan;
    int rc = tc_fire_plan(&plan, B, H, W, Cin, S, E1, E3);
    if (rc >= 0)
      rc = tc_conv_oneshot(&plan, {w_sq_dev, w_e1_dev, w_e3_dev}, {b_sq_dev, b_e1_dev, b_e3_dev},
                           nullptr, nullptr, x_dev, y_dev, stream);
    if (rc != 1) return rc;   // 1 = shape not taken by the one-kernel fire
  }
  // squeeze tensor through HBM, then the two expand convs into the concat tensor
  float* q = nullptr;
  SQ_CUDA(cudaMalloc(&q, sizeof(float) * (size_t)B * H * W * S));
  int rc = sqdet_conv2d(x_dev, w_sq_dev, b_sq_dev, nullptr, nullptr, q, B, H, W, Cin, S, 1, 1,
                        SQDET_PAD_SAME, 1, S, 0, math_mode, stream_v);
  if (!rc)
    rc = sqdet_conv2d(q, w_e1_dev, b_e1_dev, nullptr, nullptr, y_dev, B, H, W, S, E1, 1, 1,
                      SQDET_PAD_SAME, 1, E1 + E3, 0, math_mode, stream_v);
  if (!rc)
    rc = sqdet_conv2d(q, w_e3_dev, b_e3_dev, nullptr, nullptr, y_dev, B, H, W, S, E3, 3, 1,
                      SQDET_PAD_SAME, 1, E1 + E3, E1, math_mode, stream_v);
  cudaError_t ce = cudaStreamSynchronize(stream);
  cudaFree(q);
  if (rc) return rc;
  if (ce != cudaSuccess) return cuda_fail(ce, "sqdet_fire sync");
  return SQDET_OK;
}

int sqdet_maxpool_nhwc(const float* x_dev, float* y_dev, int B, int H, int W, int C, int size,
                       int stride, int padding, void* stream) {
  if (!x_dev || !y_dev) return fail(SQDET_ERR_INVALID_ARG, "sqdet_maxpool_nhwc: null pointer");
  if (padding != SQDET_PAD_SAME && padding != SQDET_PAD_VALID)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_maxpool_nhwc: padding must be SAME(0) or VALID(1)");
  return launch_maxpool(x_dev, y_dev, B, H, W, C, size, stride, padding, (cudaStream_t)stream);
}

int sqdet_preprocess_u8(const uint8_t* src_dev, int src_h, int src_w, float* dst_dev, int dst_h,
                        int dst_w, const double* bgr_means, int order, void* stream) {
  if (!src_dev || !dst_dev || !bgr_means)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_preprocess_u8: null pointer");
  if (order != SQDET_PRE_RESIZE_THEN_SUB && order != SQDET_PRE_SUB_THEN_RESIZE)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_preprocess_u8: order must be 0 (demo) or 1 (eval)");
  const FrameSource f = {{src_dev}, {3 * (int64_t)src_w}, 0, 0, src_h, src_w};
  return launch_resize_meansub_frames(SQDET_FMT_BGR, &f, 1, dst_dev, dst_h, dst_w, bgr_means,
                                      order == SQDET_PRE_SUB_THEN_RESIZE, nullptr,
                                      (cudaStream_t)stream);
}

int sqdet_interpret(const float* preds_dev, const float* anchors_f32_dev, float* det_boxes_dev,
                    float* det_probs_dev, int64_t* det_class_dev, int B, int grid_h, int grid_w,
                    int anchors_per_grid, int classes, int image_width, int image_height,
                    float exp_thresh, void* stream) {
  if (!preds_dev || !anchors_f32_dev || !det_boxes_dev || !det_probs_dev || !det_class_dev)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_interpret: null pointer");
  return launch_interpret(preds_dev, anchors_f32_dev, det_boxes_dev, det_probs_dev, det_class_dev,
                          B, grid_h, grid_w, anchors_per_grid, classes, image_width, image_height,
                          exp_thresh, (cudaStream_t)stream);
}

int sqdet_topk_nms(const float* boxes_dev, const float* probs_dev, const int64_t* cls_dev, int B,
                   int A, int classes, int top_n, float prob_thresh, float nms_thresh,
                   sqdet_det* dets_dev, int32_t* counts_dev, int max_dets, void* stream) {
  if (!boxes_dev || !probs_dev || !cls_dev || !dets_dev || !counts_dev)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_topk_nms: null pointer");
  return launch_topk_nms(boxes_dev, probs_dev, cls_dev, B, A, classes, top_n, prob_thresh,
                         nms_thresh, dets_dev, counts_dev, max_dets, (cudaStream_t)stream);
}

int sqdet_merge_tiles(const float* boxes_dev, const float* probs_dev, const int64_t* cls_dev,
                      int A, int t, const int32_t* tile_frames, const int32_t* tile_xy, int n,
                      int classes, int top_n, float prob_thresh, float nms_thresh,
                      sqdet_det* dets_dev, int32_t* counts_dev, int max_dets, void* stream) {
  if (!boxes_dev || !probs_dev || !cls_dev || !tile_frames || !tile_xy || !dets_dev || !counts_dev)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_merge_tiles: null pointer");
  return launch_merge_tiles("sqdet_merge_tiles", boxes_dev, probs_dev, cls_dev, A, t, tile_frames,
                            tile_xy, n, n, classes, top_n, prob_thresh, nms_thresh, nullptr,
                            dets_dev, counts_dev, max_dets, (cudaStream_t)stream);
}

// ---- memory helpers ------------------------------------------------------------------------------
int sqdet_malloc(int device, int64_t bytes, void** out_dev) {
  if (!out_dev || bytes <= 0) return fail(SQDET_ERR_INVALID_ARG, "sqdet_malloc: bad argument");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "sqdet_malloc: cannot select device");
  SQ_CUDA(cudaMalloc(out_dev, (size_t)bytes));
  return SQDET_OK;
}
int sqdet_free(int device, void* dev) {
  DeviceGuard guard(device);
  if (dev) SQ_CUDA(cudaFree(dev));
  return SQDET_OK;
}
int sqdet_malloc_host(int64_t bytes, void** out_pinned) {
  if (!out_pinned || bytes <= 0) return fail(SQDET_ERR_INVALID_ARG, "sqdet_malloc_host: bad argument");
  SQ_CUDA(cudaMallocHost(out_pinned, (size_t)bytes));
  return SQDET_OK;
}
int sqdet_free_host(void* pinned) {
  if (pinned) SQ_CUDA(cudaFreeHost(pinned));
  return SQDET_OK;
}
int sqdet_memcpy_h2d(void* dst_dev, const void* src, int64_t bytes, void* stream) {
  if (!dst_dev || !src || bytes < 0) return fail(SQDET_ERR_INVALID_ARG, "sqdet_memcpy_h2d: bad argument");
  SQ_CUDA(cudaMemcpyAsync(dst_dev, src, (size_t)bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return SQDET_OK;
}
int sqdet_memcpy_d2h(void* dst, const void* src_dev, int64_t bytes, void* stream) {
  if (!dst || !src_dev || bytes < 0) return fail(SQDET_ERR_INVALID_ARG, "sqdet_memcpy_d2h: bad argument");
  SQ_CUDA(cudaMemcpyAsync(dst, src_dev, (size_t)bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return SQDET_OK;
}
int sqdet_stream_sync(int device, void* stream) {
  DeviceGuard guard(device);
  SQ_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return SQDET_OK;
}

}  // extern "C"
