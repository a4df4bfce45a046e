// Shared declarations for libsqdet_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <functional>
#include <string>
#include <vector>
#include "../../include/sqdet_b200.h"

namespace sqdet {

// ---- error plumbing (nothing throws across the C ABI) ---------------------------------
void set_error(const std::string& msg);
int  fail(int code, const std::string& msg);
int  cuda_fail(cudaError_t err, const char* what);

#define SQ_CUDA(expr)                                                   \
  do {                                                                  \
    cudaError_t _e = (expr);                                            \
    if (_e != cudaSuccess) return ::sqdet::cuda_fail(_e, #expr);        \
  } while (0)

#define SQ_CHECK_LAUNCH(what)                                           \
  do {                                                                  \
    cudaError_t _e = cudaGetLastError();                                \
    if (_e != cudaSuccess) return ::sqdet::cuda_fail(_e, what);         \
  } while (0)

// ---- scratch layouts --------------------------------------------------------------------------
inline int64_t align256(int64_t v) { return (v + 255) & ~(int64_t)255; }

// Regions of a scratch at 256-byte offsets from base, in the order they are taken.  A call's layout
// is written once, taking from a Carver: with a null base it only counts the scratch size.
struct Carver {
  uint8_t* base = nullptr;
  int64_t offset = 0;
  // The offset of the next `bytes` bytes.
  int64_t next(int64_t bytes) {
    const int64_t at = offset;
    offset += align256(bytes);
    return at;
  }
  // The next `count` T (null when only counting).
  template <class T>
  T* take(int64_t count) {
    const int64_t at = next(count * (int64_t)sizeof(T));
    return base ? reinterpret_cast<T*>(base + at) : nullptr;
  }
};

// ---- TF NHWC geometry (SURVEY App. A.1; tf.nn.conv2d / tf.nn.max_pool) ------------------
struct Geom {
  int out, pad_before, pad_after;
};
inline Geom tf_geometry(int in, int k, int stride, int padding) {
  Geom g;
  if (padding == SQDET_PAD_SAME) {
    g.out = (in + stride - 1) / stride;
    int total = (g.out - 1) * stride + k - in;
    if (total < 0) total = 0;
    g.pad_before = total / 2;
    g.pad_after = total - g.pad_before;
  } else {
    g.out = (in - k) / stride + 1;
    g.pad_before = g.pad_after = 0;
  }
  return g;
}

// ---- kernel launchers (each returns a status; asynchronous on `stream`) ----------------
struct ConvArgs {
  const float* x;       // [B,H,W,Cin]
  const float* w;       // [kh,kw,Cin,Cout] (HWIO)
  const float* bias;    // [Cout] or null
  const float* scale;   // [Cout] or null   (frozen BN: rsqrt(var+eps)*gamma)
  const float* shift;   // [Cout] or null   (beta - mean*scale)
  float* y;             // [B,Ho,Wo,y_cstride], this conv owns channels [y_coff, y_coff+Cout)
  int B, H, W, Cin, Cout, size, stride, padding, relu, y_cstride, y_coff;
};
int launch_conv_simt(const ConvArgs& a, cudaStream_t stream);

bool conv_pool_simt_eligible(int Cin, int Cout, int ksize, int stride, int pool_size,
                             int pool_stride);
// The input is fp32 x, or, when x8 is non-null, uint8 BGR x8 (any byte alignment) from which the
// kernel subtracts bgr_means as it loads it.
int launch_conv_pool_simt(const float* x, const uint8_t* x8, const double* bgr_means,
                          const float* w, const float* bias, const float* scale,
                          const float* shift, float* y, int B, int H, int W, int Cout, int ksize,
                          int conv_padding, int relu, int pool_padding, cudaStream_t stream);

int launch_maxpool(const float* x, float* y, int B, int H, int W, int C, int size,
                   int stride, int padding, cudaStream_t stream);
// The memory layout of a pixel format of sqdet_forward_frames (SQDET_FMT_*).  Plane p of an h x w
// frame holds h >> y_shift rows of (w >> x_shift) * bytes_per_px bytes, and a crop at (x, y) starts
// (y >> y_shift) * pitch + (x >> x_shift) * bytes_per_px bytes into it.
struct PixPlane {
  int bytes_per_px, x_shift, y_shift;
  int64_t row_bytes(int64_t w) const { return (w >> x_shift) * bytes_per_px; }
};
struct PixFormat {
  int planes;
  bool even;                 // 4:2:0 chroma: the height and width must be even
  const char* least_pitch;   // the least row pitch, as a refusal names it
  PixPlane plane[3];
};
// The layout of SQDET_FMT_* `format`, or null for an unknown format.
const PixFormat* pix_format(int format);
// One frame of sqdet_forward_frames: its planes (as many as the format has) and their row
// pitches, and the h x w crop at (x, y) to run.
struct FrameSource {
  const uint8_t* plane[3];
  int64_t pitch[3];
  int x, y, h, w;
};
// The crops of n frames in SQDET_FMT_* `format`, each converted to BGR as the format's
// cv2.cvtColor code does, then cv2.resize (float32 INTER_LINEAR) to H x W and `- means` in either
// order, into the fp32 batch [n, H, W, 3] at dst, without writing a BGR frame: one launch per 64
// (packed), 56 (NV12) or 45 (RGB_PLANAR, I420) frames.  With scales_xy, each frame's box scales
// (W / w, H / h as float32) also go to scales_xy[2i], [2i + 1] on the device.  Refuses an unknown
// format and non-positive sizes; the frames' other checks against pix_format are the caller's.
int launch_resize_meansub_frames(int format, const FrameSource* frames, int n, float* dst, int H,
                                 int W, const double* means, int sub_first, float* scales_xy,
                                 cudaStream_t stream);

// ---- frames and buffers the caller passes in device memory (frames.cu) -------------------------
// Hidden: the library exports the sqdet_* C ABI, not these.
#pragma GCC visibility push(hidden)
// Makes `dev` the current device for the guard's scope; ok is false when that failed.
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
    if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};
// The device whose memory p points into, or -1 when it is not device memory.
int pointer_device(const void* p);
// True when the `bytes` bytes at p are device memory of `device` inside one allocation.  The
// pointer comes from outside the program: a host pointer or an overlong buffer is refused here
// rather than faulting a kernel.
bool device_range_ok(const void* p, int64_t bytes, int device);
// The crop r = (x, y, w, h) of an H x W frame, or the whole frame when r is null, into s.x, s.y,
// s.w and s.h; refuses an empty crop or one outside the frame, naming `which`.
int check_crop(const std::string& which, int64_t H, int64_t W, const int32_t* r, FrameSource& s);
// A frame encoder as its refusals name it: its call, its file format, the call that sizes its
// scratch, and the most frames per call and pixels per crop side it takes.
struct Encoder {
  const char* call;
  const char* file;
  const char* scratch_call;
  int max_frames, max_side;
};
// The crops of an encoder's n frames (heights[i] x widths[i], crops as check_crop takes them) into
// fr, or a refusal naming the call: n outside [1, enc.max_frames], an empty frame, a crop that
// check_crop refuses, or one wider or higher than enc.max_side, which the file cannot hold.  Host
// arrays only: the encoders' size functions call it too.
int encode_crops(const std::string& name, const Encoder& enc, int n, const int32_t* heights,
                 const int32_t* widths, const int32_t* crops, std::vector<FrameSource>& fr);
// accept_frames' device: the one plane 0 of frame 0 is on.
constexpr int kFrame0Device = -1;
// Every check of n frames in format pf before any device work, filling fr or refusing with a
// message that names the call and image(i) (by default "frame i").  Frame i is heights[i] x
// widths[i], its plane p at planes[3i + p] with row pitch pitches[3i + p] (tight rows when
// pitches is null), cropped to crops[4i .. 4i + 3] (the whole frame when crops is null).  Every
// plane must be inside one device allocation on *device (an engine's, as refusals call it), or
// with kFrame0Device on the device plane 0 of frame 0 is on, which *device then holds.
int accept_frames(const std::string& name, const PixFormat& pf, int n,
                  const uint8_t* const* planes, const int64_t* pitches, const int32_t* heights,
                  const int32_t* widths, const int32_t* crops,
                  const std::function<std::string(int)>& image, int* device,
                  std::vector<FrameSource>& fr);
#pragma GCC visibility pop

int launch_add_relu(const float* a, const float* b, float* y, int64_t n, cudaStream_t stream);

int launch_interpret(const float* preds, const float* anchors, float* boxes, float* probs,
                     int64_t* cls, int B, int grid_h, int grid_w, int K, int C,
                     int image_width, int image_height, float exp_thresh,
                     cudaStream_t stream);
int launch_rescale_boxes(float* boxes, const float* scales_xy, int B, int A, cudaStream_t stream);
int launch_topk_nms(const float* boxes, const float* probs, const int64_t* cls, int B,
                    int A, int classes, int top_n, float prob_thresh, float nms_thresh,
                    sqdet_det* dets, int32_t* counts, int max_dets, cudaStream_t stream);

// Tiles of whole frames (sqdet_merge_tiles, sqdet_forward_tiles): tile k is det_* row k of frame
// tile_frames[k], shifted by (tile_xy[2k], tile_xy[2k + 1]).  At most kMaxMergeTiles tiles per call,
// whose descriptors travel in the kernels' parameter blocks.
constexpr int kMaxMergeTiles = 128;
constexpr int kMergeCandBytes = 32;     // one per-tile top-N candidate in the scratch
// Bytes of scratch the per-tile top-N stage of t tiles needs (0 when top_n <= 0).
size_t merge_tiles_scratch_bytes(int t, int A, int top_n);
// Every refusal of a merge of t tiles of A anchors over n frames, before any device work; `what`
// names the call.
int check_merge_tiles(const char* what, int A, int t, const int32_t* tile_frames, int n,
                      int top_n, int max_dets);
// filter_prediction of each frame's union of tile rows into dets [rows, max_dets] / counts [rows];
// rows [n, rows) get count 0.  `scratch` holds merge_tiles_scratch_bytes, or is null to take it
// from the stream-ordered allocator.  One launch, plus the per-tile top-N launch when some frame's
// union is longer than top_n > 0.
int launch_merge_tiles(const char* what, const float* boxes, const float* probs,
                       const int64_t* cls, int A, int t, const int32_t* tile_frames,
                       const int32_t* tile_xy, int n, int rows, int classes, int top_n,
                       float prob_thresh, float nms_thresh, void* scratch, sqdet_det* dets,
                       int32_t* counts, int max_dets, cudaStream_t stream);

}  // namespace sqdet
