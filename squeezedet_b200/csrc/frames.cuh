// The per-format pixel fetch of uint8 frames in any SQDET_FMT_* format, shared by the kernels that
// read frames without writing a BGR copy (frames.cu: resize + mean subtraction into tensor 0;
// jpeg.cu, png.cu: JPEG and PNG encoding).  A FrameDesc<P> holds a crop's P planes at its origin,
// taps<F> turns it into the format's fetch, and each fetch converts to B, G, R as the format's
// cv2.cvtColor code does.  dispatch_format picks the instance of a format code for every launcher
// of these kernels and draw.cu's, and encode_frames is the front end both encoders share.
#pragma once
#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace sqdet {

// fn(std::integral_constant<int, F>{}) for the SQDET_FMT_* code F == format, whose result it
// returns; a value outside SQDET_FMT_* is refused.
template <class Fn>
int dispatch_format(int format, Fn&& fn) {
  switch (format) {
    case SQDET_FMT_BGR: return fn(std::integral_constant<int, SQDET_FMT_BGR>{});
    case SQDET_FMT_RGB: return fn(std::integral_constant<int, SQDET_FMT_RGB>{});
    case SQDET_FMT_BGRA: return fn(std::integral_constant<int, SQDET_FMT_BGRA>{});
    case SQDET_FMT_RGBA: return fn(std::integral_constant<int, SQDET_FMT_RGBA>{});
    case SQDET_FMT_RGB_PLANAR: return fn(std::integral_constant<int, SQDET_FMT_RGB_PLANAR>{});
    case SQDET_FMT_NV12: return fn(std::integral_constant<int, SQDET_FMT_NV12>{});
    case SQDET_FMT_I420: return fn(std::integral_constant<int, SQDET_FMT_I420>{});
    default: return fail(SQDET_ERR_INVALID_ARG, "unknown pixel format " + std::to_string(format));
  }
}

// The taps of a packed uint8 frame of kBpp bytes per pixel whose row r starts at src + r * pitch
// (any byte alignment), with B, G, R at byte offsets kB, kG, kR of a pixel (other bytes, such as
// alpha, are never read): a channel is a byte load served by L1.  The layout is a compile-time
// instance, so a tap costs the same address arithmetic as BGR's.
template <int kBpp, int kB, int kG, int kR>
struct PackedTaps {
  const uint8_t* __restrict__ src;
  long long pitch;
  __device__ __forceinline__ float operator()(const int (&ys)[2], const int (&xs)[2], int r, int q,
                                             int c) const {
    return (float)src[(long long)ys[r] * pitch + (long long)xs[q] * kBpp +
                      (c == 0 ? kB : c == 1 ? kG : kR)];
  }
};

// The taps of three uint8 planes holding R, G and B (torch's [3, h, w] image layout): channel c
// (B, G, R) of pixel (y, x) is byte x of row y of plane 2 - c, each plane at any byte and pitch.
struct PlanarTaps {
  const uint8_t* __restrict__ plane[3];
  long long pitch[3];
  __device__ __forceinline__ float operator()(const int (&ys)[2], const int (&xs)[2], int r, int q,
                                             int c) const {
    return (float)plane[2 - c][(long long)ys[r] * pitch[2 - c] + xs[q]];
  }
};

// The taps of a YUV 4:2:0 crop: one luma byte and the U,V samples of its 2x2 chroma block,
// converted as cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420) does (OpenCV's BT.601 limited-range
// ITUR_BT_601_* constants, 20 fraction bits; oracle.nv12.nv12_to_bgr).  kInterleaved: NV12, one
// chroma plane of U,V pairs at u; otherwise I420, separate U and V planes of half the width.
// Crop pixel (y, x) is frame pixel (y0 + y, x0 + x); luma and the chroma planes point at the crop
// origin's byte and chroma sample, and the origin's parity (x_odd, y_odd) picks the chroma block,
// so an odd origin reads the frame's own samples.  int32 suffices: every sum stays below 2^30 in
// magnitude.  Each tap is loaded and converted once, when its channel 0 is asked for.
template <bool kInterleaved>
struct Yuv420Taps {
  const uint8_t* __restrict__ luma;
  const uint8_t* __restrict__ u_plane;
  long long luma_pitch, u_pitch;
  int x_odd, y_odd;
  mutable float bgr[2][2][3];   // tap (r, q), converted at its channel 0
  const uint8_t* __restrict__ v_plane;   // I420 only
  long long v_pitch;
  __device__ __forceinline__ float operator()(const int (&ys)[2], const int (&xs)[2], int r, int q,
                                             int c) const {
    if (c == 0) {
      const int y = ys[r], x = xs[q];
      const int Y = luma[(long long)y * luma_pitch + x];
      const long long cy = (long long)((y + y_odd) >> 1);
      int u, v;
      if (kInterleaved) {
        const uint8_t* uv = u_plane + cy * u_pitch + ((x + x_odd) & ~1);
        u = (int)uv[0] - 128;
        v = (int)uv[1] - 128;
      } else {
        u = (int)u_plane[cy * u_pitch + ((x + x_odd) >> 1)] - 128;
        v = (int)v_plane[cy * v_pitch + ((x + x_odd) >> 1)] - 128;
      }
      const int yy = max(Y - 16, 0) * 1220542 + (1 << 19);
      bgr[r][q][0] = (float)min(max((yy + 2116026 * u) >> 20, 0), 255);
      bgr[r][q][1] = (float)min(max((yy - 852492 * v - 409993 * u) >> 20, 0), 255);
      bgr[r][q][2] = (float)min(max((yy + 1673527 * v) >> 20, 0), 255);
    }
    return bgr[r][q][c];
  }
};

// The planes of format F.
template <int F>
constexpr int kPlanes = F == SQDET_FMT_RGB_PLANAR || F == SQDET_FMT_I420 ? 3
                        : F == SQDET_FMT_NV12                           ? 2
                                                                        : 1;

// The h x w crop of one frame of P planes resized to H x W: plane[p] points at the crop origin's
// sample of plane p (crop_origin), (x_odd, y_odd) is the origin's parity, which picks a 4:2:0
// format's chroma block, scale_* are cv::resize's double scales and box_scale_* the eval-order box
// scales (IMAGE_WIDTH / w, IMAGE_HEIGHT / h) as float32.  56, 72 or 88 bytes.
template <int P>
struct FrameDesc {
  const uint8_t* plane[P];
  int64_t pitch[P];
  double scale_x, scale_y;
  float box_scale_x, box_scale_y;
  int h, w;
  int x_odd, y_odd;
};

// The fetch of format F from its descriptor.
template <int F>
__device__ __forceinline__ auto taps(const FrameDesc<kPlanes<F>>& f) {
  if constexpr (F == SQDET_FMT_BGR) return PackedTaps<3, 0, 1, 2>{f.plane[0], f.pitch[0]};
  else if constexpr (F == SQDET_FMT_RGB) return PackedTaps<3, 2, 1, 0>{f.plane[0], f.pitch[0]};
  else if constexpr (F == SQDET_FMT_BGRA) return PackedTaps<4, 0, 1, 2>{f.plane[0], f.pitch[0]};
  else if constexpr (F == SQDET_FMT_RGBA) return PackedTaps<4, 2, 1, 0>{f.plane[0], f.pitch[0]};
  else if constexpr (F == SQDET_FMT_RGB_PLANAR)
    return PlanarTaps{{f.plane[0], f.plane[1], f.plane[2]}, {f.pitch[0], f.pitch[1], f.pitch[2]}};
  else if constexpr (F == SQDET_FMT_NV12)
    return Yuv420Taps<true>{f.plane[0], f.plane[1], f.pitch[0], f.pitch[1], f.x_odd, f.y_odd, {},
                            nullptr, 0};
  else
    return Yuv420Taps<false>{f.plane[0], f.plane[1], f.pitch[0], f.pitch[1], f.x_odd, f.y_odd, {},
                             f.plane[2], f.pitch[2]};
}

// The B, G, R bytes of crop pixel (y, x).
template <class Taps>
__device__ __forceinline__ void fetch_bgr(const Taps& tp, int y, int x, int& b, int& g, int& r) {
  const int ys[2] = {y, y}, xs[2] = {x, x};
  b = (int)tp(ys, xs, 0, 0, 0);
  g = (int)tp(ys, xs, 0, 0, 1);
  r = (int)tp(ys, xs, 0, 0, 2);
}

// The byte of plane p at the origin of frame s's crop.
inline const uint8_t* crop_origin(const PixFormat& pf, const FrameSource& s, int p) {
  const PixPlane& q = pf.plane[p];
  return s.plane[p] + (int64_t)(s.y >> q.y_shift) * s.pitch[p] +
         (int64_t)(s.x >> q.x_shift) * q.bytes_per_px;
}

// The descriptor of frame s's crop resized to H x W.
template <int P>
FrameDesc<P> frame_desc(const PixFormat& pf, const FrameSource& s, int H, int W) {
  FrameDesc<P> f;
  for (int p = 0; p < P; ++p) {
    f.plane[p] = crop_origin(pf, s, p);
    f.pitch[p] = s.pitch[p];
  }
  // cv::resize: inv_scale = dst / src, scale = 1 / inv_scale (both double)
  f.scale_x = 1.0 / ((double)W / (double)s.w);
  f.scale_y = 1.0 / ((double)H / (double)s.h);
  // eval.py:72-74 / imdb.py:93-95: x_scale = mc.IMAGE_WIDTH / orig_w (Python floats = double)
  f.box_scale_x = (float)((double)W / (double)s.w);
  f.box_scale_y = (float)((double)H / (double)s.h);
  f.h = s.h;
  f.w = s.w;
  f.x_odd = s.x & 1;
  f.y_odd = s.y & 1;
  return f;
}

// ---- the front end of the frame encoders (jpeg.cu, png.cu) ---------------------------------------
// Frames per launch of either encoder, whose descriptors travel in the parameter block.
constexpr int kEncodeFramesPerLaunch = 16;

// fn(first, count) for each group [first, first + count) of up to kEncodeFramesPerLaunch of n
// frames, in order; returns the first nonzero result.
template <class Fn>
int for_each_group(int n, Fn&& fn) {
  for (int first = 0; first < n; first += kEncodeFramesPerLaunch) {
    const int rc = fn(first, std::min(kEncodeFramesPerLaunch, n - first));
    if (rc) return rc;
  }
  return SQDET_OK;
}

// One call of an encoder: every check before any device work, in this order (format, null
// arguments, encode_crops, the codec's settings, cap, scratch and lengths alignment, scratch_bytes,
// accept_frames, the outputs' ranges), then launch(pf, frames) on frame 0's device.  settle(fr,
// need) checks the codec's settings and sets the scratch the crops fr need, or returns a refusal.
template <class Settle, class Launch>
int encode_frames(const Encoder& enc, int n, int format, const uint8_t* const* planes,
                  const int64_t* pitches, const int32_t* heights, const int32_t* widths,
                  const int32_t* crops, uint8_t* out_dev, int64_t cap, int64_t* lengths_dev,
                  void* scratch_dev, int64_t scratch_bytes, Settle&& settle, Launch&& launch) {
  const std::string name = enc.call;
  const PixFormat* pf = pix_format(format);
  if (!pf) return fail(SQDET_ERR_INVALID_ARG, name + ": unknown format");
  if (!planes || !heights || !widths || !out_dev || !lengths_dev || !scratch_dev)
    return fail(SQDET_ERR_INVALID_ARG, name + ": null argument");
  std::vector<FrameSource> fr;
  int rc = encode_crops(name, enc, n, heights, widths, crops, fr);
  if (rc) return rc;
  int64_t need = 0;
  rc = settle(fr, need);
  if (rc) return rc;
  if (cap < 1) return fail(SQDET_ERR_INVALID_ARG, name + ": cap must be at least 1");
  // the scratches hold int4, int64, 16-bit and 32-bit atomic regions at 256-byte offsets
  if ((uintptr_t)scratch_dev % 256)
    return fail(SQDET_ERR_INVALID_ARG, name + ": scratch_dev must be 256-byte aligned");
  if ((uintptr_t)lengths_dev % alignof(int64_t))
    return fail(SQDET_ERR_INVALID_ARG, name + ": lengths_dev must be 8-byte aligned");
  if (scratch_bytes < need)
    return fail(SQDET_ERR_INVALID_ARG, name + ": scratch_bytes is below " + enc.scratch_call);
  int device = kFrame0Device;
  rc = accept_frames(name, *pf, n, planes, pitches, heights, widths, crops, nullptr, &device, fr);
  if (rc) return rc;
  const bool out_fits = cap <= INT64_MAX / n && device_range_ok(out_dev, (int64_t)n * cap, device);
  if (!out_fits || !device_range_ok(lengths_dev, (int64_t)n * 8, device) ||
      !device_range_ok(scratch_dev, scratch_bytes, device))
    return fail(SQDET_ERR_INVALID_ARG, name + ": out_dev, lengths_dev or scratch_dev is not inside one "
                                              "device allocation on frame 0's device");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select frame 0's device");
  return launch(*pf, fr.data());
}

}  // namespace sqdet
