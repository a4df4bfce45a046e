// Detection drawing on frames in device memory (sqdet_draw_dets): each kept record is drawn as
// demo.draw_detections + viz.draw_box draw it with cv2 on a uint8 BGR canvas, bit for bit: a 1-px
// cv2.rectangle and a cv2.putText label in FONT_HERSHEY_SIMPLEX, both LINE_8.
//
// OpenCV draws both from one primitive: the 8-connected integer line of cv2.LineIterator (walked
// left to right) after cv2.clipLine against the canvas.  putText places the glyph vertices at
// 16.16 fixed-point positions (pen advance and offsets in units of cvRound(font_scale * 65536)),
// rounds each segment's endpoints to pixels and draws the segment as that line.  The strokes come
// from hershey_simplex.inc (oracle/make_hershey.py); oracle/draw.py restates all of this in numpy.
//
// One CTA per frame walks the kept records in order with a block barrier between records, so a
// later record overwrites an earlier one exactly as the sequential cv2 calls do.  Within a record
// every pixel takes the same colour, so threads split its rectangle pixels and stroke segments
// freely.
#include <math.h>
#include <stdint.h>
#include <string.h>
#include "frames.cuh"

#define SQDET_HERSHEY_SPACE __constant__
#include "hershey_simplex.inc"

namespace sqdet {
namespace {

// sqdet_draw_dets' style as its kernel takes it, by value: per class the colour (B, G, R and its
// (Y, U, V) for 4:2:0 frames) and the name, plus the threshold and cvRound(font_scale * 65536).
constexpr int kDrawMaxClasses = 64;
constexpr int kDrawMaxName = 31;
constexpr int kMaxDrawFrames = 128;     // frames per sqdet_draw_dets call
struct DrawStyle {
  int64_t hscale;
  float thresh;
  int classes;
  uint8_t bgr[kDrawMaxClasses][3];
  uint8_t yuv[kDrawMaxClasses][3];
  uint8_t name_len[kDrawMaxClasses];
  char name[kDrawMaxClasses][kDrawMaxName];
};
// Frames per draw launch: their descriptors and the style stay inside the classic 4 KiB parameter
// block.
constexpr int kDrawFramesPerLaunch = 24;
constexpr int kDrawThreads = 256;
constexpr int kMaxLabel = kDrawMaxName + 9;   // name + ": (" + "-0.00" + ")"

struct DrawParams {
  FrameSource frames[kDrawFramesPerLaunch];
  DrawStyle style;
  const sqdet_det* dets;
  const int32_t* counts;
  int max_dets;
  int first;                                  // the call's index of frames[0]
};
static_assert(sizeof(DrawParams) <= 4096, "draw descriptors must fit the classic parameter block");

// One pixel of the canvas (cx, cy) of frame fs in colour (B, G, R) / (Y, U, V), in the format's
// own layout.  The alpha byte is never written.  A 4:2:0 chroma sample is the one of the pixel's
// 2x2 luma block in frame coordinates.
template <int F>
__device__ __forceinline__ void put_pixel(const FrameSource& fs, int cx, int cy, const uint8_t* bgr,
                                          const uint8_t* yuv) {
  const int64_t x = (int64_t)fs.x + cx, y = (int64_t)fs.y + cy;
  uint8_t* p0 = const_cast<uint8_t*>(fs.plane[0]);
  if (F == SQDET_FMT_RGB_PLANAR) {
    const int64_t off = x;
    p0[y * fs.pitch[0] + off] = bgr[2];
    const_cast<uint8_t*>(fs.plane[1])[y * fs.pitch[1] + off] = bgr[1];
    const_cast<uint8_t*>(fs.plane[2])[y * fs.pitch[2] + off] = bgr[0];
  } else if (F == SQDET_FMT_NV12 || F == SQDET_FMT_I420) {
    p0[y * fs.pitch[0] + x] = yuv[0];
    if (F == SQDET_FMT_NV12) {
      uint8_t* c = const_cast<uint8_t*>(fs.plane[1]) + (y >> 1) * fs.pitch[1] + (x >> 1) * 2;
      c[0] = yuv[1];
      c[1] = yuv[2];
    } else {
      const_cast<uint8_t*>(fs.plane[1])[(y >> 1) * fs.pitch[1] + (x >> 1)] = yuv[1];
      const_cast<uint8_t*>(fs.plane[2])[(y >> 1) * fs.pitch[2] + (x >> 1)] = yuv[2];
    }
  } else {
    constexpr int bpp = (F == SQDET_FMT_BGRA || F == SQDET_FMT_RGBA) ? 4 : 3;
    constexpr bool rgb = F == SQDET_FMT_RGB || F == SQDET_FMT_RGBA;
    uint8_t* q = p0 + y * fs.pitch[0] + x * bpp;
    q[rgb ? 2 : 0] = bgr[0];
    q[1] = bgr[1];
    q[rgb ? 0 : 2] = bgr[2];
  }
}

// cv2.clipLine(Size2l(w, h), p1, p2): Cohen-Sutherland with double-precision intercepts, each
// truncated toward zero and added to the endpoint being moved.
__device__ bool clip_line(int64_t w, int64_t h, int64_t& x1, int64_t& y1, int64_t& x2, int64_t& y2) {
  const int64_t right = w - 1, bottom = h - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  auto icept = [](int64_t a, int64_t b, int64_t c) {   // (int64)((double)a * b / c)
    return __double2ll_rz(__ddiv_rn(__dmul_rn((double)a, (double)b), (double)c));
  };
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    if (c1 & 12) {
      const int64_t a = c1 < 8 ? 0 : bottom;
      x1 += icept(a - y1, x2 - x1, y2 - y1);
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      const int64_t a = c2 < 8 ? 0 : bottom;
      x2 += icept(a - y2, x2 - x1, y2 - y1);
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        const int64_t a = c1 == 1 ? 0 : right;
        y1 += icept(a - x1, y2 - y1, x2 - x1);
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        const int64_t a = c2 == 1 ? 0 : right;
        y2 += icept(a - x2, y2 - y1, x2 - x1);
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// cv2.line(canvas, (x1, y1), (x2, y2), c, 1, LINE_8) on the w x h canvas: clipLine when an
// endpoint is outside, then LineIterator's 8-connected walk from the left endpoint.
template <int F>
__device__ void draw_line(const FrameSource& fs, int x1i, int y1i, int x2i, int y2i,
                          const uint8_t* bgr, const uint8_t* yuv) {
  const int w = fs.w, h = fs.h;
  int64_t x1 = x1i, y1 = y1i, x2 = x2i, y2 = y2i;
  if ((unsigned)x1i >= (unsigned)w || (unsigned)x2i >= (unsigned)w || (unsigned)y1i >= (unsigned)h ||
      (unsigned)y2i >= (unsigned)h) {
    if (!clip_line(w, h, x1, y1, x2, y2)) return;
  }
  int dx = (int)(x2 - x1), dy = (int)(y2 - y1);
  int x = (int)x1, y = (int)y1;
  if (dx < 0) {
    dx = -dx;
    dy = -dy;
    x = (int)x2;
    y = (int)y2;
  }
  const int sy = dy < 0 ? -1 : 1;
  dy = dy < 0 ? -dy : dy;
  const bool vert = dy > dx;
  if (vert) {
    const int t = dx;
    dx = dy;
    dy = t;
  }
  int err = dx - 2 * dy;
  for (int i = 0; i <= dx; ++i) {
    if ((unsigned)x < (unsigned)w && (unsigned)y < (unsigned)h) put_pixel<F>(fs, x, y, bgr, yuv);
    const bool step = err < 0;
    err += -2 * dy + (step ? 2 * dx : 0);
    if (vert) {
      y += sy;
      x += step;
    } else {
      x += 1;
      y += step ? sy : 0;
    }
  }
}

// '%.2f' of a float32 prob in [0, 1]: the exact value m / 2^k times 100, rounded half to even.
// Writes the digits (and '-' for -0.0) at out; returns their count.
__device__ int prob_digits(float prob, char* out) {
  const uint32_t bits = __float_as_uint(prob);
  const int e = (bits >> 23) & 255;
  const uint64_t m = (bits & 0x7FFFFFu) | (e ? 0x800000u : 0u);
  const int k = 150 - (e > 1 ? e : 1);
  uint32_t q = 0;
  if (k < 32) {                       // otherwise prob * 100 < 2^31 / 2^32 rounds to 0
    const uint64_t num = m * 100u;
    q = (uint32_t)(num >> k);
    if (k > 0) {
      const uint64_t r = num & ((1ull << k) - 1), half = 1ull << (k - 1);
      q += (r > half || (r == half && (q & 1))) ? 1u : 0u;
    }
  }
  int n = 0;
  if (bits >> 31) out[n++] = '-';
  out[n++] = (char)('0' + q / 100);
  out[n++] = '.';
  out[n++] = (char)('0' + q / 10 % 10);
  out[n++] = (char)('0' + q % 10);
  return n;
}

// A corner of bbox_transform as draw_box's int(): the float32 value truncated toward zero, or
// false when it is not finite or at least 2^31 in magnitude.
__device__ __forceinline__ bool corner(float v, int* out) {
  if (!(fabsf(v) < 2147483648.0f)) return false;
  *out = __float2int_rz(v);
  return true;
}

template <int F>
__global__ void __launch_bounds__(kDrawThreads) draw_dets_kernel(const __grid_constant__ DrawParams p) {
  __shared__ short s_glyph[95][3];
  __shared__ signed char s_seg[SQDET_HERSHEY_SEGMENTS][4];
  __shared__ char s_text[kMaxLabel];
  __shared__ int s_first[kMaxLabel + 1];        // label char c's first segment; [len] = total
  __shared__ long long s_pen[kMaxLabel];        // its pen x, 16.16
  __shared__ int s_rec, s_len, s_box[4];
  const int tid = threadIdx.x;
  for (int i = tid; i < 95 * 3; i += kDrawThreads) (&s_glyph[0][0])[i] = (&kHersheyGlyphs[0][0])[i];
  for (int i = tid; i < SQDET_HERSHEY_SEGMENTS * 4; i += kDrawThreads)
    (&s_seg[0][0])[i] = (&kHersheySegments[0][0])[i];
  __syncthreads();                                // thread 0 reads s_glyph before the loop's barrier

  const FrameSource& fs = p.frames[blockIdx.x];
  const DrawStyle& st = p.style;
  const int frame = p.first + (int)blockIdx.x;
  const sqdet_det* recs = p.dets + (size_t)frame * p.max_dets;
  int count = p.counts[frame];
  count = count < p.max_dets ? count : p.max_dets;     // count < 0 (overflow) draws nothing
  const int64_t hs = st.hscale;
  for (int k = 0;;) {
    if (tid == 0) {
      int rec = -1;
      for (; k < count && rec < 0; ++k) {
        const sqdet_det d = recs[k];
        if (!(d.prob > st.thresh) || d.cls < 0 || d.cls >= st.classes) continue;
        // bbox_transform in float32 (w / 2 == w * 0.5 exactly), no contraction
        const float hw = __fmul_rn(d.w, 0.5f), hh = __fmul_rn(d.h, 0.5f);
        if (!corner(__fsub_rn(d.cx, hw), &s_box[0]) || !corner(__fsub_rn(d.cy, hh), &s_box[1]) ||
            !corner(__fadd_rn(d.cx, hw), &s_box[2]) || !corner(__fadd_rn(d.cy, hh), &s_box[3]))
          continue;
        rec = k;
        int len = 0;
        if (d.prob >= 0.f && d.prob <= 1.f) {        // no label outside [0, 1]
          for (int i = 0; i < st.name_len[d.cls]; ++i) s_text[len++] = st.name[d.cls][i];
          s_text[len++] = ':';
          s_text[len++] = ' ';
          s_text[len++] = '(';
          len += prob_digits(d.prob, s_text + len);
          s_text[len++] = ')';
        }
        long long pen = (long long)s_box[0] * 65536;
        int segs = 0;
        for (int c = 0; c < len; ++c) {
          const short* g = s_glyph[s_text[c] - 32];
          s_first[c] = segs;
          s_pen[c] = pen;
          segs += g[2];
          pen += g[0] * hs;
        }
        s_first[len] = segs;
        s_len = len;
      }
      s_rec = rec;
    }
    __syncthreads();
    const int rec = s_rec;
    if (rec < 0) break;
    const int cls = recs[rec].cls;
    const uint8_t* bgr = st.bgr[cls];
    const uint8_t* yuv = st.yuv[cls];
    const int x0 = s_box[0], y0 = s_box[1], x1 = s_box[2], y1 = s_box[3];
    // the rectangle: two horizontal and two vertical runs clipped to the canvas
    const int64_t W = fs.w, H = fs.h;
    auto run = [&](int64_t fixed, int64_t a, int64_t b, int64_t extent, int64_t across,
                   int64_t* lo) -> int64_t {
      if (fixed < 0 || fixed >= across) return 0;
      *lo = max(min(a, b), (int64_t)0);
      const int64_t hi = min(max(a, b), extent - 1);
      return hi >= *lo ? hi - *lo + 1 : 0;
    };
    int64_t lo[4];
    const int64_t n0 = run(y0, x0, x1, W, H, &lo[0]), n1 = run(x1, y0, y1, H, W, &lo[1]),
                  n2 = run(y1, x0, x1, W, H, &lo[2]), n3 = run(x0, y0, y1, H, W, &lo[3]);
    for (int64_t i = tid; i < n0 + n1 + n2 + n3; i += kDrawThreads) {
      if (i < n0) put_pixel<F>(fs, (int)(lo[0] + i), y0, bgr, yuv);
      else if (i < n0 + n1) put_pixel<F>(fs, x1, (int)(lo[1] + i - n0), bgr, yuv);
      else if (i < n0 + n1 + n2) put_pixel<F>(fs, (int)(lo[2] + i - n0 - n1), y1, bgr, yuv);
      else put_pixel<F>(fs, x0, (int)(lo[3] + i - n0 - n1 - n2), bgr, yuv);
    }
    // the label's stroke segments, from the text origin (xmin, ymax)
    const int len = s_len;
    const long long py = (long long)y1 * 65536;
    for (int s = tid; s < s_first[len]; s += kDrawThreads) {
      int c = 0;
      while (s_first[c + 1] <= s) ++c;
      const signed char* seg = s_seg[s_glyph[s_text[c] - 32][1] + (s - s_first[c])];
      const long long px = s_pen[c];
      auto pix = [](long long v) { return (int)((v + 0x8000) >> 16); };   // narrowed as cv2 does
      draw_line<F>(fs, pix(px + seg[0] * hs), pix(py + seg[1] * hs), pix(px + seg[2] * hs),
                   pix(py + seg[3] * hs), bgr, yuv);
    }
    k = rec + 1;
    __syncthreads();
  }
}

template <int F>
int launch_format(const FrameSource* frames, int n, const sqdet_det* dets, const int32_t* counts,
                  int max_dets, const DrawStyle& style, cudaStream_t stream) {
  for (int first = 0; first < n; first += kDrawFramesPerLaunch) {
    const int m = n - first < kDrawFramesPerLaunch ? n - first : kDrawFramesPerLaunch;
    DrawParams p;
    for (int i = 0; i < m; ++i) p.frames[i] = frames[first + i];
    p.style = style;
    p.dets = dets;
    p.counts = counts;
    p.max_dets = max_dets;
    p.first = first;
    draw_dets_kernel<F><<<(unsigned)m, kDrawThreads, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("draw_dets_kernel");
  }
  return SQDET_OK;
}

// Draws frame i's records dets[i * max_dets + k], k < min(counts[i], max_dets), on the crop of
// frames[i] (FrameSource: planes, pitches, canvas = the h x w crop at (x, y)), one CTA per frame,
// one launch per kDrawFramesPerLaunch frames.  The frames' checks are the caller's.
int launch_draw_dets(int format, const FrameSource* frames, int n, const sqdet_det* dets,
                     const int32_t* counts, int max_dets, const DrawStyle& style,
                     cudaStream_t stream) {
  return dispatch_format(format, [&](auto f) {
    return launch_format<decltype(f)::value>(frames, n, dets, counts, max_dets, style, stream);
  });
}

}  // namespace
}  // namespace sqdet

using namespace sqdet;

int sqdet_draw_dets(int n, int format, uint8_t* const* planes, const int64_t* pitches,
                    const int32_t* heights, const int32_t* widths, const int32_t* crops,
                    const sqdet_det* dets_dev, const int32_t* counts_dev, int max_dets,
                    const sqdet_draw_style* style, void* stream) {
  const std::string name = "sqdet_draw_dets";
  const PixFormat* pf = pix_format(format);
  if (!pf) return fail(SQDET_ERR_INVALID_ARG, name + ": unknown format");
  if (!planes || !heights || !widths || !dets_dev || !counts_dev || !style || !style->class_names ||
      !style->class_bgr)
    return fail(SQDET_ERR_INVALID_ARG, name + ": null argument");
  if (n < 1 || n > kMaxDrawFrames)
    return fail(SQDET_ERR_INVALID_ARG, name + ": n must be in [1, " + std::to_string(kMaxDrawFrames) + "]");
  if (max_dets < 1) return fail(SQDET_ERR_INVALID_ARG, name + ": max_dets must be at least 1");
  if (style->classes < 1 || style->classes > kDrawMaxClasses)
    return fail(SQDET_ERR_INVALID_ARG, name + ": classes must be in [1, " + std::to_string(kDrawMaxClasses) + "]");
  const float fs = style->font_scale;
  if (!(fs > 0.f && fs <= 1024.f))
    return fail(SQDET_ERR_INVALID_ARG, name + ": font_scale must be finite, positive and at most 1024");
  DrawStyle st = {};
  st.hscale = (int64_t)nearbyint((double)fs * 65536.0);   // cvRound: half to even
  st.thresh = style->plot_prob_thresh;
  st.classes = style->classes;
  for (int c = 0; c < st.classes; ++c) {
    const char* s = style->class_names[c];
    const size_t len = s ? strnlen(s, kDrawMaxName + 1) : kDrawMaxName + 1;
    bool printable = len <= (size_t)kDrawMaxName;
    for (size_t i = 0; printable && i < len; ++i) printable = s[i] >= 32 && s[i] <= 126;
    if (!printable)
      return fail(SQDET_ERR_INVALID_ARG, name + ": class name " + std::to_string(c) +
                                             " is not printable ASCII of at most " +
                                             std::to_string(kDrawMaxName) + " characters");
    memcpy(st.name[c], s, len);
    st.name_len[c] = (uint8_t)len;
    const int b = style->class_bgr[3 * c], g = style->class_bgr[3 * c + 1], r = style->class_bgr[3 * c + 2];
    st.bgr[c][0] = (uint8_t)b;
    st.bgr[c][1] = (uint8_t)g;
    st.bgr[c][2] = (uint8_t)r;
    // cv2.cvtColor(solid BGR patch, COLOR_BGR2YUV_I420): OpenCV's BT.601 coefficients, 20 bits
    const int half = 1 << 19;
    st.yuv[c][0] = (uint8_t)((269484 * r + 528482 * g + 102760 * b + (16 << 20) + half) >> 20);
    st.yuv[c][1] = (uint8_t)((-155188 * r - 305135 * g + 460324 * b + (128 << 20) + half) >> 20);
    st.yuv[c][2] = (uint8_t)((460324 * r - 385875 * g - 74448 * b + (128 << 20) + half) >> 20);
  }
  // the device the call runs on is the one frame 0's first plane lives on, whatever is current
  std::vector<FrameSource> fr;
  int device = kFrame0Device;
  const int rc = accept_frames(name, *pf, n, planes, pitches, heights, widths, crops, nullptr,
                               &device, fr);
  if (rc) return rc;
  if (!device_range_ok(dets_dev, (int64_t)n * max_dets * (int64_t)sizeof(sqdet_det), device) ||
      !device_range_ok(counts_dev, (int64_t)n * sizeof(int32_t), device))
    return fail(SQDET_ERR_INVALID_ARG,
                name + ": dets_dev or counts_dev is not inside one device allocation on frame 0's device");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select frame 0's device");
  return launch_draw_dets(format, fr.data(), n, dets_dev, counts_dev, max_dets, st,
                          (cudaStream_t)stream);
}
