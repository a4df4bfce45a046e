// Baseline JPEG encoding of uint8 frames in device memory (sqdet_encode_jpeg): frame i's crop,
// converted to BGR as its format's cv2.cvtColor code does, becomes the bytes
// cv2.imencode('.jpg', crop, [IMWRITE_JPEG_QUALITY, quality]) writes, bit for bit.  That is
// libjpeg-turbo's default integer pipeline: 16-bit fixed-point YCbCr, 4:2:0 with edge replication
// and the 1, 2 bias, jpeg_fdct_islow, quantization by 8 q, Annex K Huffman tables, no restart
// markers.  oracle/jpeg.py restates it in numpy.
//
// The entropy-coded segment is one bit stream per frame, made parallel by knowing where each block's
// codes start:
//   1. transform    one thread per 8x8 block fetches its samples straight from the frame's planes
//                   (frames.cuh), converts, downsamples, transforms and quantizes them, and
//                   writes the quantized coefficients (natural order) to the scratch
//   2. block_bits   the bit length of each block's codes: its DC difference (the previous block
//                   of its component is another thread's) and its AC codes; sums per chunk of
//                   kChunk blocks
//   3. scan         per frame, the exclusive scan of the chunk sums: each chunk's first bit
//   4. pack         each block scans its chunk for its own first bit and ORs its codes into the
//                   frame's zeroed bit buffer (32-bit atomicOr: neighbours share only edge
//                   words); the last block adds the 1-bit padding
//   5. count_ff     the 0xFF bytes per kStuffChunk bytes of the stream
//   6. scan         per frame, their exclusive scan
//   7. stuff        each chunk copies its bytes to the output with a 0x00 after every 0xFF, and
//                   the frame's first chunk writes the header (a host template with the frame's
//                   height and width), EOI and the length, or -1 when the file does not fit
// Frames run kJpegFramesPerLaunch at a time through these launches, reusing one scratch.
#include <algorithm>
#include <cstring>

#include "frames.cuh"
#include "scan.cuh"

namespace sqdet {
namespace {

constexpr int kChunk = 256;            // blocks per transform / pack CTA
constexpr int kStuffThreads = 256;
constexpr int kStuffBytes = 16;        // bytes per stuffing thread
constexpr int kStuffChunk = kStuffThreads * kStuffBytes;
constexpr int kScanThreads = 1024;
constexpr int kMaxBlockBits = 22 + 63 * 26;   // a chroma DC of category 11, 63 AC codes of 16 + 10 bits
constexpr int kHeaderBytes = 623;
constexpr int kSofSize = 163;         // the header's offset of SOF0's height (then its width)

// ---- Annex K tables ---------------------------------------------------------------------------
constexpr uint8_t kStdLumaQ[64] = {
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
    14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr uint8_t kStdChromaQ[64] = {
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
    24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
    99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
    99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
constexpr uint8_t kZigzag[64] = {        // natural index of zigzag position k
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5,
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
constexpr uint8_t kDcLumaBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
constexpr uint8_t kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
constexpr uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
constexpr uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
constexpr uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
constexpr uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5,
    0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
    0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa};
constexpr uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
    0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0,
    0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26,
    0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5,
    0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
    0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa};

// The canonical codes of the four tables: code and length by symbol (length 0: not in the table).
struct HuffCodes {
  uint16_t dc_code[2][12];
  uint8_t dc_len[2][12];
  uint16_t ac_code[2][256];
  uint8_t ac_len[2][256];
};
constexpr void canonical(const uint8_t* bits, const uint8_t* vals, uint16_t* code, uint8_t* len) {
  int c = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    for (int i = 0; i < bits[l - 1]; ++i, ++k, ++c) {
      code[vals[k]] = (uint16_t)c;
      len[vals[k]] = (uint8_t)l;
    }
    c <<= 1;
  }
}
constexpr HuffCodes huff_codes() {
  HuffCodes h{};
  canonical(kDcLumaBits, kDcVals, h.dc_code[0], h.dc_len[0]);
  canonical(kDcChromaBits, kDcVals, h.dc_code[1], h.dc_len[1]);
  canonical(kAcLumaBits, kAcLumaVals, h.ac_code[0], h.ac_len[0]);
  canonical(kAcChromaBits, kAcChromaVals, h.ac_code[1], h.ac_len[1]);
  return h;
}
__constant__ HuffCodes kHuff = huff_codes();
__constant__ uint8_t kZigzagDev[64] = {     // kZigzag, for device code
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5,
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ---- per-frame geometry and scratch ---------------------------------------------------------------
// One frame of a launch group: its crop, MCU grid and where its pieces of the scratch and output
// are.  Blocks are numbered in stream order (per MCU: Y0 Y1 Y2 Y3 Cb Cr) from blk (a multiple of
// kChunk); the chunk sums of its `chunks` block chunks start at csum and those of its `schunks`
// stuffing chunks at ssum, each followed by one slot that the scan fills with the total.
struct JpegGeom {
  int h, w, mcu_cols, blocks;           // blocks = 6 * MCUs
  int chunks, schunks;
  int64_t blk, csum, ssum, words;       // words: the first 32-bit word of the bit buffer
  uint8_t* out;
  int64_t* length;
};
constexpr int kJpegFramesPerLaunch = 16;
constexpr int kMaxJpegFrames = 128;     // frames per sqdet_encode_jpeg call
// libjpeg-turbo's JPEG_MAX_DIMENSION: cv2.imencode refuses a longer side, and libjpeg does not
// read a file whose SOF0 says one (its 16-bit fields would hold up to 65535)
constexpr int kJpegMaxSide = 65500;

struct JpegParams {
  JpegGeom g[kJpegFramesPerLaunch];
  int16_t* coef;                        // [blocks][64], natural order
  uint32_t* bits;                       // [blocks]
  int64_t* sums;                        // chunk sums of blocks and of stuffing chunks
  uint32_t* stream;                     // bit buffers
  int64_t cap;
};

// The reciprocal of each divisor 8 q (luma, chroma; natural order) as libjpeg-turbo builds it for
// 16-bit coefficients (compute_reciprocal): |x| / (8 q) rounded is (|x| + corr) * recip >> shift.
struct QuantRecip {
  uint16_t recip[2][64], corr[2][64];
  uint8_t shift[2][64];
};

template <int F>
struct TransformParams {
  JpegParams p;
  FrameDesc<kPlanes<F>> f[kJpegFramesPerLaunch];
  QuantRecip quant;
};
static_assert(sizeof(TransformParams<SQDET_FMT_I420>) <= 4096, "transform parameters exceed 4 KiB");

struct StuffParams {
  JpegParams p;
  uint8_t header[kHeaderBytes];
};
static_assert(sizeof(StuffParams) <= 4096, "stuffing parameters exceed 4 KiB");

__device__ __forceinline__ int nbits(int v) { return v ? 32 - __clz(abs(v)) : 0; }

// Is block u (0..3 luma, 4, 5 chroma) of MCU m a luma block right of or below the image's blocks?
__device__ __forceinline__ bool dummy_block(const JpegGeom& g, int m, int u) {
  if (u >= 4) return false;
  const int bx = (m % g.mcu_cols) * 2 + (u & 1), by = (m / g.mcu_cols) * 2 + (u >> 1);
  return bx * 8 >= g.w || by * 8 >= g.h;
}

// The quantized DC that block b codes against: the previous block of its component in stream order,
// a dummy block standing for the last real block before it (its DC is that block's), 0 at the start.
__device__ int prev_dc(const JpegGeom& g, const int16_t* coef, int b) {
  const int u = b % 6;
  if (u >= 4) return b >= 6 ? coef[(int64_t)(b - 6) * 64] : 0;
  for (int k = b - 1; k >= 0; --k) {
    const int uk = k % 6;
    if (uk >= 4) continue;
    if (!dummy_block(g, k / 6, uk)) return coef[(int64_t)k * 64];
  }
  return 0;
}

// ---- 1. transform -------------------------------------------------------------------------------
// jpeg_fdct_islow on one row or column of 8 (in place): pass 1 scales by 2^PASS1_BITS, pass 2
// removes it.
template <bool kFirst>
__device__ __forceinline__ void fdct8(int* d, int stride) {
  constexpr int CB = 13, PB = 2, SH = kFirst ? CB - PB : CB + PB;
  auto desc = [](int x, int n) { return (x + (1 << (n - 1))) >> n; };
  const int t0 = d[0] + d[7 * stride], t7 = d[0] - d[7 * stride];
  const int t1 = d[stride] + d[6 * stride], t6 = d[stride] - d[6 * stride];
  const int t2 = d[2 * stride] + d[5 * stride], t5 = d[2 * stride] - d[5 * stride];
  const int t3 = d[3 * stride] + d[4 * stride], t4 = d[3 * stride] - d[4 * stride];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  d[0] = kFirst ? (t10 + t11) * (1 << PB) : desc(t10 + t11, PB);
  d[4 * stride] = kFirst ? (t10 - t11) * (1 << PB) : desc(t10 - t11, PB);
  const int z1 = (t12 + t13) * 4433;
  d[2 * stride] = desc(z1 + t13 * 6270, SH);
  d[6 * stride] = desc(z1 - t12 * 15137, SH);
  const int z5 = (t4 + t6 + t5 + t7) * 9633;
  const int a1 = (t4 + t7) * -7373, a2 = (t5 + t6) * -20995;
  const int a3 = (t4 + t6) * -16069 + z5, a4 = (t5 + t7) * -3196 + z5;
  d[7 * stride] = desc(t4 * 2446 + a1 + a3, SH);
  d[5 * stride] = desc(t5 * 16819 + a2 + a4, SH);
  d[3 * stride] = desc(t6 * 25172 + a2 + a3, SH);
  d[stride] = desc(t7 * 12299 + a1 + a4, SH);
}

// rgb_ycc_convert: 16 fraction bits, Cb and Cr rounded with ONE_HALF - 1.
__device__ __forceinline__ int to_y(int b, int g, int r) {
  return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
}
__device__ __forceinline__ int to_c(int b, int g, int r, bool cr) {
  return cr ? (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16
            : (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
}

template <int F>
__global__ void __launch_bounds__(kChunk) transform_kernel(const __grid_constant__ TransformParams<F> tp) {
  const JpegGeom& g = tp.p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  const int b = blockIdx.x * kChunk + threadIdx.x;
  const int64_t gb = g.blk + b;
  int blk[64];
  const int m = b / 6, u = b % 6;
  const bool real = b < g.blocks && !dummy_block(g, m, u);
  if (b >= g.blocks) return;
  const auto taps_ = taps<F>(tp.f[blockIdx.y]);
  const int mx = m % g.mcu_cols, my = m / g.mcu_cols;
  if (!real) {
#pragma unroll
    for (int i = 0; i < 64; ++i) blk[i] = 0;
  } else if (u < 4) {
    // luma: rows and columns past the crop repeat its last ones
    const int y0 = my * 16 + (u >> 1) * 8, x0 = mx * 16 + (u & 1) * 8;
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        int B, G, R;
        fetch_bgr(taps_, min(y0 + r, g.h - 1), min(x0 + c, g.w - 1), B, G, R);
        blk[r * 8 + c] = to_y(B, G, R) - 128;
      }
  } else {
    // chroma: h2v2 of the full-size plane (last row repeated to a 2-row group, last column to the
    // block's width), then the last downsampled row repeated to the MCU row
    const bool cr = u == 5;
    const int last_row = (g.h + 1) / 2 - 1;
#pragma unroll 1
    for (int r = 0; r < 8; ++r) {
      const int dr = min(my * 8 + r, last_row);
      const int ya = min(2 * dr, g.h - 1), yb = min(2 * dr + 1, g.h - 1);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int xa = min(mx * 16 + 2 * c, g.w - 1), xb = min(mx * 16 + 2 * c + 1, g.w - 1);
        int s = 0, B, G, R;
        fetch_bgr(taps_, ya, xa, B, G, R); s += to_c(B, G, R, cr);
        fetch_bgr(taps_, ya, xb, B, G, R); s += to_c(B, G, R, cr);
        fetch_bgr(taps_, yb, xa, B, G, R); s += to_c(B, G, R, cr);
        fetch_bgr(taps_, yb, xb, B, G, R); s += to_c(B, G, R, cr);
        blk[r * 8 + c] = ((s + 1 + (c & 1)) >> 2) - 128;
      }
    }
  }
  if (real) {
#pragma unroll
    for (int r = 0; r < 8; ++r) fdct8<true>(blk + 8 * r, 1);
#pragma unroll
    for (int c = 0; c < 8; ++c) fdct8<false>(blk + c, 8);
  }
  // quantize: libjpeg-turbo's reciprocal multiply by 1 / (8 q), sign restored
  const int t = u >= 4;
  int16_t z[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int x = blk[i];
    const uint32_t a = ((uint32_t)abs(x) + tp.quant.corr[t][i]) * tp.quant.recip[t][i] >> tp.quant.shift[t][i];
    z[i] = (int16_t)(x < 0 ? -(int)a : (int)a);
  }
  int4* o4 = reinterpret_cast<int4*>(tp.p.coef + gb * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) o4[i] = reinterpret_cast<const int4*>(z)[i];
}

// ---- 2. code lengths and chunk sums -------------------------------------------------------------
// The bits of block b's codes: its DC difference (the block before it of its component is another
// thread's), then its AC run/size codes with ZRLs and EOB.
__device__ int block_bits(const JpegGeom& g, const int16_t* coef, int b) {
  const int u = b % 6, t = u >= 4;
  const int16_t* z = coef + (int64_t)b * 64;
  const int diff = dummy_block(g, b / 6, u) ? 0 : z[0] - prev_dc(g, coef, b);
  int bits = kHuff.dc_len[t][nbits(diff)] + nbits(diff), run = 0;
#pragma unroll 4
  for (int k = 1; k < 64; ++k) {
    const int v = z[kZigzagDev[k]];
    if (v == 0) {
      ++run;
    } else {
      const int nb = nbits(v);
      bits += (run >> 4) * kHuff.ac_len[t][0xF0] + kHuff.ac_len[t][((run & 15) << 4) | nb] + nb;
      run = 0;
    }
  }
  return bits + (run ? kHuff.ac_len[t][0] : 0);
}

__global__ void __launch_bounds__(kChunk) block_bits_kernel(const __grid_constant__ JpegParams p) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  const int b = blockIdx.x * kChunk + threadIdx.x;
  const int bits = b < g.blocks ? block_bits(g, p.coef + g.blk * 64, b) : 0;
  p.bits[g.blk + b] = (uint32_t)bits;
  int64_t total;
  block_exclusive_scan(bits, warp, &total);
  if (threadIdx.x == 0) p.sums[g.csum + blockIdx.x] = total;
}

// ---- 3, 6. per-frame exclusive scans of chunk sums ------------------------------------------------
// Frame blockIdx.x's `count` chunk sums from sums[first] become their exclusive scan, and the slot
// after them the total.
__global__ void __launch_bounds__(kScanThreads) scan_kernel(const __grid_constant__ JpegParams p,
                                                            int stuffing) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.x];
  int64_t* s = p.sums + (stuffing ? g.ssum : g.csum);
  const int count = stuffing ? g.schunks : g.chunks;
  int64_t carry = 0;
  for (int base = 0; base < count; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const int64_t v = i < count ? s[i] : 0;
    int64_t total;
    const int64_t ex = block_exclusive_scan(v, warp, &total);
    if (i < count) s[i] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) s[count] = carry;
}

// ---- 4. pack ------------------------------------------------------------------------------------
// Bits MSB first into 32-bit words (word j's most significant bit is stream bit 32 j), ORed in.
struct BitWriter {
  uint32_t* word;
  uint64_t acc;
  int n;                                // pending bits in acc, including the leading offset
  __device__ void put(uint32_t v, int len) {
    acc = (acc << len) | v;
    n += len;
    if (n >= 32) {
      atomicOr(word++, (uint32_t)(acc >> (n - 32)));
      n -= 32;
    }
  }
  __device__ void flush() {
    if (n > 0) atomicOr(word, (uint32_t)(acc << (32 - n)));
  }
};

__global__ void __launch_bounds__(kChunk) pack_kernel(const __grid_constant__ JpegParams p) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  const int b = blockIdx.x * kChunk + threadIdx.x;
  const int64_t gb = g.blk + b;
  const int64_t bits = b < g.blocks ? p.bits[gb] : 0;
  int64_t total;
  const int64_t pos = p.sums[g.csum + blockIdx.x] + block_exclusive_scan(bits, warp, &total);
  if (b >= g.blocks) return;
  const int u = b % 6, t = u >= 4;
  BitWriter w{p.stream + g.words + (pos >> 5), 0, (int)(pos & 31)};
  const bool dummy = dummy_block(g, b / 6, u);
  const int16_t* z = p.coef + gb * 64;
  const int diff = dummy ? 0 : z[0] - prev_dc(g, p.coef + g.blk * 64, b);
  const int dn = nbits(diff);
  w.put(kHuff.dc_code[t][dn], kHuff.dc_len[t][dn]);
  if (dn) w.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << dn) - 1), dn);
  int run = 0;
#pragma unroll 1
  for (int k = 1; k < 64; ++k) {
    const int v = z[kZigzagDev[k]];
    if (v == 0) {
      ++run;
      continue;
    }
    for (; run > 15; run -= 16) w.put(kHuff.ac_code[t][0xF0], kHuff.ac_len[t][0xF0]);
    const int nb = nbits(v), sym = (run << 4) | nb;
    w.put(kHuff.ac_code[t][sym], kHuff.ac_len[t][sym]);
    w.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << nb) - 1), nb);
    run = 0;
  }
  if (run) w.put(kHuff.ac_code[t][0], kHuff.ac_len[t][0]);
  if (b == g.blocks - 1) {                  // 1-bits to the byte boundary
    const int pad = (int)(-p.sums[g.csum + g.chunks] & 7);
    if (pad) w.put((1u << pad) - 1, pad);
  }
  w.flush();
}

// ---- 5. 0xFF counts -----------------------------------------------------------------------------
__device__ __forceinline__ uint8_t stream_byte(const uint32_t* words, int64_t j) {
  return (uint8_t)(words[j >> 2] >> (24 - 8 * (j & 3)));
}

__global__ void __launch_bounds__(kStuffThreads) count_ff_kernel(const __grid_constant__ JpegParams p) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.schunks) return;
  const int64_t bytes = (p.sums[g.csum + g.chunks] + 7) >> 3;
  const int64_t first = (int64_t)blockIdx.x * kStuffChunk + threadIdx.x * kStuffBytes;
  const uint32_t* words = p.stream + g.words;
  int ff = 0;
  for (int i = 0; i < kStuffBytes && first + i < bytes; ++i) ff += stream_byte(words, first + i) == 0xFF;
  int64_t total;
  block_exclusive_scan(ff, warp, &total);
  if (threadIdx.x == 0) p.sums[g.ssum + blockIdx.x] = total;
}

// ---- 7. stuff, header, EOI, length --------------------------------------------------------------
__global__ void __launch_bounds__(kStuffThreads) stuff_kernel(const __grid_constant__ StuffParams sp) {
  __shared__ int64_t warp[32];
  const JpegParams& p = sp.p;
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.schunks) return;
  const int64_t bytes = (p.sums[g.csum + g.chunks] + 7) >> 3;
  const int64_t size = kHeaderBytes + bytes + p.sums[g.ssum + g.schunks] + 2;
  if (blockIdx.x == 0 && threadIdx.x == 0) *g.length = size <= p.cap ? size : -1;
  if (size > p.cap) return;
  const int64_t first = (int64_t)blockIdx.x * kStuffChunk + threadIdx.x * kStuffBytes;
  const uint32_t* words = p.stream + g.words;
  uint8_t v[kStuffBytes];
  int ff = 0;
#pragma unroll
  for (int i = 0; i < kStuffBytes; ++i) {
    v[i] = first + i < bytes ? stream_byte(words, first + i) : 0;
    ff += first + i < bytes && v[i] == 0xFF;
  }
  int64_t total;
  int64_t o = kHeaderBytes + first + p.sums[g.ssum + blockIdx.x] + block_exclusive_scan(ff, warp, &total);
  for (int i = 0; i < kStuffBytes && first + i < bytes; ++i) {
    g.out[o++] = v[i];
    if (v[i] == 0xFF) g.out[o++] = 0;
  }
  if (blockIdx.x == 0) {
    // the template with SOF0's height and width (bytes kSofSize.. of jpeg_header) filled in
    const int hw[4] = {g.h >> 8, g.h & 255, g.w >> 8, g.w & 255};
    for (int i = threadIdx.x; i < kHeaderBytes; i += kStuffThreads)
      g.out[i] = i >= kSofSize && i < kSofSize + 4 ? (uint8_t)hw[i - kSofSize] : sp.header[i];
    if (threadIdx.x == 0) {
      g.out[size - 2] = 0xFF;
      g.out[size - 1] = 0xD9;
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------
// The header of `quality` with height and width 0: SOI, JFIF APP0, DQT x 2, SOF0, DHT x 4, SOS.
void jpeg_header(const uint16_t (&q)[2][64], uint8_t* out) {
  int n = 0;
  auto put = [&](std::initializer_list<int> bytes) { for (int b : bytes) out[n++] = (uint8_t)b; };
  auto seg = [&](int marker, int len) { put({0xFF, marker, (len + 2) >> 8, (len + 2) & 255}); };
  put({0xFF, 0xD8});
  seg(0xE0, 14);
  put({'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0});
  for (int t = 0; t < 2; ++t) {
    seg(0xDB, 65);
    put({t});
    for (int k = 0; k < 64; ++k) out[n++] = (uint8_t)q[t][kZigzag[k]];
  }
  seg(0xC0, 15);                          // height and width at kSofSize, filled in per frame
  put({8, 0, 0, 0, 0, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1});
  const uint8_t* bits[4] = {kDcLumaBits, kAcLumaBits, kDcChromaBits, kAcChromaBits};
  const uint8_t* vals[4] = {kDcVals, kAcLumaVals, kDcVals, kAcChromaVals};
  const int ids[4] = {0x00, 0x10, 0x01, 0x11};
  for (int t = 0; t < 4; ++t) {
    int count = 0;
    for (int l = 0; l < 16; ++l) count += bits[t][l];
    seg(0xC4, 17 + count);
    put({ids[t]});
    for (int l = 0; l < 16; ++l) out[n++] = bits[t][l];
    for (int k = 0; k < count; ++k) out[n++] = vals[t][k];
  }
  seg(0xDA, 10);
  put({3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});
}

// One frame's sizes in the scratch.
struct FrameSizes {
  int blocks, chunks, schunks;
  int64_t words;
};
FrameSizes frame_sizes(int h, int w) {
  FrameSizes s;
  s.blocks = ((h + 15) / 16) * ((w + 15) / 16) * 6;
  s.chunks = (s.blocks + kChunk - 1) / kChunk;
  const int64_t max_bytes = ((int64_t)s.blocks * kMaxBlockBits + 7) / 8;
  s.schunks = (int)((max_bytes + kStuffChunk - 1) / kStuffChunk);
  s.words = (max_bytes + 3) / 4 + 1;
  return s;
}

int64_t align256(int64_t v) { return (v + 255) & ~(int64_t)255; }

// The scratch of the frames [first, first + count): coefficients, bit lengths, chunk sums, bit
// buffers, in that order.
struct GroupLayout {
  int64_t coef, bits, sums, stream, total;
};
GroupLayout group_layout(const FrameSource* fr, int first, int count, JpegGeom* g) {
  int64_t blocks = 0, sums = 0, words = 0;
  for (int i = 0; i < count; ++i) {
    const FrameSource& s = fr[first + i];
    const FrameSizes z = frame_sizes(s.h, s.w);
    if (g) {
      g[i].h = s.h;
      g[i].w = s.w;
      g[i].mcu_cols = (s.w + 15) / 16;
      g[i].blocks = z.blocks;
      g[i].chunks = z.chunks;
      g[i].schunks = z.schunks;
      g[i].blk = blocks;
      g[i].csum = sums;
      g[i].ssum = sums + z.chunks + 1;
      g[i].words = words;
    }
    blocks += (int64_t)z.chunks * kChunk;
    sums += z.chunks + 1 + z.schunks + 1;
    words += z.words;
  }
  GroupLayout L;
  L.coef = 0;
  L.bits = L.coef + align256(blocks * 64 * 2);
  L.sums = L.bits + align256(blocks * 4);
  L.stream = L.sums + align256(sums * 8);
  L.total = L.stream + align256(words * 4);
  return L;
}

template <int F>
int launch_group(const PixFormat& pf, const FrameSource* fr, int first, int count,
                 const QuantRecip& quant, const uint8_t* header, uint8_t* out, int64_t cap,
                 int64_t* lengths, uint8_t* scratch, cudaStream_t stream) {
  TransformParams<F> tp;
  JpegParams& p = tp.p;
  const GroupLayout L = group_layout(fr, first, count, p.g);
  int max_chunks = 0, max_schunks = 0;
  for (int i = 0; i < count; ++i) {
    p.g[i].out = out + (int64_t)(first + i) * cap;
    p.g[i].length = lengths + first + i;
    tp.f[i] = frame_desc<kPlanes<F>>(pf, fr[first + i], fr[first + i].h, fr[first + i].w);
    max_chunks = std::max(max_chunks, p.g[i].chunks);
    max_schunks = std::max(max_schunks, p.g[i].schunks);
  }
  p.coef = reinterpret_cast<int16_t*>(scratch + L.coef);
  p.bits = reinterpret_cast<uint32_t*>(scratch + L.bits);
  p.sums = reinterpret_cast<int64_t*>(scratch + L.sums);
  p.stream = reinterpret_cast<uint32_t*>(scratch + L.stream);
  p.cap = cap;
  tp.quant = quant;
  SQ_CUDA(cudaMemsetAsync(p.stream, 0, (size_t)(L.total - L.stream), stream));
  const dim3 grid((unsigned)max_chunks, (unsigned)count), sgrid((unsigned)max_schunks, (unsigned)count);
  transform_kernel<F><<<grid, kChunk, 0, stream>>>(tp);
  SQ_CHECK_LAUNCH("jpeg transform_kernel");
  block_bits_kernel<<<grid, kChunk, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg block_bits_kernel");
  scan_kernel<<<(unsigned)count, kScanThreads, 0, stream>>>(p, 0);
  SQ_CHECK_LAUNCH("jpeg scan_kernel");
  pack_kernel<<<grid, kChunk, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg pack_kernel");
  count_ff_kernel<<<sgrid, kStuffThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg count_ff_kernel");
  scan_kernel<<<(unsigned)count, kScanThreads, 0, stream>>>(p, 1);
  SQ_CHECK_LAUNCH("jpeg scan_kernel");
  StuffParams sp;
  sp.p = p;
  memcpy(sp.header, header, kHeaderBytes);
  stuff_kernel<<<sgrid, kStuffThreads, 0, stream>>>(sp);
  SQ_CHECK_LAUNCH("jpeg stuff_kernel");
  return SQDET_OK;
}

// The largest file of an h x w crop.
int64_t jpeg_max_bytes(int h, int w) {
  const FrameSizes s = frame_sizes(h, w);
  return kHeaderBytes + 2 * (((int64_t)s.blocks * kMaxBlockBits + 7) / 8) + 2;
}

// The scratch the encode of the crops of `frames` needs.
int64_t jpeg_scratch_bytes(const FrameSource* frames, int n) {
  int64_t most = 0;
  for (int first = 0; first < n; first += kJpegFramesPerLaunch)
    most = std::max(most, group_layout(frames, first, std::min(kJpegFramesPerLaunch, n - first), nullptr).total);
  return most;
}

// The encode of the crops of `frames` (the frames' checks are the caller's).
int launch_encode_jpeg(int format, const FrameSource* frames, int n, int quality, uint8_t* out,
                       int64_t cap, int64_t* lengths, void* scratch, cudaStream_t stream) {
  const PixFormat* pf = pix_format(format);
  if (!pf) return fail(SQDET_ERR_INVALID_ARG, "sqdet_encode_jpeg: unknown format");
  // jpeg_quality_scaling, then the standard tables scaled, rounded and clamped to 1..255
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  uint16_t q[2][64];
  QuantRecip quant;
  for (int i = 0; i < 64; ++i) {
    const uint8_t base[2] = {kStdLumaQ[i], kStdChromaQ[i]};
    for (int t = 0; t < 2; ++t) {
      const int v = std::min(std::max((base[t] * scale + 50) / 100, 1), 255);
      q[t][i] = (uint16_t)v;
      // compute_reciprocal of d = 8 v >= 8: r = 16 + floor(log2 d); a power of two drops a bit
      const uint32_t d = 8u * v;
      int r = 16 + (31 - __builtin_clz(d));
      uint32_t fq = (1u << r) / d;
      const uint32_t fr = (1u << r) % d;
      uint32_t c = d / 2;
      if (fr == 0) {
        fq >>= 1;
        --r;
      } else if (fr <= d / 2) {
        ++c;
      } else {
        ++fq;
      }
      quant.recip[t][i] = (uint16_t)fq;
      quant.corr[t][i] = (uint16_t)c;
      quant.shift[t][i] = (uint8_t)r;
    }
  }
  uint8_t header[kHeaderBytes];
  jpeg_header(q, header);
  uint8_t* s = static_cast<uint8_t*>(scratch);
  for (int first = 0; first < n; first += kJpegFramesPerLaunch) {
    const int count = std::min(kJpegFramesPerLaunch, n - first);
    int rc;
    switch (format) {
#define SQ_JPEG_CASE(F) \
  case F: rc = launch_group<F>(*pf, frames, first, count, quant, header, out, cap, lengths, s, stream); break;
      SQ_JPEG_CASE(SQDET_FMT_BGR)
      SQ_JPEG_CASE(SQDET_FMT_RGB)
      SQ_JPEG_CASE(SQDET_FMT_BGRA)
      SQ_JPEG_CASE(SQDET_FMT_RGBA)
      SQ_JPEG_CASE(SQDET_FMT_RGB_PLANAR)
      SQ_JPEG_CASE(SQDET_FMT_NV12)
      default: rc = launch_group<SQDET_FMT_I420>(*pf, frames, first, count, quant, header, out, cap, lengths, s, stream);
#undef SQ_JPEG_CASE
    }
    if (rc) return rc;
  }
  return SQDET_OK;
}

}  // namespace
}  // namespace sqdet

using namespace sqdet;

int64_t sqdet_jpeg_max_bytes(int h, int w) {
  if (h < 1 || w < 1 || h > kJpegMaxSide || w > kJpegMaxSide) {
    fail(SQDET_ERR_INVALID_ARG, "sqdet_jpeg_max_bytes: h and w must be in [1, 65500]");
    return -1;
  }
  return jpeg_max_bytes(h, w);
}

int64_t sqdet_jpeg_scratch_bytes(int n, const int32_t* heights, const int32_t* widths,
                                 const int32_t* crops) {
  std::vector<FrameSource> fr;
  if (encode_crops("sqdet_jpeg_scratch_bytes", "JPEG", kMaxJpegFrames, kJpegMaxSide, n, heights, widths, crops, fr))
    return -1;
  return jpeg_scratch_bytes(fr.data(), n);
}

int sqdet_encode_jpeg(int n, int format, const uint8_t* const* planes, const int64_t* pitches,
                      const int32_t* heights, const int32_t* widths, const int32_t* crops,
                      int quality, uint8_t* out_dev, int64_t cap, int64_t* lengths_dev,
                      void* scratch_dev, int64_t scratch_bytes, void* stream) {
  const std::string name = "sqdet_encode_jpeg";
  const PixFormat* pf = pix_format(format);
  if (!pf) return fail(SQDET_ERR_INVALID_ARG, name + ": unknown format");
  if (!planes || !heights || !widths || !out_dev || !lengths_dev || !scratch_dev)
    return fail(SQDET_ERR_INVALID_ARG, name + ": null argument");
  std::vector<FrameSource> fr;
  int rc = encode_crops(name, "JPEG", kMaxJpegFrames, kJpegMaxSide, n, heights, widths, crops, fr);
  if (rc) return rc;
  if (quality < 1 || quality > 100) return fail(SQDET_ERR_INVALID_ARG, name + ": quality must be in [1, 100]");
  if (cap < 1) return fail(SQDET_ERR_INVALID_ARG, name + ": cap must be at least 1");
  // the scratch holds int4, int64 and 32-bit atomic regions at 256-byte offsets from its start
  if ((uintptr_t)scratch_dev % 256)
    return fail(SQDET_ERR_INVALID_ARG, name + ": scratch_dev must be 256-byte aligned");
  if ((uintptr_t)lengths_dev % alignof(int64_t))
    return fail(SQDET_ERR_INVALID_ARG, name + ": lengths_dev must be 8-byte aligned");
  if (scratch_bytes < jpeg_scratch_bytes(fr.data(), n))
    return fail(SQDET_ERR_INVALID_ARG, name + ": scratch_bytes is below sqdet_jpeg_scratch_bytes");
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
  return launch_encode_jpeg(format, fr.data(), n, quality, out_dev, cap, lengths_dev, scratch_dev,
                            (cudaStream_t)stream);
}
