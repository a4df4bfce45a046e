// Baseline JPEG encoding of uint8 frames in device memory (sqdet_encode_jpeg_params): frame i's
// crop, converted to BGR as its format's cv2.cvtColor code does, becomes the bytes
// cv2.imencode('.jpg', crop, params) writes, bit for bit, for cv2's IMWRITE_JPEG_QUALITY,
// _LUMA_QUALITY, _CHROMA_QUALITY, _SAMPLING_FACTOR, _OPTIMIZE and _RST_INTERVAL.  That is
// libjpeg-turbo's integer pipeline: 16-bit fixed-point YCbCr; luma sampled 4x1, 2x2, 2x1, 1x2 or
// 1x1 against 1x1 chroma, with edge replication and jcsample.c's downsampler of each; jpeg_fdct_islow;
// quantization by 8 q; Annex K Huffman tables or, with optimize, each frame's own
// jpeg_gen_optimal_table tables; restart markers every restart_interval MCUs.  oracle/jpeg.py
// restates the defaults in numpy and oracle/jpeg_params.py the rest.
//
// The entropy-coded segment is one bit stream per frame, made parallel by knowing where each block's
// codes start:
//   1. transform    one thread per 8x8 block fetches its samples straight from the frame's planes
//                   (frames.cuh), converts, downsamples, transforms and quantizes them, and
//                   writes the quantized coefficients (natural order) to the scratch; templated
//                   over the sampling
//   (optimize only)
//   1a. hist        the symbol counts of the four tables (DC, AC x luma, chroma), per chunk in
//                   shared memory, then added to the frame's 64-bit counts
//   1b. table       per frame, one warp per table builds jpeg_gen_optimal_table's code lengths and
//                   symbol order, and the canonical codes
//   2. block_bits   the bit length of each block's codes: its DC difference (the previous block
//                   of its component is another thread's) and its AC codes; sums per chunk of
//                   kChunk blocks
//   3. scan         per frame, the exclusive scan of the chunk sums: each chunk's first bit
//   (restart markers only)
//   3a. interval    each restart interval's first bit and its length in bytes (padded)
//   3b. scan        per frame, their exclusive scan: each interval's first byte
//   4. pack         each block scans its chunk for its own first bit and ORs its codes into the
//                   frame's zeroed bit buffer (32-bit atomicOr: neighbours share only edge
//                   words); the last block of each interval adds the 1-bit padding
//   5. count_ff     the 0xFF bytes (and 2 per RSTn marker) per kStuffChunk bytes of the stream
//   6. scan         per frame, their exclusive scan
//   7. stuff        each chunk copies its bytes to the output with a 0x00 after every 0xFF and
//                   RSTn before each interval's first byte, and the frame's first chunk writes
//                   the header (a host template with the frame's height, width and Huffman
//                   tables filled in), EOI and the length, or -1 when the file does not fit
// Frames run kEncodeFramesPerLaunch at a time through these launches, reusing one scratch.
// Progressive files (sqdet_encode_jpeg_progressive) reuse the transform and then code the ten scans
// of jpeg_simple_progression in launches P1-P7 below, every launch covering all scans of all frames
// of the group; oracle/jpeg_progressive.py restates them.
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
// a chroma DC of category 11 (Annex K: an 11-bit code; optimized: up to 16 bits), 63 AC codes of
// 16 + 10 bits
constexpr int kMaxBlockBits = 22 + 63 * 26;
constexpr int kMaxBlockBitsOpt = 27 + 63 * 26;
constexpr int kPrefixBytes = 177;     // SOI, JFIF APP0, DQT x 2, SOF0
constexpr int kSofSize = 163;         // the header's offset of SOF0's height (then its width)
constexpr int kSosBytes = 14, kDriBytes = 6;
constexpr int kHeaderBytes = 623;     // with the Annex K tables and no DRI; optimized tables are no longer
constexpr int kTableThreads = 128;    // one warp per table

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

// The tables as DHT writes them: bits[t][l] symbols of length l + 1 and the symbols in order, for
// t = DC luma, AC luma, DC chroma, AC chroma; count[t] symbols in all.
struct HuffSpec {
  uint8_t bits[4][16];
  uint8_t vals[4][256];
  int16_t count[4];
};
// A frame's optimized tables: its codes and its DHT contents.
struct FrameHuff {
  HuffCodes c;
  HuffSpec s;
};

// A progressive frame's tables, by slot: scan s's table in slot s (scan 0's the DC luma one), scan
// 0's DC chroma table in slot kChromaDcSlot; slot 6 (the DC refinement) stays empty.  The frame's
// tail and symbol-block chunk sums (see prog_units_kernel) start at JpegGeom::tsum.
constexpr int kScans = 10, kSlots = 11, kChromaDcSlot = 10;
struct ProgHuff {
  uint16_t code[kSlots][256];
  uint8_t len[kSlots][256];
  uint8_t bits[kSlots][16];
  uint8_t vals[kSlots][256];
  int16_t count[kSlots];
};

// ---- per-frame geometry and scratch ---------------------------------------------------------------
// One frame of a launch group: its crop, MCU grid and where its pieces of the scratch and output
// are.  Blocks are numbered in stream order (per MCU: the luma blocks row by row, then Cb, Cr)
// from blk (a multiple of kChunk); the chunk sums of its `chunks` block chunks start at csum,
// those of its `schunks` stuffing chunks at ssum and those of its `ints` restart intervals at isum
// (with restart markers only), each followed by one slot that the scan fills with the total.
struct JpegGeom {
  int h, w, mcu_cols, blocks;           // blocks = MCUs * blocks per MCU
  int chunks, schunks, ints;            // ints: restart intervals (1 without restart markers)
  int64_t blk, csum, ssum, isum, ipos;  // ipos: the first of its intervals' first bits
  int64_t words;                        // the first 32-bit word of the bit buffer
  int64_t cblk, tsum;                   // progressive: the first block in coef (blk counts units) and
                                        // the first tail chunk sum (the symbol-unit sums follow)
  uint8_t* out;
  int64_t* length;
};
// 128 frames per sqdet_encode_jpeg call; sides up to libjpeg-turbo's JPEG_MAX_DIMENSION:
// cv2.imencode refuses a longer side, and libjpeg does not read a file whose SOF0 says one (its
// 16-bit fields would hold up to 65535)
constexpr int kJpegMaxSide = 65500;
constexpr Encoder kJpeg = {"sqdet_encode_jpeg", "JPEG", "sqdet_jpeg_scratch_bytes", 128, kJpegMaxSide};
constexpr Encoder kJpegProg = {"sqdet_encode_jpeg_progressive", "JPEG", "sqdet_jpeg_scratch_bytes_progressive",
                               128, kJpegMaxSide};

struct JpegParams {
  JpegGeom g[kEncodeFramesPerLaunch];
  int16_t* coef;                        // [blocks][64], natural order
  uint32_t* bits;                       // [blocks]
  int64_t* sums;                        // chunk sums of blocks, of stuffing chunks and of intervals
  int64_t* ipos;                        // each interval's first bit, before padding
  uint32_t* stream;                     // bit buffers
  unsigned long long* freq;             // [frame][4][256] symbol counts (optimize)
  FrameHuff* huff;                      // [frame] (optimize)
  uint32_t *flags, *pre, *flush;        // [units] (progressive)
  ProgHuff* phuff;                      // [frame] (progressive)
  int64_t cap;
  int hs, vs, luma, per;                // luma sampling factors, luma blocks and blocks per MCU
  int rst;                              // MCUs per restart interval, 0 for none
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
  FrameDesc<kPlanes<F>> f[kEncodeFramesPerLaunch];
  QuantRecip quant;
};
static_assert(sizeof(TransformParams<SQDET_FMT_I420>) <= 4096, "transform parameters exceed 4 KiB");

struct StuffParams {
  JpegParams p;
  HuffSpec std;                         // the Annex K tables
  uint8_t prefix[kPrefixBytes];         // SOI .. SOF0, height and width 0
  uint8_t suffix[kDriBytes + kSosBytes];  // DRI (with restart markers), SOS
  int suffix_bytes;
  uint8_t sos[10][kSosBytes];           // progressive: each scan's SOS
};
static_assert(sizeof(StuffParams) <= 4096, "stuffing parameters exceed 4 KiB");

__device__ __forceinline__ int nbits(int v) { return v ? 32 - __clz(abs(v)) : 0; }

// Is block u (luma blocks 0 .. luma - 1 row by row, then Cb, Cr) of MCU m a luma block right of or
// below the image's blocks?
__device__ __forceinline__ bool dummy_block(const JpegParams& p, const JpegGeom& g, int m, int u) {
  if (u >= p.luma) return false;
  const int bx = (m % g.mcu_cols) * p.hs + u % p.hs, by = (m / g.mcu_cols) * p.vs + u / p.hs;
  return bx * 8 >= g.w || by * 8 >= g.h;
}

// The quantized DC that block b codes against: the previous block of its component in stream order,
// a dummy block standing for the last real block before it (its DC is that block's), 0 at the start
// of the frame and of each restart interval.
__device__ int prev_dc(const JpegParams& p, const JpegGeom& g, const int16_t* coef, int b) {
  const int m = b / p.per, u = b - m * p.per;
  const int first = p.rst ? (m - m % p.rst) * p.per : 0;     // the interval's first block
  if (u >= p.luma) return b - p.per >= first ? coef[(int64_t)(b - p.per) * 64] : 0;
  for (int k = b - 1; k >= first; --k) {
    const int uk = k % p.per;
    if (uk >= p.luma) continue;
    if (!dummy_block(p, g, k / p.per, uk)) return coef[(int64_t)k * 64];
  }
  return 0;
}

// The code tables block_bits and pack read: the Annex K ones, or the frame's optimized ones.
template <bool kOpt>
__device__ __forceinline__ const HuffCodes& huff_codes_of(const JpegParams& p, int frame) {
  if constexpr (kOpt) return p.huff[frame].c;
  else return kHuff;
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

// Luma HS x VS against 1x1 chroma: an MCU is 8 HS x 8 VS pixels.
template <int F, int HS, int VS>
__global__ void __launch_bounds__(kChunk) transform_kernel(const __grid_constant__ TransformParams<F> tp) {
  constexpr int kLuma = HS * VS, kPer = kLuma + 2;
  const JpegGeom& g = tp.p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  const int b = blockIdx.x * kChunk + threadIdx.x;
  const int64_t gb = g.blk + b;
  int blk[64];
  const int m = b / kPer, u = b % kPer;
  const bool real = b < g.blocks && !dummy_block(tp.p, g, m, u);
  if (b >= g.blocks) return;
  const auto taps_ = taps<F>(tp.f[blockIdx.y]);
  const int mx = m % g.mcu_cols, my = m / g.mcu_cols;
  if (!real) {
#pragma unroll
    for (int i = 0; i < 64; ++i) blk[i] = 0;
  } else if (u < kLuma) {
    // luma: rows and columns past the crop repeat its last ones
    const int y0 = my * 8 * VS + (u / HS) * 8, x0 = mx * 8 * HS + (u % HS) * 8;
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        int B, G, R;
        fetch_bgr(taps_, min(y0 + r, g.h - 1), min(x0 + c, g.w - 1), B, G, R);
        blk[r * 8 + c] = to_y(B, G, R) - 128;
      }
  } else {
    // chroma: the full-size plane with its last row repeated to a VS-row group and its last column
    // to the MCU's width, downsampled, then the last downsampled row repeated to the MCU row.
    // h2v2 rounds with the bias 1, 2, 1, 2, ..., h2v1 with 0, 1, 0, 1, ..., int_downsample (4x1,
    // 1x2) to nearest, halves up
    const bool cr = u == kLuma + 1;
    const int last_row = (g.h + VS - 1) / VS - 1;
#pragma unroll 1
    for (int r = 0; r < 8; ++r) {
      const int dr = min(my * 8 + r, last_row);
      if constexpr (HS == 2 && VS == 2) {
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
      } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          int s = 0;
#pragma unroll
          for (int i = 0; i < VS; ++i)
#pragma unroll(HS == 4 ? 1 : HS)          // 4x1: 32 fetches per row unrolled spill
            for (int j = 0; j < HS; ++j) {
              int B, G, R;
              fetch_bgr(taps_, min(VS * dr + i, g.h - 1), min(HS * (mx * 8 + c) + j, g.w - 1), B, G, R);
              s += to_c(B, G, R, cr);
            }
          if constexpr (HS == 2) s = (s + (c & 1)) >> 1;
          else if constexpr (kLuma == 4) s = (s + 2) >> 2;
          else if constexpr (kLuma == 2) s = (s + 1) >> 1;
          blk[r * 8 + c] = s - 128;
        }
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
  const int t = u >= kLuma;
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

// ---- 1a. symbol counts (optimize) ----------------------------------------------------------------
// Every Huffman symbol of block b, in stream order, to f(table, symbol): table 0 / 2 the DC of luma /
// chroma, 1 / 3 their AC.
template <typename Fn>
__device__ __forceinline__ void block_symbols(const JpegParams& p, const JpegGeom& g, const int16_t* coef,
                                              int b, Fn f) {
  const int u = b % p.per, t = u >= p.luma ? 2 : 0;
  const int16_t* z = coef + (int64_t)b * 64;
  f(t, nbits(dummy_block(p, g, b / p.per, u) ? 0 : z[0] - prev_dc(p, g, coef, b)));
  int run = 0;
#pragma unroll 1
  for (int k = 1; k < 64; ++k) {
    const int v = z[kZigzagDev[k]];
    if (v == 0) {
      ++run;
      continue;
    }
    for (; run > 15; run -= 16) f(t + 1, 0xF0);
    f(t + 1, (run << 4) | nbits(v));
    run = 0;
  }
  if (run) f(t + 1, 0);
}

__global__ void __launch_bounds__(kChunk) hist_kernel(const __grid_constant__ JpegParams p) {
  __shared__ uint32_t count[4 * 256];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  for (int i = threadIdx.x; i < 4 * 256; i += kChunk) count[i] = 0;
  __syncthreads();
  const int b = blockIdx.x * kChunk + threadIdx.x;
  if (b < g.blocks)
    block_symbols(p, g, p.coef + g.blk * 64, b, [&](int t, int sym) { atomicAdd(&count[t * 256 + sym], 1u); });
  __syncthreads();
  unsigned long long* freq = p.freq + (int64_t)blockIdx.y * 4 * 256;
  for (int i = threadIdx.x; i < 4 * 256; i += kChunk)
    if (count[i]) atomicAdd(freq + i, (unsigned long long)count[i]);
}

// ---- 1b. optimal tables (optimize) ----------------------------------------------------------------
// The symbol with the smallest nonzero count other than `skip`, the larger symbol on ties (-1 for
// none): one of jpeg_gen_optimal_table's searches, over the warp.
__device__ __forceinline__ int warp_min_symbol(const unsigned long long* f, int skip, int lane) {
  unsigned long long best = ~0ull;
  int sym = -1;
  for (int i = lane; i < 257; i += 32)
    if (f[i] && i != skip && f[i] <= best) {
      best = f[i];
      sym = i;
    }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const unsigned long long ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int os = __shfl_xor_sync(0xffffffffu, sym, o);
    if (os >= 0 && (sym < 0 || ob < best || (ob == best && os > sym))) {
      best = ob;
      sym = os;
    }
  }
  return sym;
}

// jpeg_gen_optimal_table (JPEG Annex K.2 with libjpeg's tie-breaking and the reserved symbol 256,
// whose all-ones code no real symbol gets) of the 256 counts at src, built by one warp in its shared
// f, sz, ot (257 each) and nb (33), then its DHT contents (bits, vals, count) and canonical codes.
__device__ __forceinline__ void optimal_table(const unsigned long long* src, unsigned long long* f, int16_t* sz,
                                              int16_t* ot, int* nb, uint8_t* bits, uint8_t* vals,
                                              int16_t* count, uint16_t* code, uint8_t* len, int lane) {
  for (int i = lane; i < 257; i += 32) {
    f[i] = i < 256 ? src[i] : 1;
    sz[i] = 0;
    ot[i] = -1;
  }
  for (int i = lane; i < 33; i += 32) nb[i] = 0;
  __syncwarp();
  for (;;) {
    int c1 = warp_min_symbol(f, -1, lane);
    int c2 = warp_min_symbol(f, c1, lane);
    if (c2 < 0) break;
    if (lane == 0) {
      f[c1] += f[c2];
      f[c2] = 0;
      ++sz[c1];
      while (ot[c1] >= 0) ++sz[c1 = ot[c1]];
      ot[c1] = (int16_t)c2;
      ++sz[c2];
      while (ot[c2] >= 0) ++sz[c2 = ot[c2]];
    }
    __syncwarp();
  }
  if (lane == 0) {
    for (int i = 0; i < 257; ++i)
      if (sz[i]) ++nb[min((int)sz[i], 32)];  // libjpeg refuses longer codes (2^31 symbols and more)
    for (int i = 32; i > 16; --i)           // lengths above 16 moved up the tree
      while (nb[i] > 0) {
        int j = i - 2;
        while (nb[j] == 0) --j;
        nb[i] -= 2;
        ++nb[i - 1];
        nb[j + 1] += 2;
        --nb[j];
      }
    int i = 16;
    while (nb[i] == 0) --i;
    --nb[i];                                // the reserved symbol's code
    int n = 0;
    for (int l = 1; l <= 16; ++l) {
      bits[l - 1] = (uint8_t)nb[l];
      n += nb[l];
    }
    *count = (int16_t)n;
  }
  __syncwarp();
  // the symbols by (length before the limit, symbol)
  for (int s = lane; s < 256; s += 32) {
    if (!sz[s]) continue;
    int rank = 0;
    for (int u = 0; u < 256; ++u) rank += sz[u] && (sz[u] < sz[s] || (sz[u] == sz[s] && u < s));
    vals[rank] = (uint8_t)s;
  }
  __syncwarp();
  if (lane == 0) {                          // canonical codes, as Annex C assigns them
    int c = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
      for (int i = 0; i < bits[l - 1]; ++i, ++k, ++c) {
        code[vals[k]] = (uint16_t)c;
        len[vals[k]] = (uint8_t)l;
      }
      c <<= 1;
    }
  }
}

// The optimal tables of frame blockIdx.x's four tables, warp t building table t.
__global__ void __launch_bounds__(kTableThreads) table_kernel(const __grid_constant__ JpegParams p) {
  __shared__ unsigned long long freq[4][257];
  __shared__ int16_t size[4][257], others[4][257];
  __shared__ int bits[4][33];
  const int t = threadIdx.x >> 5, lane = threadIdx.x & 31;
  FrameHuff& fh = p.huff[blockIdx.x];
  const bool ac = t & 1;
  optimal_table(p.freq + ((int64_t)blockIdx.x * 4 + t) * 256, freq[t], size[t], others[t], bits[t],
                fh.s.bits[t], fh.s.vals[t], &fh.s.count[t], ac ? fh.c.ac_code[t >> 1] : fh.c.dc_code[t >> 1],
                ac ? fh.c.ac_len[t >> 1] : fh.c.dc_len[t >> 1], lane);
}

// ---- 2. code lengths and chunk sums -------------------------------------------------------------
// The bits of block b's codes: its DC difference (the block before it of its component is another
// thread's), then its AC run/size codes with ZRLs and EOB.
__device__ __forceinline__ int block_bits(const JpegParams& p, const JpegGeom& g, const HuffCodes& H, const int16_t* coef, int b) {
  const int u = b % p.per, t = u >= p.luma;
  const int16_t* z = coef + (int64_t)b * 64;
  const int diff = dummy_block(p, g, b / p.per, u) ? 0 : z[0] - prev_dc(p, g, coef, b);
  int bits = H.dc_len[t][nbits(diff)] + nbits(diff), run = 0;
#pragma unroll 4
  for (int k = 1; k < 64; ++k) {
    const int v = z[kZigzagDev[k]];
    if (v == 0) {
      ++run;
    } else {
      const int nb = nbits(v);
      bits += (run >> 4) * H.ac_len[t][0xF0] + H.ac_len[t][((run & 15) << 4) | nb] + nb;
      run = 0;
    }
  }
  return bits + (run ? H.ac_len[t][0] : 0);
}

template <bool kOpt>
__global__ void __launch_bounds__(kChunk) block_bits_kernel(const __grid_constant__ JpegParams p) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  const int b = blockIdx.x * kChunk + threadIdx.x;
  const int bits = b < g.blocks ? block_bits(p, g, huff_codes_of<kOpt>(p, blockIdx.y), p.coef + g.blk * 64, b) : 0;
  p.bits[g.blk + b] = (uint32_t)bits;
  int64_t total;
  block_exclusive_scan(bits, warp, &total);
  if (threadIdx.x == 0) p.sums[g.csum + blockIdx.x] = total;
}

// ---- 3, 3b, 6. per-frame exclusive scans of chunk sums ----------------------------------------------
enum ScanOf { kScanBlocks, kScanStuffing, kScanIntervals };
// Frame blockIdx.x's `count` chunk sums from sums[first] become their exclusive scan, and the slot
// after them the total.
__global__ void __launch_bounds__(kScanThreads) scan_kernel(const __grid_constant__ JpegParams p,
                                                            int which) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.x];
  int64_t* s = p.sums + (which == kScanBlocks ? g.csum : which == kScanStuffing ? g.ssum : g.isum);
  const int count = which == kScanBlocks ? g.chunks : which == kScanStuffing ? g.schunks : g.ints;
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

// ---- 3a. restart intervals --------------------------------------------------------------------------
// The first bit of block b (b <= blocks) in the unpadded stream, from its chunk's first bit.
__device__ int64_t block_first_bit(const JpegParams& p, const JpegGeom& g, int b) {
  if (b == g.blocks) return p.sums[g.csum + g.chunks];
  int64_t s = p.sums[g.csum + b / kChunk];
  for (int k = b - b % kChunk; k < b; ++k) s += p.bits[g.blk + k];
  return s;
}

// One thread per interval: its first bit, and its bytes once padded to a byte.
__global__ void __launch_bounds__(kChunk) interval_kernel(const __grid_constant__ JpegParams p) {
  const JpegGeom& g = p.g[blockIdx.y];
  const int i = blockIdx.x * kChunk + threadIdx.x;
  if (i >= g.ints) return;
  const int first = i * p.rst * p.per, end = min(first + p.rst * p.per, g.blocks);
  const int64_t a = block_first_bit(p, g, first), e = block_first_bit(p, g, end);
  p.ipos[g.ipos + i] = a;
  p.sums[g.isum + i] = (e - a + 7) >> 3;
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

template <bool kOpt>
__global__ void __launch_bounds__(kChunk) pack_kernel(const __grid_constant__ JpegParams p) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  const int b = blockIdx.x * kChunk + threadIdx.x;
  const int64_t gb = g.blk + b;
  const int64_t bits = b < g.blocks ? p.bits[gb] : 0;
  int64_t total;
  int64_t pos = p.sums[g.csum + blockIdx.x] + block_exclusive_scan(bits, warp, &total);
  if (b >= g.blocks) return;
  bool last = b == g.blocks - 1;          // the last block of its interval pads it to a byte
  if (p.rst) {                            // from the interval's first bit to its first byte
    const int span = p.rst * p.per, i = b / span;
    pos += 8 * p.sums[g.isum + i] - p.ipos[g.ipos + i];
    last |= (b + 1) % span == 0;
  }
  const HuffCodes& H = huff_codes_of<kOpt>(p, blockIdx.y);
  const int u = b % p.per, t = u >= p.luma;
  BitWriter w{p.stream + g.words + (pos >> 5), 0, (int)(pos & 31)};
  const bool dummy = dummy_block(p, g, b / p.per, u);
  const int16_t* z = p.coef + gb * 64;
  const int diff = dummy ? 0 : z[0] - prev_dc(p, g, p.coef + g.blk * 64, b);
  const int dn = nbits(diff);
  w.put(H.dc_code[t][dn], H.dc_len[t][dn]);
  if (dn) w.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << dn) - 1), dn);
  int run = 0;
#pragma unroll 1
  for (int k = 1; k < 64; ++k) {
    const int v = z[kZigzagDev[k]];
    if (v == 0) {
      ++run;
      continue;
    }
    for (; run > 15; run -= 16) w.put(H.ac_code[t][0xF0], H.ac_len[t][0xF0]);
    const int nb = nbits(v), sym = (run << 4) | nb;
    w.put(H.ac_code[t][sym], H.ac_len[t][sym]);
    w.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << nb) - 1), nb);
    run = 0;
  }
  if (run) w.put(H.ac_code[t][0], H.ac_len[t][0]);
  if (last) {                               // 1-bits to the byte boundary
    const int pad = (int)(-(pos + bits) & 7);
    if (pad) w.put((1u << pad) - 1, pad);
  }
  w.flush();
}

// ---- progressive: ten scans ------------------------------------------------------------------------
// jpeg_simple_progression for YCbCr, one 6-bit field per scan: Ss, Se, Ah, Al and the component (3:
// all three, interleaved over the MCUs as the baseline scan is).
constexpr uint64_t scan_fields(const int (&v)[kScans]) {
  uint64_t r = 0;
  for (int s = 0; s < kScans; ++s) r |= (uint64_t)v[s] << (6 * s);
  return r;
}
constexpr uint64_t kScanSs = scan_fields({0, 1, 1, 1, 6, 1, 0, 1, 1, 1});
constexpr uint64_t kScanSe = scan_fields({0, 5, 63, 63, 63, 63, 0, 63, 63, 63});
constexpr uint64_t kScanAh = scan_fields({0, 0, 0, 0, 0, 2, 1, 1, 1, 1});
constexpr uint64_t kScanAl = scan_fields({1, 2, 1, 1, 2, 1, 0, 0, 0, 0});
constexpr uint64_t kScanComp = scan_fields({3, 0, 2, 1, 0, 0, 3, 2, 1, 0});
__host__ __device__ __forceinline__ int scan_field(uint64_t f, int s) { return (int)(f >> (6 * s)) & 63; }
constexpr int kEobrunMax = 0x7FFF;       // EOBRUN is emitted when it reaches this
constexpr int kMaxBe = 1000 - 64 + 1;    // or when the buffered correction bits pass MAX_CORR_BITS - 64 + 1

// The most bits one unit of scan s codes, with the EOBRUN flush after it (16 + 14 bits): a DC
// difference of 16 + 11 bits; a refinement bit; 16 + 10 bits per first-scan coefficient (a ZRL
// costs at most a bit per zero); 16 + 1 per newly nonzero refinement coefficient and 1 per other.
__host__ __device__ inline int prog_max_unit_bits(int s) {
  const int n = scan_field(kScanSe, s) - scan_field(kScanSs, s) + 1;
  if (scan_field(kScanSs, s) == 0) return scan_field(kScanAh, s) ? 1 : 27;
  return (scan_field(kScanAh, s) ? 17 : 26) * n + 30;
}

// A scan of an h x w frame: its units (the blocks it codes: every block of the MCUs for the DC
// scans, the component's ceil(w_c / 8) x ceil(h_c / 8) blocks in raster order for the AC scans),
// the frame's unit of its first (scans start at chunk boundaries), units per restart interval (all
// of them without), its intervals and the frame's index of its first.
struct ScanGeom {
  int units, first, span, ints, iseg;
};
enum FindBy { kByScan, kByUnit, kByInterval };

__host__ __device__ inline int scan_units(int h, int w, int hs, int vs, int s) {
  const int mcus = ((h + 8 * vs - 1) / (8 * vs)) * ((w + 8 * hs - 1) / (8 * hs));
  const int c = scan_field(kScanComp, s);
  return c == 3 ? mcus * (hs * vs + 2) : c ? mcus : ((h + 7) >> 3) * ((w + 7) >> 3);
}

// The scan numbered i (kByScan), or holding the frame's unit (kByUnit) or interval (kByInterval) i,
// and its geometry in q.  Scan kScans is the frame's end: q.first and q.iseg are its units (padded)
// and intervals.
__host__ __device__ __forceinline__ int find_scan(int h, int w, int hs, int vs, int rst, FindBy by, int i, ScanGeom& q) {
  q = ScanGeom{0, 0, 0, 0, 0};
  for (int k = 0;; ++k) {
    q.units = k < kScans ? scan_units(h, w, hs, vs, k) : 0;
    q.span = rst ? rst * (k < kScans && scan_field(kScanComp, k) == 3 ? hs * vs + 2 : 1) : (q.units ? q.units : 1);
    q.ints = (q.units + q.span - 1) / q.span;
    const int padded = (q.units + kChunk - 1) / kChunk * kChunk;
    if (k == kScans || (by == kByScan ? k == i : by == kByUnit ? i < q.first + padded : i < q.iseg + q.ints)) return k;
    q.first += padded;
    q.iseg += q.ints;
  }
}
__device__ __forceinline__ int find_scan(const JpegParams& p, const JpegGeom& g, FindBy by, int i, ScanGeom& q) {
  return find_scan(g.h, g.w, p.hs, p.vs, p.rst, by, i, q);
}

// The block (stream order) of unit u of a scan of component c.
__device__ __forceinline__ int unit_block(const JpegParams& p, const JpegGeom& g, int c, int u) {
  if (c == 3) return u;
  if (c) return u * p.per + p.luma + c - 1;
  const int wib = (g.w + 7) >> 3, bx = u % wib, by = u / wib;
  return ((by / p.vs) * g.mcu_cols + bx / p.hs) * p.per + (by % p.vs) * p.hs + bx % p.hs;
}

// The DC of block b: a dummy block's is the last real block's before it (its MCU's first luma block
// is real), as libjpeg fills dummy blocks in for multi-scan files.
__device__ __forceinline__ int eff_dc(const JpegParams& p, const JpegGeom& g, const int16_t* coef, int b) {
  const int m = b / p.per;
  int u = b - m * p.per;
  while (dummy_block(p, g, m, u)) --u;
  return coef[(int64_t)(m * p.per + u) * 64];
}

// What a unit leaves after its codes: whether it coded a symbol (so that a pending EOBRUN is
// emitted before its codes), whether it adds one to EOBRUN, and its correction bits buffered behind
// the run (refinement: the last `tail` bits of tail_bits).
struct UnitEnd {
  bool sym, eob;
  int tail;
  uint64_t tail_bits;
};

// Raw bits, at most 64, to f.
template <class Fn>
__device__ __forceinline__ void put_raw(Fn& f, uint64_t bits, int n) {
  if (n > 32) f(-1, 0, (uint32_t)(bits >> 32), n - 32);
  if (n) f(-1, 0, (uint32_t)bits, min(n, 32));
}

// The codes of unit u (the frame's index) of scan s (geometry q), in order, to f(slot, symbol,
// extra bits, their length); slot -1: `extra` is raw bits.  EOBRUN flushes are not the unit's.
template <class Fn>
__device__ __forceinline__ UnitEnd unit_codes(const JpegParams& p, const JpegGeom& g, const int16_t* coef, int s,
                              const ScanGeom& q, int u, Fn&& f) {
  const int ss = scan_field(kScanSs, s), se = scan_field(kScanSe, s), ah = scan_field(kScanAh, s);
  const int al = scan_field(kScanAl, s), c = scan_field(kScanComp, s);
  const int local = u - q.first;
  UnitEnd e{false, false, 0, 0};
  if (ss == 0) {                          // DC: the point transform is an arithmetic shift
    const int b = local, dc = eff_dc(p, g, coef, b) >> al;
    if (ah) {
      f(-1, 0, (uint32_t)dc & 1, 1);
      return e;
    }
    const int m = b / p.per, k = b - m * p.per;
    const int prev = k >= p.luma ? b - p.per : k ? b - 1 : b - p.per + p.luma - 1;
    const int first = p.rst ? (m - m % p.rst) * p.per : 0;     // the interval's first block
    const int diff = dc - (prev >= first ? eff_dc(p, g, coef, prev) >> al : 0), nb = nbits(diff);
    f(k >= p.luma ? kChromaDcSlot : 0, nb, (uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << nb) - 1), nb);
    e.sym = true;
    return e;
  }
  const int16_t* z = coef + (int64_t)unit_block(p, g, c, local) * 64;
  int run = 0;
  if (!ah) {                              // AC first: |v| >> Al
#pragma unroll 1
    for (int k = ss; k <= se; ++k) {
      const int v = z[kZigzagDev[k]], a = abs(v) >> al;
      if (!a) {
        ++run;
        continue;
      }
      for (; run > 15; run -= 16) f(s, 0xF0, 0u, 0);
      const int nb = nbits(a);
      f(s, (run << 4) | nb, (uint32_t)(v < 0 ? ~a : a) & ((1u << nb) - 1), nb);
      run = 0;
      e.sym = true;
    }
    e.eob = run > 0;
    return e;
  }
  // AC refinement: |v| >> Al == 1 is newly nonzero, larger values get a correction bit; runs count
  // the coefficients still zero, and ZRLs past the last newly nonzero one fold into the EOB run
  int eob = 0, br = 0;
  uint64_t bb = 0;
#pragma unroll 1
  for (int k = ss; k <= se; ++k)
    if ((abs(z[kZigzagDev[k]]) >> al) == 1) eob = k;
#pragma unroll 1
  for (int k = ss; k <= se; ++k) {
    const int v = z[kZigzagDev[k]], a = abs(v) >> al;
    if (!a) {
      ++run;
      continue;
    }
    for (; run > 15 && k <= eob; run -= 16) {
      f(s, 0xF0, 0u, 0);
      put_raw(f, bb, br);
      bb = 0;
      br = 0;
      e.sym = true;
    }
    if (a > 1) {
      bb = bb << 1 | (a & 1);
      ++br;
      continue;
    }
    f(s, (run << 4) | 1, (uint32_t)(v >= 0), 1);
    put_raw(f, bb, br);
    bb = 0;
    br = run = 0;
    e.sym = true;
  }
  e.eob = run > 0 || br > 0;
  e.tail = br;
  e.tail_bits = bb;
  return e;
}

// The frame's tails (buffered correction bits) and symbol-coding units before unit k, from the
// chunk sums at tsum (tails, then symbol units) and the in-chunk prefixes in pre.
__device__ __forceinline__ int64_t tails_before(const JpegParams& p, const JpegGeom& g, int k) {
  return p.sums[g.tsum + k / kChunk] + (k % kChunk ? p.pre[g.blk + k] & 0xFFFF : 0);
}
__device__ __forceinline__ int64_t syms_before(const JpegParams& p, const JpegGeom& g, int k) {
  return p.sums[g.tsum + g.chunks + 1 + k / kChunk] + (k % kChunk ? p.pre[g.blk + k] >> 16 : 0);
}

// ---- P1. units: flags, prefixes, symbol counts -------------------------------------------------------
// Grid (unit chunk, frame): each unit's UnitEnd as flags (sym | eob << 1 | tail << 2), the in-chunk
// exclusive prefixes of tails and symbol units (pre: tails | syms << 16) and their chunk sums, and
// the counts of the unit's own symbols.  A chunk lies in one scan, so it counts into at most two
// tables (scan 0's DC luma and chroma).
__global__ void __launch_bounds__(kChunk) prog_units_kernel(const __grid_constant__ JpegParams p) {
  __shared__ uint32_t count[2][256];
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  for (int i = threadIdx.x; i < 2 * 256; i += kChunk) count[i >> 8][i & 255] = 0;
  __syncthreads();
  const int u = blockIdx.x * kChunk + threadIdx.x;
  ScanGeom q;
  const int s = find_scan(p, g, kByUnit, u, q);
  uint32_t flags = 0;
  if (u - q.first < q.units) {
    const UnitEnd e = unit_codes(p, g, p.coef + g.cblk * 64, s, q, u, [&](int slot, int sym, uint32_t, int) {
      if (slot >= 0) atomicAdd(&count[slot == kChromaDcSlot][sym], 1u);
    });
    flags = (uint32_t)e.sym | (uint32_t)e.eob << 1 | (uint32_t)e.tail << 2;
  }
  p.flags[g.blk + u] = flags;
  int64_t tails, syms;
  const int64_t tb = block_exclusive_scan(flags >> 2, warp, &tails);
  const int64_t sb = block_exclusive_scan(flags & 1, warp, &syms);
  p.pre[g.blk + u] = (uint32_t)tb | (uint32_t)sb << 16;
  if (threadIdx.x == 0) {
    p.sums[g.tsum + blockIdx.x] = tails;
    p.sums[g.tsum + g.chunks + 1 + blockIdx.x] = syms;
  }
  __syncthreads();
  unsigned long long* freq = p.freq + (int64_t)blockIdx.y * kSlots * 256;
  for (int i = threadIdx.x; i < 2 * 256; i += kChunk) {
    const uint32_t n = count[i >> 8][i & 255];
    if (n) atomicAdd(freq + (i >> 8 ? kChromaDcSlot : s) * 256 + (i & 255), (unsigned long long)n);
  }
}

// ---- P2. EOBRUN flushes -------------------------------------------------------------------------------
// A flush word: the EOBRUN emitted after a unit's codes and the correction bits buffered with it
// (E | B << 15); 0 for none.  An AC scan's units that code a symbol, and each interval's first,
// split it into segments whose other units code none.  The thread of the unit before a segment
// (of its first unit, at an interval's start) walks it from flush to flush: each unit adds one
// to EOBRUN and its tail to BE, a flush comes where EOBRUN reaches 0x7FFF (closed form) or BE
// passes kMaxBe (a binary search on the tails' prefix sums), and the segment's end flushes what is
// pending, before the next symbol or at the interval's end.  Its cost is its flushes.
__global__ void __launch_bounds__(kChunk) prog_eobrun_kernel(const __grid_constant__ JpegParams p) {
  __shared__ uint32_t count[256];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  for (int i = threadIdx.x; i < 256; i += kChunk) count[i] = 0;
  __syncthreads();
  const int u = blockIdx.x * kChunk + threadIdx.x;
  ScanGeom q;
  const int s = find_scan(p, g, kByUnit, u, q);
  const int local = u - q.first;
  const uint32_t fl = local < q.units ? p.flags[g.blk + u] : 0;
  if (scan_field(kScanSs, s) && local < q.units && ((fl & 1) || local % q.span == 0)) {
    const int iend = q.first + min((local / q.span + 1) * q.span, q.units);
    int E = 0, next = u;
    int64_t B = 0;
    if (fl & 1) {
      E = (fl >> 1) & 1;
      B = fl >> 2;
      next = u + 1;
    }
    auto flush = [&](int k, int e, int64_t b) {
      p.flush[g.blk + k] = (uint32_t)e | (uint32_t)b << 15;
      atomicAdd(&count[(nbits(e) - 1) << 4], 1u);
    };
    // the segment's last unit: before the next unit coding a symbol, or the interval's last
    const int64_t h0 = syms_before(p, g, u + 1);
    int lo = u + 1, hi = iend;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (syms_before(p, g, mid + 1) > h0) hi = mid;
      else lo = mid + 1;
    }
    const int e = lo - 1;
    for (;;) {
      const int64_t t0 = tails_before(p, g, next);
      int k = next + (kEobrunMax - E) - 1;
      if (B + tails_before(p, g, e + 1) - t0 > kMaxBe) {
        int a = next, z = e;
        while (a < z) {
          const int mid = (a + z) >> 1;
          if (B + tails_before(p, g, mid + 1) - t0 > kMaxBe) z = mid;
          else a = mid + 1;
        }
        k = min(k, a);
      }
      if (k > e) break;
      flush(k, E + k - next + 1, B + tails_before(p, g, k + 1) - t0);
      E = 0;
      B = 0;
      next = k + 1;
    }
    E += e - next + 1;
    if (E > 0) flush(e, E, B + tails_before(p, g, e + 1) - tails_before(p, g, next));
  }
  __syncthreads();
  unsigned long long* freq = p.freq + ((int64_t)blockIdx.y * kSlots + s) * 256;
  for (int i = threadIdx.x; i < 256; i += kChunk)
    if (count[i]) atomicAdd(freq + i, (unsigned long long)count[i]);
}

// ---- P3. tables ---------------------------------------------------------------------------------------
// Frame blockIdx.x's optimal tables, warp t building slot t's (none for the DC refinement).
__global__ void __launch_bounds__(kSlots * 32) prog_table_kernel(const __grid_constant__ JpegParams p) {
  __shared__ unsigned long long freq[kSlots][257];
  __shared__ int16_t size[kSlots][257], others[kSlots][257];
  __shared__ int bits[kSlots][33];
  const int t = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (t == 6) return;
  ProgHuff& h = p.phuff[blockIdx.x];
  optimal_table(p.freq + ((int64_t)blockIdx.x * kSlots + t) * 256, freq[t], size[t], others[t], bits[t],
                h.bits[t], h.vals[t], &h.count[t], h.code[t], h.len[t], lane);
}

// ---- P4. unit lengths and chunk sums -------------------------------------------------------------------
// The bits of a flush word's EOBRUN code, its low bits and the buffered correction bits.
__device__ __forceinline__ int flush_bits(const ProgHuff& h, int s, uint32_t fw) {
  if (!fw) return 0;
  const int nb = nbits((int)(fw & 0x7FFF)) - 1;
  return h.len[s][nb << 4] + nb + (int)(fw >> 15);
}

__global__ void __launch_bounds__(kChunk) prog_bits_kernel(const __grid_constant__ JpegParams p) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  const int u = blockIdx.x * kChunk + threadIdx.x;
  ScanGeom q;
  const int s = find_scan(p, g, kByUnit, u, q);
  const ProgHuff& h = p.phuff[blockIdx.y];
  int bits = 0;
  if (u - q.first < q.units) {
    unit_codes(p, g, p.coef + g.cblk * 64, s, q, u,
               [&](int slot, int sym, uint32_t, int nb) { bits += (slot >= 0 ? h.len[slot][sym] : 0) + nb; });
    bits += flush_bits(h, s, p.flush[g.blk + u]);
  }
  p.bits[g.blk + u] = (uint32_t)bits;
  int64_t total;
  block_exclusive_scan(bits, warp, &total);
  if (threadIdx.x == 0) p.sums[g.csum + blockIdx.x] = total;
}

// ---- P5. intervals: one per restart interval of each scan (one per scan without) ------------------------
__global__ void __launch_bounds__(kChunk) prog_interval_kernel(const __grid_constant__ JpegParams p) {
  const JpegGeom& g = p.g[blockIdx.y];
  const int i = blockIdx.x * kChunk + threadIdx.x;
  if (i >= g.ints) return;
  ScanGeom q;
  find_scan(p, g, kByInterval, i, q);
  const int j = i - q.iseg;
  const int first = q.first + j * q.span, end = q.first + min((j + 1) * q.span, q.units);
  const int64_t a = block_first_bit(p, g, first), e = block_first_bit(p, g, end);
  p.ipos[g.ipos + i] = a;
  p.sums[g.isum + i] = (e - a + 7) >> 3;
}

// ---- P6. pack --------------------------------------------------------------------------------------------
// Each unit ORs in its codes, then its flush: the EOBRUN code and the tails of the run's units (the
// last E units, each adding one), found by binary search on the tails' prefix sums; the last unit
// of an interval pads it to a byte with 1-bits.
// A unit's codes with the frame's tables (slot -1: raw bits) into a BitWriter.
struct CodeWriter {
  BitWriter w;
  const ProgHuff& h;
  __device__ __forceinline__ void operator()(int slot, int sym, uint32_t extra, int nb) {
    if (slot >= 0) w.put(h.code[slot][sym], h.len[slot][sym]);
    if (nb) w.put(extra, nb);
  }
};

__global__ void __launch_bounds__(kChunk) prog_pack_kernel(const __grid_constant__ JpegParams p) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.chunks) return;
  const int u = blockIdx.x * kChunk + threadIdx.x;
  const int64_t bits = p.bits[g.blk + u];
  int64_t total;
  int64_t pos = p.sums[g.csum + blockIdx.x] + block_exclusive_scan(bits, warp, &total);
  ScanGeom q;
  const int s = find_scan(p, g, kByUnit, u, q);
  const int local = u - q.first;
  if (local >= q.units) return;
  const int i = q.iseg + local / q.span;
  pos += 8 * p.sums[g.isum + i] - p.ipos[g.ipos + i];
  const bool last = local + 1 == q.units || (local + 1) % q.span == 0;
  const ProgHuff& h = p.phuff[blockIdx.y];
  const int16_t* coef = p.coef + g.cblk * 64;
  CodeWriter put{{p.stream + g.words + (pos >> 5), 0, (int)(pos & 31)}, h};
  unit_codes(p, g, coef, s, q, u, put);
  const uint32_t fw = p.flush[g.blk + u];
  if (fw) {
    const int E = (int)(fw & 0x7FFF), nb = nbits(E) - 1;
    put(s, nb << 4, (uint32_t)E & ((1u << nb) - 1), nb);
    const int64_t end = tails_before(p, g, u + 1);
    for (int k = u - E + 1; k <= u;) {
      const int64_t t = tails_before(p, g, k);
      if (t == end) break;
      int lo = k, hi = u;                 // the first unit from k on with a tail
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (tails_before(p, g, mid + 1) > t) hi = mid;
        else lo = mid + 1;
      }
      // its tail: the correction bits after its last newly nonzero coefficient (no code follows it)
      const int16_t* z = coef + (int64_t)unit_block(p, g, scan_field(kScanComp, s), lo - q.first) * 64;
      const int ss = scan_field(kScanSs, s), se = scan_field(kScanSe, s), al = scan_field(kScanAl, s);
      int eob = 0;
#pragma unroll 1
      for (int j = ss; j <= se; ++j)
        if ((abs(z[kZigzagDev[j]]) >> al) == 1) eob = j;
#pragma unroll 1
      for (int j = max(eob + 1, ss); j <= se; ++j) {
        const int a = abs(z[kZigzagDev[j]]) >> al;
        if (a > 1) put(-1, 0, (uint32_t)a & 1, 1);
      }
      k = lo + 1;
    }
  }
  if (last) {                               // 1-bits to the byte boundary
    const int pad = (int)(-(pos + bits) & 7);
    if (pad) put.w.put((1u << pad) - 1, pad);
  }
  put.w.flush();
}

// ---- P7. markers between intervals ---------------------------------------------------------------------
// A DHT segment of slot t's table as class/id `id`, byte i.
__device__ __forceinline__ uint8_t dht_byte(const ProgHuff& h, int t, int id, int i) {
  if (i < 2) return i ? 0xC4 : 0xFF;
  const int len = 19 + h.count[t];
  if (i < 4) return (uint8_t)(i == 2 ? len >> 8 : len);
  if (i == 4) return (uint8_t)id;
  return i < 21 ? h.bits[t][i - 5] : h.vals[t][i - 21];
}

// The bytes before interval i >= 1 of a progressive frame: RSTn within a scan, and at a scan's start
// its DHT (AC scans) and SOS.
__device__ __forceinline__ int prog_marker_bytes(const JpegParams& p, const JpegGeom& g, int i) {
  ScanGeom q;
  const int s = find_scan(p, g, kByInterval, i, q);
  if (i > q.iseg) return 2;
  return scan_field(kScanSs, s) ? 21 + p.phuff[blockIdx.y].count[s] + 10 : 14;
}

// ---- 5. 0xFF counts -----------------------------------------------------------------------------
__device__ __forceinline__ uint8_t stream_byte(const uint32_t* words, int64_t j) {
  return (uint8_t)(words[j >> 2] >> (24 - 8 * (j & 3)));
}

// The bytes of the frame's stream before stuffing (progressive files always have intervals).
template <bool kProg>
__device__ __forceinline__ int64_t stream_bytes(const JpegParams& p, const JpegGeom& g) {
  return kProg || p.rst ? p.sums[g.isum + g.ints] : (p.sums[g.csum + g.chunks] + 7) >> 3;
}

// The first interval after the first (which has no marker) starting at byte `first` or later.
__device__ int first_marker(const JpegParams& p, const JpegGeom& g, int64_t first) {
  int lo = 1, hi = g.ints;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (p.sums[g.isum + mid] < first) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

template <bool kProg>
__global__ void __launch_bounds__(kStuffThreads) count_ff_kernel(const __grid_constant__ JpegParams p) {
  __shared__ int64_t warp[32];
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.schunks) return;
  const int64_t bytes = stream_bytes<kProg>(p, g);
  const int64_t first = (int64_t)blockIdx.x * kStuffChunk + threadIdx.x * kStuffBytes;
  const uint32_t* words = p.stream + g.words;
  int ff = 0;
  for (int i = 0; i < kStuffBytes && first + i < bytes; ++i) ff += stream_byte(words, first + i) == 0xFF;
  if ((kProg || p.rst) && first < bytes)    // RSTn: 2 bytes before an interval's first byte
    for (int i = first_marker(p, g, first); i < g.ints && p.sums[g.isum + i] < first + kStuffBytes; ++i)
      ff += kProg ? prog_marker_bytes(p, g, i) : 2;
  int64_t total;
  block_exclusive_scan(ff, warp, &total);
  if (threadIdx.x == 0) p.sums[g.ssum + blockIdx.x] = total;
}

// ---- 7. stuff, header, EOI, length --------------------------------------------------------------
// Byte i of the frame's header: the template's SOI .. SOF0 with the frame's height and width, the
// four DHT segments of `hs`, then the template's DRI and SOS.
__device__ __forceinline__ uint8_t header_byte(const StuffParams& sp, const JpegGeom& g, const HuffSpec& hs, int i) {
  if (i < kPrefixBytes) {
    if (i < kSofSize || i >= kSofSize + 4) return sp.prefix[i];
    const int v = i < kSofSize + 2 ? g.h : g.w;
    return (uint8_t)(i & 1 ? v >> 8 : v);          // kSofSize is odd: the high byte first
  }
  i -= kPrefixBytes;
  for (int t = 0; t < 4; ++t) {
    const int len = 21 + hs.count[t];
    if (i < len) {
      if (i < 2) return i ? 0xC4 : 0xFF;
      if (i < 4) return (uint8_t)(i == 2 ? (len - 2) >> 8 : len - 2);
      if (i == 4) return (uint8_t)(((t & 1) << 4) | (t >> 1));
      return i < 21 ? hs.bits[t][i - 5] : hs.vals[t][i - 21];
    }
    i -= len;
  }
  return sp.suffix[i];
}

// A progressive file's header: the template's SOI .. SOF2, scan 0's two DHT segments, the
// template's DRI and scan 0's SOS.
__device__ __forceinline__ uint8_t prog_header_byte(const StuffParams& sp, const JpegGeom& g, const ProgHuff& h, int i) {
  if (i < kPrefixBytes) return header_byte(sp, g, sp.std, i);
  i -= kPrefixBytes;
  for (int t = 0; t < 2; ++t) {
    const int len = 21 + h.count[t ? kChromaDcSlot : 0];
    if (i < len) return dht_byte(h, t ? kChromaDcSlot : 0, t, i);
    i -= len;
  }
  return i < sp.suffix_bytes ? sp.suffix[i] : sp.sos[0][i - sp.suffix_bytes];
}

// Writes the bytes before interval i >= 1 of a progressive frame at out + o; returns the new o.
__device__ __forceinline__ int64_t put_prog_marker(const StuffParams& sp, const JpegGeom& g, int i, int64_t o) {
  ScanGeom q;
  const int s = find_scan(sp.p, g, kByInterval, i, q);
  if (i > q.iseg) {
    g.out[o++] = 0xFF;
    g.out[o++] = (uint8_t)(0xD0 + ((i - q.iseg - 1) & 7));
    return o;
  }
  const int ss = scan_field(kScanSs, s);
  if (ss) {
    const ProgHuff& h = sp.p.phuff[blockIdx.y];
    const int id = 0x10 | (scan_field(kScanComp, s) ? 1 : 0);
    for (int k = 0; k < 21 + h.count[s]; ++k) g.out[o++] = dht_byte(h, s, id, k);
  }
  for (int k = 0; k < (ss ? 10 : 14); ++k) g.out[o++] = sp.sos[s][k];
  return o;
}

template <bool kOpt, bool kProg = false>
__global__ void __launch_bounds__(kStuffThreads) stuff_kernel(const __grid_constant__ StuffParams sp) {
  __shared__ int64_t warp[32];
  const JpegParams& p = sp.p;
  const JpegGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.schunks) return;
  const HuffSpec& hs = kOpt ? p.huff[blockIdx.y].s : sp.std;
  int header = kPrefixBytes + 84 + hs.count[0] + hs.count[1] + hs.count[2] + hs.count[3] + sp.suffix_bytes;
  if constexpr (kProg)
    header = kPrefixBytes + 42 + p.phuff[blockIdx.y].count[0] + p.phuff[blockIdx.y].count[kChromaDcSlot] +
             sp.suffix_bytes + kSosBytes;
  const int64_t bytes = stream_bytes<kProg>(p, g);
  const int64_t size = header + bytes + p.sums[g.ssum + g.schunks] + 2;
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
  int marker = g.ints;
  if ((kProg || p.rst) && first < bytes) {
    marker = first_marker(p, g, first);
    for (int i = marker; i < g.ints && p.sums[g.isum + i] < first + kStuffBytes; ++i)
      ff += kProg ? prog_marker_bytes(p, g, i) : 2;
  }
  int64_t total;
  int64_t o = header + first + p.sums[g.ssum + blockIdx.x] + block_exclusive_scan(ff, warp, &total);
  for (int i = 0; i < kStuffBytes && first + i < bytes; ++i) {
    if (marker < g.ints && p.sums[g.isum + marker] == first + i) {
      if constexpr (kProg) {
        o = put_prog_marker(sp, g, marker, o);
      } else {
        g.out[o++] = 0xFF;
        g.out[o++] = (uint8_t)(0xD0 + ((marker - 1) & 7));
      }
      ++marker;
    }
    // (progressive: the marker writes keep this loop rolled, so the byte is read again rather than
    // indexing v, which would put v in local memory)
    const uint8_t b = kProg ? stream_byte(words, first + i) : v[i];
    g.out[o++] = b;
    if (b == 0xFF) g.out[o++] = 0;
  }
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < header; i += kStuffThreads)
      g.out[i] = kProg ? prog_header_byte(sp, g, p.phuff[blockIdx.y], i) : header_byte(sp, g, hs, i);
    if (threadIdx.x == 0) {
      g.out[size - 2] = 0xFF;
      g.out[size - 1] = 0xD9;
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------
// What one call encodes with (cv2's parameters resolved): the luma and chroma qualities, the luma
// sampling factors, optimized tables or not, the restart interval in MCUs, and progressive or not.
struct Settings {
  int lq, cq, hs, vs, optimize, rst, prog;
};
constexpr Settings kDefaultSettings = {95, 95, 2, 2, 0, 0, 0};

// The parameters' settings, or a refusal naming the call: a quality outside [1, 100] (-1 leaves
// luma_quality and chroma_quality unset), a sampling other than cv2's five, optimize other than 0
// or 1, a restart interval outside [0, 65535].  As cv2: luma_quality replaces quality, chroma_quality
// counts only with it, and two different ones make the file 4:4:4.
int resolve_params(const std::string& name, const sqdet_jpeg_params* jp, Settings* s) {
  if (!jp) return fail(SQDET_ERR_INVALID_ARG, name + ": null params");
  if (jp->quality < 1 || jp->quality > 100) return fail(SQDET_ERR_INVALID_ARG, name + ": quality must be in [1, 100]");
  for (int q : {jp->luma_quality, jp->chroma_quality})
    if (q != -1 && (q < 1 || q > 100))
      return fail(SQDET_ERR_INVALID_ARG, name + ": luma_quality and chroma_quality must be -1 or in [1, 100]");
  const int f = jp->sampling;
  if (f != 0x411111 && f != 0x221111 && f != 0x211111 && f != 0x121111 && f != 0x111111)
    return fail(SQDET_ERR_INVALID_ARG, name + ": sampling must be 0x411111, 0x221111, 0x211111, 0x121111 or 0x111111");
  if (jp->optimize != 0 && jp->optimize != 1) return fail(SQDET_ERR_INVALID_ARG, name + ": optimize must be 0 or 1");
  if (jp->restart_interval < 0 || jp->restart_interval > 65535)
    return fail(SQDET_ERR_INVALID_ARG, name + ": restart_interval must be in [0, 65535]");
  s->hs = f >> 20;
  s->vs = (f >> 16) & 15;
  s->lq = s->cq = jp->quality;
  if (jp->luma_quality != -1) {
    s->lq = jp->luma_quality;
    s->cq = jp->chroma_quality != -1 ? jp->chroma_quality : s->lq;
    if (s->cq != s->lq) s->hs = s->vs = 1;
  }
  s->optimize = jp->optimize;
  s->rst = jp->restart_interval;
  s->prog = 0;
  return SQDET_OK;
}

// The header's template: SOI, JFIF APP0, DQT x 2 and SOF0 (progressive: SOF2; height and width 0)
// into prefix, DRI (with restart markers) and (baseline only) SOS into suffix; returns the suffix's
// bytes.
int jpeg_header(const uint16_t (&q)[2][64], const Settings& st, uint8_t* prefix, uint8_t* suffix) {
  uint8_t* out = prefix;
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
  seg(st.prog ? 0xC2 : 0xC0, 15);         // height and width at kSofSize, filled in per frame
  put({8, 0, 0, 0, 0, 3, 1, st.hs << 4 | st.vs, 0, 2, 0x11, 1, 3, 0x11, 1});
  out = suffix;
  n = 0;
  if (st.rst) {
    seg(0xDD, 2);
    put({st.rst >> 8, st.rst & 255});
  }
  if (st.prog) return n;
  seg(0xDA, 10);
  put({3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});
  return n;
}

// Each progressive scan's SOS: its components with their tables (DC first: the DC tables; AC: the
// component's AC table; 0 for a table the scan does not use), Ss, Se, Ah << 4 | Al.
void prog_sos(uint8_t (&sos)[kScans][kSosBytes]) {
  for (int s = 0; s < kScans; ++s) {
    const int c = scan_field(kScanComp, s), ss = scan_field(kScanSs, s), n = c == 3 ? 3 : 1;
    uint8_t* o = sos[s];
    int k = 0;
    for (int v : {0xFF, 0xDA, 0, 6 + 2 * n, n}) o[k++] = (uint8_t)v;
    for (int i = 0; i < n; ++i) {
      const int comp = c == 3 ? i : c;
      o[k++] = (uint8_t)(comp + 1);
      o[k++] = (uint8_t)(ss ? (comp ? 0x01 : 0x00) : scan_field(kScanAh, s) || !comp ? 0x00 : 0x10);
    }
    o[k++] = (uint8_t)ss;
    o[k++] = (uint8_t)scan_field(kScanSe, s);
    o[k++] = (uint8_t)(scan_field(kScanAh, s) << 4 | scan_field(kScanAl, s));
  }
}

// The Annex K tables as DHT writes them.
HuffSpec std_spec() {
  HuffSpec h{};
  const uint8_t* bits[4] = {kDcLumaBits, kAcLumaBits, kDcChromaBits, kAcChromaBits};
  const uint8_t* vals[4] = {kDcVals, kAcLumaVals, kDcVals, kAcChromaVals};
  for (int t = 0; t < 4; ++t) {
    int count = 0;
    for (int l = 0; l < 16; ++l) count += h.bits[t][l] = bits[t][l];
    for (int k = 0; k < count; ++k) h.vals[t][k] = vals[t][k];
    h.count[t] = (int16_t)count;
  }
  return h;
}

// One frame's sizes in the scratch.  A progressive frame codes units, the blocks of each of its
// scans (ScanGeom), in uchunks chunks; its ints are the intervals of all its scans.
struct FrameSizes {
  int blocks, chunks, schunks, ints, uchunks;
  int64_t bytes, words;                 // the stream's largest bytes before stuffing, its words
};
FrameSizes frame_sizes(int h, int w, const Settings& st) {
  FrameSizes s;
  const int64_t mcus = (int64_t)((h + 8 * st.vs - 1) / (8 * st.vs)) * ((w + 8 * st.hs - 1) / (8 * st.hs));
  s.blocks = (int)(mcus * (st.hs * st.vs + 2));
  s.chunks = (s.blocks + kChunk - 1) / kChunk;
  s.ints = st.rst ? (int)((mcus + st.rst - 1) / st.rst) : 1;
  s.uchunks = s.chunks;
  // each interval is padded to a byte
  s.bytes = ((int64_t)s.blocks * (st.optimize ? kMaxBlockBitsOpt : kMaxBlockBits) + 7) / 8 + (st.rst ? s.ints : 0);
  if (st.prog) {
    ScanGeom q;
    s.bytes = 0;
    for (int k = 0; k < kScans; ++k) {
      find_scan(h, w, st.hs, st.vs, st.rst, kByScan, k, q);
      s.bytes += ((int64_t)q.units * prog_max_unit_bits(k) + 7) / 8 + q.ints;
    }
    find_scan(h, w, st.hs, st.vs, st.rst, kByScan, kScans, q);
    s.uchunks = q.first / kChunk;
    s.ints = q.iseg;
  }
  s.schunks = (int)((s.bytes + kStuffChunk - 1) / kStuffChunk);
  s.words = (s.bytes + 3) / 4 + 1;
  return s;
}

// The scratch of the frames [first, first + count): coefficients, bit lengths, chunk sums,
// intervals' first bits, bit buffers, symbol counts and tables, in that order.
// A progressive frame's unit lengths, flags, prefixes and flush words follow the bit lengths, and
// its tail and symbol-unit chunk sums the interval sums; g then describes the frame's units (blk,
// blocks and chunks count units) and cblk its first block.
struct GroupLayout {
  int64_t coef, bits, flags, pre, sums, ipos, flush, stream, freq, huff, total;
};
GroupLayout group_layout(const FrameSource* fr, int first, int count, const Settings& st, JpegGeom* g) {
  int64_t blocks = 0, units = 0, sums = 0, ints = 0, words = 0;
  for (int i = 0; i < count; ++i) {
    const FrameSource& s = fr[first + i];
    const FrameSizes z = frame_sizes(s.h, s.w, st);
    const int isums = st.rst || st.prog ? z.ints + 1 : 0;
    if (g && st.prog) {
      g[i].h = s.h;
      g[i].w = s.w;
      g[i].mcu_cols = (s.w + 8 * st.hs - 1) / (8 * st.hs);
      g[i].blocks = z.uchunks * kChunk;
      g[i].chunks = z.uchunks;
      g[i].schunks = z.schunks;
      g[i].ints = z.ints;
      g[i].blk = units;
      g[i].cblk = blocks;
      g[i].csum = sums;
      g[i].ssum = sums + z.uchunks + 1;
      g[i].isum = sums + z.uchunks + 1 + z.schunks + 1;
      g[i].tsum = g[i].isum + isums;
      g[i].ipos = ints;
      g[i].words = words;
    } else if (g) {
      g[i].h = s.h;
      g[i].w = s.w;
      g[i].mcu_cols = (s.w + 8 * st.hs - 1) / (8 * st.hs);
      g[i].blocks = z.blocks;
      g[i].chunks = z.chunks;
      g[i].schunks = z.schunks;
      g[i].ints = z.ints;
      g[i].blk = blocks;
      g[i].csum = sums;
      g[i].ssum = sums + z.chunks + 1;
      g[i].isum = sums + z.chunks + 1 + z.schunks + 1;
      g[i].ipos = ints;
      g[i].words = words;
    }
    blocks += (int64_t)z.chunks * kChunk;
    units += (int64_t)z.uchunks * kChunk;
    sums += z.uchunks + 1 + z.schunks + 1 + isums + (st.prog ? 2 * (z.uchunks + 1) : 0);
    ints += st.rst || st.prog ? z.ints : 0;
    words += z.words;
  }
  const int64_t unit_words = st.prog ? align256(units * 4) : 0;
  GroupLayout L;
  L.coef = 0;
  L.bits = L.coef + align256(blocks * 64 * 2);
  L.flags = L.bits + align256(units * 4);
  L.pre = L.flags + unit_words;
  L.sums = L.pre + unit_words;
  L.ipos = L.sums + align256(sums * 8);
  L.flush = L.ipos + align256(ints * 8);
  L.stream = L.flush + unit_words;
  L.freq = L.stream + align256(words * 4);
  L.huff = L.freq + (st.prog ? align256((int64_t)count * kSlots * 256 * 8)
                             : st.optimize ? align256((int64_t)count * 4 * 256 * 8) : 0);
  L.total = L.huff + (st.prog ? align256((int64_t)count * sizeof(ProgHuff))
                              : st.optimize ? align256((int64_t)count * sizeof(FrameHuff)) : 0);
  return L;
}

// After the transform, a progressive group's ten scans: every launch runs all of them for every frame,
// its grid over (unit chunk, frame) or (interval block, frame).  p describes the units.
int launch_progressive(const JpegParams& p, const StuffParams& templ, int max_uchunks, int max_schunks,
                       int max_ints, int count, cudaStream_t stream) {
  const dim3 grid((unsigned)max_uchunks, (unsigned)count), sgrid((unsigned)max_schunks, (unsigned)count);
  prog_units_kernel<<<grid, kChunk, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg prog_units_kernel");
  JpegParams sums = p;                    // the tails' and then the symbol units' chunk sums
  for (int k = 0; k < 2; ++k) {
    for (int i = 0; i < count; ++i) sums.g[i].csum = p.g[i].tsum + k * (p.g[i].chunks + 1);
    scan_kernel<<<(unsigned)count, kScanThreads, 0, stream>>>(sums, kScanBlocks);
    SQ_CHECK_LAUNCH("jpeg scan_kernel");
  }
  prog_eobrun_kernel<<<grid, kChunk, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg prog_eobrun_kernel");
  prog_table_kernel<<<(unsigned)count, kSlots * 32, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg prog_table_kernel");
  prog_bits_kernel<<<grid, kChunk, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg prog_bits_kernel");
  scan_kernel<<<(unsigned)count, kScanThreads, 0, stream>>>(p, kScanBlocks);
  SQ_CHECK_LAUNCH("jpeg scan_kernel");
  prog_interval_kernel<<<dim3((unsigned)((max_ints + kChunk - 1) / kChunk), (unsigned)count), kChunk, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg prog_interval_kernel");
  scan_kernel<<<(unsigned)count, kScanThreads, 0, stream>>>(p, kScanIntervals);
  SQ_CHECK_LAUNCH("jpeg scan_kernel");
  prog_pack_kernel<<<grid, kChunk, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg prog_pack_kernel");
  count_ff_kernel<true><<<sgrid, kStuffThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg count_ff_kernel");
  scan_kernel<<<(unsigned)count, kScanThreads, 0, stream>>>(p, kScanStuffing);
  SQ_CHECK_LAUNCH("jpeg scan_kernel");
  StuffParams sp = templ;
  sp.p = p;
  stuff_kernel<false, true><<<sgrid, kStuffThreads, 0, stream>>>(sp);
  SQ_CHECK_LAUNCH("jpeg stuff_kernel");
  return SQDET_OK;
}

template <int F, int HS, int VS>
void launch_transform(const dim3& grid, const TransformParams<F>& tp, cudaStream_t stream) {
  transform_kernel<F, HS, VS><<<grid, kChunk, 0, stream>>>(tp);
}

template <int F>
int launch_group(const PixFormat& pf, const FrameSource* fr, int first, int count, const Settings& st,
                 const QuantRecip& quant, const StuffParams& templ, uint8_t* out, int64_t cap,
                 int64_t* lengths, uint8_t* scratch, cudaStream_t stream) {
  TransformParams<F> tp;
  JpegParams& p = tp.p;
  const GroupLayout L = group_layout(fr, first, count, st, p.g);
  int max_chunks = 0, max_schunks = 0, max_ints = 0;
  for (int i = 0; i < count; ++i) {
    p.g[i].out = out + (int64_t)(first + i) * cap;
    p.g[i].length = lengths + first + i;
    tp.f[i] = frame_desc<kPlanes<F>>(pf, fr[first + i], fr[first + i].h, fr[first + i].w);
    max_chunks = std::max(max_chunks, p.g[i].chunks);
    max_schunks = std::max(max_schunks, p.g[i].schunks);
    max_ints = std::max(max_ints, p.g[i].ints);
  }
  p.coef = reinterpret_cast<int16_t*>(scratch + L.coef);
  p.bits = reinterpret_cast<uint32_t*>(scratch + L.bits);
  p.sums = reinterpret_cast<int64_t*>(scratch + L.sums);
  p.ipos = reinterpret_cast<int64_t*>(scratch + L.ipos);
  p.stream = reinterpret_cast<uint32_t*>(scratch + L.stream);
  p.freq = reinterpret_cast<unsigned long long*>(scratch + L.freq);
  p.huff = reinterpret_cast<FrameHuff*>(scratch + L.huff);
  p.flags = reinterpret_cast<uint32_t*>(scratch + L.flags);
  p.pre = reinterpret_cast<uint32_t*>(scratch + L.pre);
  p.flush = reinterpret_cast<uint32_t*>(scratch + L.flush);
  p.phuff = reinterpret_cast<ProgHuff*>(scratch + L.huff);
  p.cap = cap;
  p.hs = st.hs;
  p.vs = st.vs;
  p.luma = st.hs * st.vs;
  p.per = p.luma + 2;
  p.rst = st.rst;
  tp.quant = quant;
  // progressive: p describes the units and tp.p the blocks the transform writes
  const JpegParams up = p;
  const int max_uchunks = max_chunks;
  if (st.prog) {
    max_chunks = 0;
    for (int i = 0; i < count; ++i) {
      const FrameSizes z = frame_sizes(p.g[i].h, p.g[i].w, st);
      p.g[i].blk = p.g[i].cblk;
      p.g[i].blocks = z.blocks;
      p.g[i].chunks = z.chunks;
      max_chunks = std::max(max_chunks, z.chunks);
    }
  }
  // the bit buffers, the symbol counts and (progressive) the flush words
  SQ_CUDA(cudaMemsetAsync(scratch + L.flush, 0, (size_t)(L.huff - L.flush), stream));
  const dim3 grid((unsigned)max_chunks, (unsigned)count), sgrid((unsigned)max_schunks, (unsigned)count);
  switch (st.hs * 16 + st.vs) {
    case 0x41: launch_transform<F, 4, 1>(grid, tp, stream); break;
    case 0x21: launch_transform<F, 2, 1>(grid, tp, stream); break;
    case 0x12: launch_transform<F, 1, 2>(grid, tp, stream); break;
    case 0x11: launch_transform<F, 1, 1>(grid, tp, stream); break;
    default: launch_transform<F, 2, 2>(grid, tp, stream);
  }
  SQ_CHECK_LAUNCH("jpeg transform_kernel");
  if (st.prog) return launch_progressive(up, templ, max_uchunks, max_schunks, max_ints, count, stream);
  if (st.optimize) {
    hist_kernel<<<grid, kChunk, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg hist_kernel");
    table_kernel<<<(unsigned)count, kTableThreads, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg table_kernel");
    block_bits_kernel<true><<<grid, kChunk, 0, stream>>>(p);
  } else {
    block_bits_kernel<false><<<grid, kChunk, 0, stream>>>(p);
  }
  SQ_CHECK_LAUNCH("jpeg block_bits_kernel");
  scan_kernel<<<(unsigned)count, kScanThreads, 0, stream>>>(p, kScanBlocks);
  SQ_CHECK_LAUNCH("jpeg scan_kernel");
  if (st.rst) {
    interval_kernel<<<dim3((unsigned)((max_ints + kChunk - 1) / kChunk), (unsigned)count), kChunk, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg interval_kernel");
    scan_kernel<<<(unsigned)count, kScanThreads, 0, stream>>>(p, kScanIntervals);
    SQ_CHECK_LAUNCH("jpeg scan_kernel");
  }
  if (st.optimize) pack_kernel<true><<<grid, kChunk, 0, stream>>>(p);
  else pack_kernel<false><<<grid, kChunk, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg pack_kernel");
  count_ff_kernel<false><<<sgrid, kStuffThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg count_ff_kernel");
  scan_kernel<<<(unsigned)count, kScanThreads, 0, stream>>>(p, kScanStuffing);
  SQ_CHECK_LAUNCH("jpeg scan_kernel");
  StuffParams sp = templ;
  sp.p = p;
  if (st.optimize) stuff_kernel<true><<<sgrid, kStuffThreads, 0, stream>>>(sp);
  else stuff_kernel<false><<<sgrid, kStuffThreads, 0, stream>>>(sp);
  SQ_CHECK_LAUNCH("jpeg stuff_kernel");
  return SQDET_OK;
}

// The largest progressive header and scan preambles: SOI .. SOF2, ten DHT segments of at most 256
// symbols (two before scan 0, one before each AC scan), two SOS of three components and eight of
// one.
constexpr int kProgHeaderBytes = kPrefixBytes + kScans * (21 + 256) + 2 * kSosBytes + 8 * (kSosBytes - 4);

// The largest file of an h x w crop.
int64_t jpeg_max_bytes(int h, int w, const Settings& st) {
  const FrameSizes s = frame_sizes(h, w, st);
  // progressive: the headers, every scan's longest units with every interval padded, every byte
  // stuffed, RSTn between the intervals of a scan, EOI
  if (st.prog)
    return kProgHeaderBytes + (st.rst ? kDriBytes : 0) + 2 * s.bytes + 2 * (int64_t)(s.ints - kScans) + 2;
  // the header (optimized tables are no longer than Annex K's), the stream with every byte
  // stuffed, RSTn between intervals, EOI
  return kHeaderBytes + (st.rst ? kDriBytes : 0) + 2 * s.bytes + 2 * (int64_t)(s.ints - 1) + 2;
}

// The scratch the encode of the crops of `frames` needs.
int64_t jpeg_scratch_bytes(const FrameSource* frames, int n, const Settings& st) {
  int64_t most = 0;
  for_each_group(n, [&](int first, int count) {
    most = std::max(most, group_layout(frames, first, count, st, nullptr).total);
    return SQDET_OK;
  });
  return most;
}

// The encode of the crops of `frames` in `format` (the frames' checks are the caller's).
int launch_encode_jpeg(int format, const PixFormat& pf, const FrameSource* frames, int n,
                       const Settings& st, uint8_t* out, int64_t cap, int64_t* lengths,
                       void* scratch, cudaStream_t stream) {
  // jpeg_quality_scaling of each table's quality, then the standard tables scaled, rounded and
  // clamped to 1..255
  const int scale[2] = {st.lq < 50 ? 5000 / st.lq : 200 - 2 * st.lq, st.cq < 50 ? 5000 / st.cq : 200 - 2 * st.cq};
  uint16_t q[2][64];
  QuantRecip quant;
  for (int i = 0; i < 64; ++i) {
    const uint8_t base[2] = {kStdLumaQ[i], kStdChromaQ[i]};
    for (int t = 0; t < 2; ++t) {
      const int v = std::min(std::max((base[t] * scale[t] + 50) / 100, 1), 255);
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
  StuffParams sp{};
  sp.std = std_spec();
  sp.suffix_bytes = jpeg_header(q, st, sp.prefix, sp.suffix);
  if (st.prog) prog_sos(sp.sos);
  uint8_t* s = static_cast<uint8_t*>(scratch);
  return for_each_group(n, [&](int first, int count) {
    return dispatch_format(format, [&](auto f) {
      return launch_group<decltype(f)::value>(pf, frames, first, count, st, quant, sp, out, cap,
                                              lengths, s, stream);
    });
  });
}

// sqdet_jpeg_params of cv2's defaults with `quality`.
sqdet_jpeg_params default_params(int quality) {
  return sqdet_jpeg_params{quality, -1, -1, 0x221111, 0, 0};
}

}  // namespace
}  // namespace sqdet

using namespace sqdet;

namespace sqdet {
namespace {

// The three entry points of baseline (prog 0) or progressive (prog 1) files.
int64_t max_bytes_entry(int h, int w, const sqdet_jpeg_params* params, int prog) {
  const std::string name = prog ? "sqdet_jpeg_max_bytes_progressive" : "sqdet_jpeg_max_bytes";
  Settings st;
  if (resolve_params(name, params, &st)) return -1;
  st.prog = prog;
  if (h < 1 || w < 1 || h > kJpegMaxSide || w > kJpegMaxSide) {
    fail(SQDET_ERR_INVALID_ARG, name + ": h and w must be in [1, 65500]");
    return -1;
  }
  return jpeg_max_bytes(h, w, st);
}

int64_t scratch_bytes_entry(int n, const int32_t* heights, const int32_t* widths, const int32_t* crops,
                            const sqdet_jpeg_params* params, int prog) {
  const Encoder& enc = prog ? kJpegProg : kJpeg;
  std::vector<FrameSource> fr;
  Settings st;
  if (resolve_params(enc.scratch_call, params, &st)) return -1;
  st.prog = prog;
  if (encode_crops(enc.scratch_call, enc, n, heights, widths, crops, fr)) return -1;
  return jpeg_scratch_bytes(fr.data(), n, st);
}

int encode_entry(int n, int format, const uint8_t* const* planes, const int64_t* pitches, const int32_t* heights,
                 const int32_t* widths, const int32_t* crops, const sqdet_jpeg_params* params, uint8_t* out_dev,
                 int64_t cap, int64_t* lengths_dev, void* scratch_dev, int64_t scratch_bytes, void* stream,
                 int prog) {
  const Encoder& enc = prog ? kJpegProg : kJpeg;
  Settings st;
  auto settle = [&](const std::vector<FrameSource>& fr, int64_t& need) {
    const int rc = resolve_params(enc.call, params, &st);
    st.prog = prog;
    if (!rc) need = jpeg_scratch_bytes(fr.data(), n, st);
    return rc;
  };
  auto launch = [&](const PixFormat& pf, const FrameSource* fr) {
    return launch_encode_jpeg(format, pf, fr, n, st, out_dev, cap, lengths_dev, scratch_dev,
                              (cudaStream_t)stream);
  };
  return encode_frames(enc, n, format, planes, pitches, heights, widths, crops, out_dev, cap,
                       lengths_dev, scratch_dev, scratch_bytes, settle, launch);
}

}  // namespace
}  // namespace sqdet

int64_t sqdet_jpeg_max_bytes_params(int h, int w, const sqdet_jpeg_params* params) {
  return max_bytes_entry(h, w, params, 0);
}

int64_t sqdet_jpeg_max_bytes_progressive(int h, int w, const sqdet_jpeg_params* params) {
  return max_bytes_entry(h, w, params, 1);
}

int64_t sqdet_jpeg_max_bytes(int h, int w) {
  const sqdet_jpeg_params d = default_params(kDefaultSettings.lq);
  return sqdet_jpeg_max_bytes_params(h, w, &d);
}

int64_t sqdet_jpeg_scratch_bytes_params(int n, const int32_t* heights, const int32_t* widths,
                                        const int32_t* crops, const sqdet_jpeg_params* params) {
  return scratch_bytes_entry(n, heights, widths, crops, params, 0);
}

int64_t sqdet_jpeg_scratch_bytes_progressive(int n, const int32_t* heights, const int32_t* widths,
                                             const int32_t* crops, const sqdet_jpeg_params* params) {
  return scratch_bytes_entry(n, heights, widths, crops, params, 1);
}

int64_t sqdet_jpeg_scratch_bytes(int n, const int32_t* heights, const int32_t* widths,
                                 const int32_t* crops) {
  const sqdet_jpeg_params d = default_params(kDefaultSettings.lq);
  return sqdet_jpeg_scratch_bytes_params(n, heights, widths, crops, &d);
}

int sqdet_encode_jpeg_params(int n, int format, const uint8_t* const* planes, const int64_t* pitches,
                             const int32_t* heights, const int32_t* widths, const int32_t* crops,
                             const sqdet_jpeg_params* params, uint8_t* out_dev, int64_t cap,
                             int64_t* lengths_dev, void* scratch_dev, int64_t scratch_bytes, void* stream) {
  return encode_entry(n, format, planes, pitches, heights, widths, crops, params, out_dev, cap, lengths_dev,
                      scratch_dev, scratch_bytes, stream, 0);
}

int sqdet_encode_jpeg_progressive(int n, int format, const uint8_t* const* planes, const int64_t* pitches,
                                  const int32_t* heights, const int32_t* widths, const int32_t* crops,
                                  const sqdet_jpeg_params* params, uint8_t* out_dev, int64_t cap,
                                  int64_t* lengths_dev, void* scratch_dev, int64_t scratch_bytes, void* stream) {
  return encode_entry(n, format, planes, pitches, heights, widths, crops, params, out_dev, cap, lengths_dev,
                      scratch_dev, scratch_bytes, stream, 1);
}

int sqdet_encode_jpeg(int n, int format, const uint8_t* const* planes, const int64_t* pitches,
                      const int32_t* heights, const int32_t* widths, const int32_t* crops,
                      int quality, uint8_t* out_dev, int64_t cap, int64_t* lengths_dev,
                      void* scratch_dev, int64_t scratch_bytes, void* stream) {
  const sqdet_jpeg_params d = default_params(quality);
  return sqdet_encode_jpeg_params(n, format, planes, pitches, heights, widths, crops, &d, out_dev, cap,
                                  lengths_dev, scratch_dev, scratch_bytes, stream);
}
