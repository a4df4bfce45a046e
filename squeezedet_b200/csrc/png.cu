// PNG encoding of uint8 frames in device memory (sqdet_encode_png): frame i's crop, converted to BGR
// as its format's cv2.cvtColor code does, becomes the bytes cv2.imencode('.png', crop) writes, bit
// for bit.  That is libpng 1.6 over zlib 1.2.11 at cv2's defaults: 8-bit RGB, the SUB filter on
// every row (NONE for a 1-pixel-wide image), zlib level 1 with strategy Z_RLE, 8192-byte IDATs.
// oracle/png.py restates it in numpy and documents the format.
//
// Z_RLE makes deflate's parse a closed-form function of the runs of equal bytes: in a run of L
// bytes, one literal, then matches of distance 1 and length min(258, bytes left) while 3 or more
// bytes are left, then literals.  So every stage is a map, a scan or a per-block reduction:
//   1. filter       one thread per pixel fetches it and its left neighbour (frames.cuh) and writes
//                   the filtered R, G, B bytes; the row's first thread writes its filter byte
//   2. mark         per segment of kSegBytes filtered bytes: the last run start in it, and its
//                   terms of the Adler-32 sums
//   3. scan (max)   per frame: the run start in force at each segment's first byte
//   4. count        per segment: the symbols that start in it (each byte knows its run offset from
//                   the run start and the bytes left in its run from a look-ahead of <= 258)
//   5. scan (sum)   per frame: each segment's first symbol index
//   6. emit         each symbol, as its byte or 256 + length - 3, at its index; the first symbol of
//                   each deflate block (16383 symbols) records its byte position
//   7. tree         one CTA per deflate block: the histogram, then one thread builds zlib's trees,
//                   compares the stored, static and dynamic sizes as _tr_flush_block does and keeps
//                   the chosen codes
//   8. frame        one CTA per frame: the Adler-32, then one thread walks the blocks for their bit
//                   positions (a stored block's padding depends on where it starts), the zlib header
//                   and trailer, and the file's length (-1 when it does not fit)
//   9. pack         one CTA per deflate block: a scan of its symbols' code lengths, then the codes
//                   ORed into the frame's zeroed bit buffer (LSB first, 32-bit atomicOr, so that
//                   blocks share only edge words); stored blocks copy their bytes
//  10. idat         one CTA per IDAT chunk: its bytes and CRC-32 (per-thread CRCs of 32-byte
//                   pieces combined by multiplication with x^(8 n) mod P); the first CTA writes the
//                   signature and IHDR, the last IEND
// Frames run kEncodeFramesPerLaunch at a time through these launches, reusing one scratch.
#include "frames.cuh"
#include "scan.cuh"

namespace sqdet {
namespace {

constexpr int kSegThreads = 256;
constexpr int kSegBytesPerThread = 16;
constexpr int kSegBytes = kSegThreads * kSegBytesPerThread;   // filtered bytes per segment
constexpr int kFilterThreads = 256;
constexpr int kFilterPixels = kFilterThreads * 4;               // pixels per filter CTA
constexpr int kBlockSymbols = 16383;    // zlib's lit_bufsize - 1 at memLevel 8
// tree_kernel: after the histogram one thread builds the trees, so a CTA is small and many run per SM
constexpr int kTreeThreads = 64;
constexpr int kPackThreads = 1024;      // kPackThreads * 16 >= kBlockSymbols
constexpr int kPackPerThread = 16;
constexpr int kIdatBytes = 8192;        // libpng's zbuffer: the IDAT data size
constexpr int kIdatThreads = 256;
constexpr int kCrcPiece = 32;           // bytes per thread of a chunk's CRC
constexpr int kFrameThreads = 1024;
constexpr int kPngMaxSide = 1000000;    // libpng's PNG_USER_WIDTH_MAX / PNG_USER_HEIGHT_MAX
constexpr Encoder kPng = {"sqdet_encode_png", "PNG", "sqdet_png_scratch_bytes", 128, kPngMaxSide};
constexpr int kLCodes = 286, kDCodes = 30, kBlCodes = 19, kEndBlock = 256;
constexpr int kHeapSize = 2 * kLCodes + 1;
constexpr int kFixedBytes = 8 + 25 + 12;  // signature, IHDR, IEND
enum { kStored = 0, kStatic = 1, kDynamic = 2 };

// ---- deflate tables ----------------------------------------------------------------------------
__constant__ uint8_t kExtraLBits[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2,
                                         2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint8_t kBaseLength[29] = {0,  1,  2,  3,  4,  5,  6,   7,   8,   10,  12,  14,  16, 20, 24,
                                         28, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 255};
__constant__ uint8_t kExtraBlBits[kBlCodes] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 3, 7};
__constant__ uint8_t kBlOrder[kBlCodes] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// The length code (0..28) of match length lc + 3: codes 4 k .. 4 k + 3 (k >= 2) cover lc of
// k + 1 significant bits in steps of 2^(k - 1), and 258 has its own.
__device__ __forceinline__ int length_code(int lc) {
  if (lc < 8) return lc;
  if (lc == 255) return 28;
  const int nb = 31 - __clz(lc);
  return 4 * (nb - 1) + ((lc >> (nb - 2)) & 3);
}

__host__ __device__ constexpr int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }
// The static literal/length code of n (not bit-reversed).  Its canonical order counts all 288
// symbols of the static tree, 286 and 287 included, so the codes are written out rather than
// rebuilt from the 286 lengths.
__device__ __forceinline__ uint32_t static_lcode(int n) {
  return n < 144 ? 0x30 + n : n < 256 ? 0x190 + n - 144 : n < 280 ? n - 256 : 0xC0 + n - 280;
}

__device__ __forceinline__ uint32_t bit_reverse(uint32_t code, int len) { return __brev(code) >> (32 - len); }

// ---- CRC-32 (reflected, polynomial 0xEDB88320) -------------------------------------------------
constexpr uint32_t kCrcPoly = 0xEDB88320u;
// a * b mod P, polynomials in the reflected representation (x^0 at bit 31)
__host__ __device__ constexpr uint32_t mult_mod_p(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (uint32_t m = 1u << 31; m; m >>= 1) {
    if (a & m) p ^= b;
    b = b & 1 ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return p;
}
// x^(2^k) mod P, k = 0..31
struct X2n {
  uint32_t t[32];
};
constexpr X2n x2n_table() {
  X2n x{};
  uint32_t p = 1u << 30;                // x^1
  x.t[0] = p;
  for (int k = 1; k < 32; ++k) x.t[k] = p = mult_mod_p(p, p);
  return x;
}
__constant__ X2n kX2n = x2n_table();
// x^(8 n) mod P
__device__ uint32_t x8n_mod_p(int64_t n) {
  uint32_t p = 1u << 31;                // x^0
  for (int k = 3; n; n >>= 1, ++k)
    if (n & 1) p = mult_mod_p(kX2n.t[k & 31], p);
  return p;
}
__host__ __device__ constexpr uint32_t crc_byte(uint32_t c) {
  for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ kCrcPoly : c >> 1;
  return c;
}

// ---- per-frame geometry and scratch ---------------------------------------------------------------
// One frame of a launch group: its crop, filtered stream of n bytes and where its pieces of the
// scratch and output are.  Per-segment values start at seg (segs of them, then one slot the scans
// fill with the total), deflate blocks at blk (at most max_blocks), stream words at words.
struct PngGeom {
  int h, w, segs, max_blocks, max_chunks;
  int64_t n;                            // filtered bytes: h (3 w + 1)
  int64_t data, seg, blk, words;        // offsets: filtered bytes, segment slots, blocks, words
  uint8_t* out;
  int64_t* length;
};

// A deflate block: the filtered bytes [start, end) its symbols cover, its kind, its size in bits
// (static and dynamic), the bits before its first symbol, its stream position, and its codes
// (bit-reversed, literal/length then distance) and the bit-length tree of a dynamic block.
struct DBlock {
  int64_t start, end, bits, pos;
  int32_t kind, head_bits;
  int16_t lmax, dmax, max_blindex, pad_;
  uint16_t code[kLCodes + kDCodes];
  uint8_t len[kLCodes + kDCodes];
  uint16_t bl_code[kBlCodes];
  uint8_t bl_len[kBlCodes];
};

// Per frame, written by the frame pass.
struct FrameRec {
  int64_t symbols, blocks, zbytes, size;
};

struct PngParams {
  PngGeom g[kEncodeFramesPerLaunch];
  uint8_t* data;                        // filtered streams
  int64_t* brk;                         // per segment: last run start, then the scanned run starts
  int64_t* cnt;                         // per segment: symbols, then the scanned first indices
  int64_t* adler;                       // per segment: two Adler-32 partial sums
  uint16_t* sym;                        // symbols
  DBlock* blocks;
  FrameRec* rec;                        // [count]
  uint32_t* stream;                     // zlib streams, 32-bit little-endian words
  int64_t cap;
};

template <int F>
struct FilterParams {
  PngParams p;
  FrameDesc<kPlanes<F>> f[kEncodeFramesPerLaunch];
};
static_assert(sizeof(FilterParams<SQDET_FMT_I420>) <= 4096, "filter parameters exceed 4 KiB");

// ---- 1. filter ------------------------------------------------------------------------------------
template <int F>
__global__ void __launch_bounds__(kFilterThreads) filter_kernel(const __grid_constant__ FilterParams<F> fp) {
  const PngGeom& g = fp.p.g[blockIdx.y];
  const auto taps_ = taps<F>(fp.f[blockIdx.y]);
  uint8_t* d = fp.p.data + g.data;
  const int64_t row = 3 * (int64_t)g.w + 1;
#pragma unroll 1
  for (int k = 0; k < kFilterPixels / kFilterThreads; ++k) {
    const int64_t i = (int64_t)blockIdx.x * kFilterPixels + k * kFilterThreads + threadIdx.x;
    if (i >= (int64_t)g.h * g.w) return;
    const int y = (int)(i / g.w), x = (int)(i % g.w);
    int b, gr, r, pb = 0, pg = 0, pr = 0;
    fetch_bgr(taps_, y, x, b, gr, r);
    if (x > 0) fetch_bgr(taps_, y, x - 1, pb, pg, pr);
    uint8_t* o = d + y * row + 1 + 3 * (int64_t)x;
    o[0] = (uint8_t)(r - pr);
    o[1] = (uint8_t)(gr - pg);
    o[2] = (uint8_t)(b - pb);
    if (x == 0) o[-1] = g.w > 1 ? 1 : 0;   // SUB; libpng writes NONE when a row is one pixel
  }
}

// ---- 2. run starts and Adler-32 terms per segment -------------------------------------------------
// The thread's bytes [p0, p0 + 16) of the segment (clipped to n) and the byte before them.
struct Bytes16 {
  uint8_t v[kSegBytesPerThread];
  int prev;                             // byte p0 - 1, or -1 at p0 = 0
  int count;
  int64_t p0;
};
__device__ __forceinline__ Bytes16 load16(const uint8_t* d, int64_t n, int64_t p0) {
  Bytes16 b;
  b.p0 = p0;
  b.count = (int)max((int64_t)0, min((int64_t)kSegBytesPerThread, n - p0));
  b.prev = p0 > 0 && p0 <= n ? d[p0 - 1] : -1;
#pragma unroll
  for (int i = 0; i < kSegBytesPerThread; ++i) b.v[i] = i < b.count ? d[p0 + i] : 0;
  return b;
}
// The last position in b that starts a run (its byte differs from the one before), or -1.
__device__ __forceinline__ int64_t last_run_start(const Bytes16& b) {
  int64_t last = -1;
#pragma unroll
  for (int i = 0; i < kSegBytesPerThread; ++i) {
    const int before = i ? b.v[i - 1] : b.prev;
    if (i < b.count && (int)b.v[i] != before) last = b.p0 + i;
  }
  return last;
}

__global__ void __launch_bounds__(kSegThreads) mark_kernel(const __grid_constant__ PngParams p) {
  __shared__ int64_t warp[32];
  const PngGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.segs) return;
  const uint8_t* d = p.data + g.data;
  const Bytes16 b = load16(d, g.n, (int64_t)blockIdx.x * kSegBytes + threadIdx.x * kSegBytesPerThread);
  // Adler-32: a = 1 + sum d_p, b = n + sum (n - p) d_p, mod 65521
  uint64_t s1 = 0, s2 = 0;
  uint32_t wgt = (uint32_t)((g.n - b.p0) % 65521);
#pragma unroll
  for (int i = 0; i < kSegBytesPerThread; ++i) {
    if (i < b.count) {
      s1 += b.v[i];
      s2 += (uint64_t)wgt * b.v[i];
      wgt = wgt ? wgt - 1 : 65520;
    }
  }
  int64_t total;
  block_exclusive_scan(last_run_start(b), warp, &total, ScanMax());
  if (threadIdx.x == 0) p.brk[g.seg + blockIdx.x] = total;
  int64_t t1, t2;
  block_exclusive_scan((int64_t)(s1 % 65521), warp, &t1);
  block_exclusive_scan((int64_t)(s2 % 65521), warp, &t2);
  if (threadIdx.x == 0) {
    p.adler[2 * (g.seg + blockIdx.x)] = t1 % 65521;
    p.adler[2 * (g.seg + blockIdx.x) + 1] = t2 % 65521;
  }
}

// ---- 3, 5. per-frame exclusive scans of segment values ------------------------------------------
// Frame blockIdx.x's segs values from v[seg] become their exclusive scan (max: the run start in
// force at each segment's first byte; sum: its first symbol's index), the slot after them the total.
template <class Op>
__global__ void __launch_bounds__(1024) seg_scan_kernel(const __grid_constant__ PngParams p, int64_t* v) {
  __shared__ int64_t warp[32];
  const PngGeom& g = p.g[blockIdx.x];
  int64_t* s = v + g.seg;
  int64_t carry = Op::kIdentity;
  for (int base = 0; base < g.segs; base += 1024) {
    const int i = base + threadIdx.x;
    const int64_t x = i < g.segs ? s[i] : Op::kIdentity;
    int64_t total;
    const int64_t ex = block_exclusive_scan(x, warp, &total, Op());
    if (i < g.segs) s[i] = Op()(carry, ex);
    carry = Op()(carry, total);
  }
  if (threadIdx.x == 0) s[g.segs] = carry;
}

// ---- 4, 6. the symbols of each segment ------------------------------------------------------------
// Calls sym(position, length) for every symbol starting in the thread's 16 bytes, in order: length
// 1 for a literal, 3..258 for a distance-1 match.  A byte at offset o of its run with e bytes of the
// run left from it (e counted to 258) is a literal when o = 0 or e + q < 3, q = (o - 1) mod 258;
// otherwise it starts a match of min(e, 258) when q = 0 and lies inside one when not.
template <class Sym>
__device__ __forceinline__ void segment_symbols(const uint8_t* d, int64_t n, const Bytes16& b,
                                                int64_t run_start, Sym sym) {
  if (b.count == 0) return;
  int e[kSegBytesPerThread];
  {
    // the run left from the last byte: a look-ahead of at most 258 bytes
    const int64_t last = b.p0 + b.count - 1;
    const uint8_t v = d[last];
    int k = 1;
    while (k < 258 && last + k < n && d[last + k] == v) ++k;
    int run = k;
#pragma unroll
    for (int i = kSegBytesPerThread - 1; i >= 0; --i) {
      if (i < b.count) {
        if (i < b.count - 1) run = b.v[i] == b.v[i + 1] ? min(run + 1, 258) : 1;
        e[i] = run;
      }
    }
  }
  int64_t a = run_start;
#pragma unroll
  for (int i = 0; i < kSegBytesPerThread; ++i) {
    if (i < b.count) {
      const int64_t pos = b.p0 + i;
      const int before = i ? b.v[i - 1] : b.prev;
      if ((int)b.v[i] != before) a = pos;
      const int64_t o = pos - a;
      const int q = o > 0 ? (int)((o - 1) % 258) : 0;
      if (o == 0 || e[i] + q < 3) sym(pos, 1, b.v[i]);
      else if (q == 0) sym(pos, min(e[i], 258), b.v[i]);
    }
  }
}

// The run start in force at the thread's first byte: the segment's, then the threads' before it.
__device__ __forceinline__ int64_t thread_run_start(const PngParams& p, const PngGeom& g,
                                                    const Bytes16& b, int64_t* warp) {
  int64_t total;
  const int64_t before = block_exclusive_scan(last_run_start(b), warp, &total, ScanMax());
  return max(before, p.brk[g.seg + blockIdx.x]);
}

__global__ void __launch_bounds__(kSegThreads) count_kernel(const __grid_constant__ PngParams p) {
  __shared__ int64_t warp[32];
  const PngGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.segs) return;
  const uint8_t* d = p.data + g.data;
  const Bytes16 b = load16(d, g.n, (int64_t)blockIdx.x * kSegBytes + threadIdx.x * kSegBytesPerThread);
  const int64_t a = thread_run_start(p, g, b, warp);
  int count = 0;
  segment_symbols(d, g.n, b, a, [&](int64_t, int, int) { ++count; });
  int64_t total;
  block_exclusive_scan(count, warp, &total);
  if (threadIdx.x == 0) p.cnt[g.seg + blockIdx.x] = total;
}

__global__ void __launch_bounds__(kSegThreads) emit_kernel(const __grid_constant__ PngParams p) {
  __shared__ int64_t warp[32];
  const PngGeom& g = p.g[blockIdx.y];
  if ((int)blockIdx.x >= g.segs) return;
  const uint8_t* d = p.data + g.data;
  const Bytes16 b = load16(d, g.n, (int64_t)blockIdx.x * kSegBytes + threadIdx.x * kSegBytesPerThread);
  const int64_t a = thread_run_start(p, g, b, warp);
  int count = 0;
  segment_symbols(d, g.n, b, a, [&](int64_t, int, int) { ++count; });
  int64_t total;
  int64_t k = p.cnt[g.seg + blockIdx.x] + block_exclusive_scan(count, warp, &total);
  uint16_t* sym = p.sym + g.data;
  DBlock* blocks = p.blocks + g.blk;
  segment_symbols(d, g.n, b, a, [&](int64_t pos, int len, int v) {
    sym[k] = (uint16_t)(len == 1 ? v : 256 + len - 3);
    if (k % kBlockSymbols == 0) blocks[k / kBlockSymbols].start = pos;
    ++k;
  });
}

// ---- 7. trees ---------------------------------------------------------------------------------------
// zlib's build_tree + gen_bitlen over freq[0..elems), in the CTA's shared arrays, one thread.  Leaves
// get their code lengths in len[] (0 for an absent symbol); freq of forced codes becomes 1.
struct TreeWork {
  uint32_t freq[kHeapSize];
  int16_t heap[kHeapSize + 1];
  int16_t dad[kHeapSize];
  uint8_t depth[kHeapSize];
  uint8_t len[kHeapSize];
  int bl_count[16], next_code[16];
};

__device__ __forceinline__ bool smaller(const TreeWork& t, int n, int m) {
  return t.freq[n] < t.freq[m] || (t.freq[n] == t.freq[m] && t.depth[n] <= t.depth[m]);
}
__device__ __forceinline__ void pq_down(TreeWork& t, int heap_len, int k) {
  const int v = t.heap[k];
  int j = k << 1;
  while (j <= heap_len) {
    if (j < heap_len && smaller(t, t.heap[j + 1], t.heap[j])) ++j;
    if (smaller(t, v, t.heap[j])) break;
    t.heap[k] = t.heap[j];
    k = j;
    j <<= 1;
  }
  t.heap[k] = (int16_t)v;
}

// -> max_code; adds the tree's cost to *opt and, with a static tree (static_len), to *stat.
// extra(n): the extra bits of symbol n.
template <class StaticLen, class Extra>
__device__ __forceinline__ int build_tree(TreeWork& t, int elems, int max_length, bool has_static, StaticLen static_len,
                          Extra extra, int64_t* opt, int64_t* stat) {
  int heap_len = 0, heap_max = kHeapSize, max_code = -1;
  for (int n = 0; n < elems; ++n) {
    if (t.freq[n]) {
      t.heap[++heap_len] = (int16_t)n;
      max_code = n;
      t.depth[n] = 0;
    }
  }
  while (heap_len < 2) {
    const int node = max_code < 2 ? ++max_code : 0;
    t.heap[++heap_len] = (int16_t)node;
    t.freq[node] = 1;
    t.depth[node] = 0;
    --*opt;
    if (has_static) *stat -= static_len(node);
  }
  for (int k = heap_len / 2; k >= 1; --k) pq_down(t, heap_len, k);
  int node = elems;
  do {
    const int n = t.heap[1];
    t.heap[1] = t.heap[heap_len--];
    pq_down(t, heap_len, 1);
    const int m = t.heap[1];
    t.heap[--heap_max] = (int16_t)n;
    t.heap[--heap_max] = (int16_t)m;
    t.freq[node] = t.freq[n] + t.freq[m];
    t.depth[node] = (uint8_t)(max(t.depth[n], t.depth[m]) + 1);
    t.dad[n] = t.dad[m] = (int16_t)node;
    t.heap[1] = (int16_t)node++;
    pq_down(t, heap_len, 1);
  } while (heap_len >= 2);
  t.heap[--heap_max] = t.heap[1];

  // gen_bitlen
  for (int b = 0; b < 16; ++b) t.bl_count[b] = 0;
  t.len[t.heap[heap_max]] = 0;
  int overflow = 0, h;
  for (h = heap_max + 1; h < kHeapSize; ++h) {
    const int n = t.heap[h];
    int bits = t.len[t.dad[n]] + 1;
    if (bits > max_length) {
      bits = max_length;
      ++overflow;
    }
    t.len[n] = (uint8_t)bits;
    if (n > max_code) continue;
    t.bl_count[bits]++;
    const int xb = extra(n);
    *opt += (int64_t)t.freq[n] * (bits + xb);
    if (has_static) *stat += (int64_t)t.freq[n] * (static_len(n) + xb);
  }
  if (overflow) {
    do {
      int bits = max_length - 1;
      while (t.bl_count[bits] == 0) --bits;
      t.bl_count[bits]--;
      t.bl_count[bits + 1] += 2;
      t.bl_count[max_length]--;
      overflow -= 2;
    } while (overflow > 0);
    for (int bits = max_length; bits != 0; --bits) {
      int k = t.bl_count[bits];
      while (k != 0) {
        const int m = t.heap[--h];
        if (m > max_code) continue;
        if (t.len[m] != bits) {
          *opt += ((int64_t)bits - t.len[m]) * t.freq[m];
          t.len[m] = (uint8_t)bits;
        }
        --k;
      }
    }
  }
  for (int n = 0; n < elems; ++n)
    if (n > max_code || t.freq[n] == 0) t.len[n] = 0;
  return max_code;
}

// gen_codes: bit-reversed canonical codes of len[0..count) into code[] (t's counts as work space).
__device__ __forceinline__ void gen_codes(TreeWork& t, const uint8_t* len, int count, uint16_t* code) {
  for (int b = 0; b < 16; ++b) t.bl_count[b] = 0;
  for (int n = 0; n < count; ++n) t.bl_count[len[n]]++;
  t.bl_count[0] = 0;
  int c = 0;
  for (int bits = 1; bits <= 15; ++bits) {
    c = (c + t.bl_count[bits - 1]) << 1;
    t.next_code[bits] = c;
  }
  for (int n = 0; n < count; ++n)
    code[n] = len[n] ? (uint16_t)bit_reverse((uint32_t)t.next_code[len[n]]++, len[n]) : 0;
}

// scan_tree / send_tree: calls put(bl symbol, extra value, extra bits) for the run-length coding of
// len[0..max_code].
template <class Put>
__device__ __forceinline__ void tree_runs(const uint8_t* len, int max_code, Put put) {
  int prevlen = -1, nextlen = len[0], count = 0;
  int max_count = nextlen == 0 ? 138 : 7, min_count = nextlen == 0 ? 3 : 4;
  for (int n = 0; n <= max_code; ++n) {
    const int curlen = nextlen;
    nextlen = n + 1 <= max_code ? len[n + 1] : -1;
    if (++count < max_count && curlen == nextlen) continue;
    if (count < min_count) {
      for (int k = 0; k < count; ++k) put(curlen, 0, 0);
    } else if (curlen != 0) {
      if (curlen != prevlen) {
        put(curlen, 0, 0);
        --count;
      }
      put(16, count - 3, 2);
    } else if (count <= 10) {
      put(17, count - 3, 3);
    } else {
      put(18, count - 11, 7);
    }
    count = 0;
    prevlen = curlen;
    if (nextlen == 0) {
      max_count = 138;
      min_count = 3;
    } else if (curlen == nextlen) {
      max_count = 6;
      min_count = 3;
    } else {
      max_count = 7;
      min_count = 4;
    }
  }
}

__global__ void __launch_bounds__(kTreeThreads, 8) tree_kernel(const __grid_constant__ PngParams p) {
  __shared__ TreeWork t;
  __shared__ uint32_t lfreq[kLCodes];
  __shared__ uint32_t matches;
  __shared__ uint8_t llen[kLCodes], dlen[kDCodes];
  const PngGeom& g = p.g[blockIdx.y];
  const int64_t nsym = p.cnt[g.seg + g.segs];
  const int64_t nblocks = nsym / kBlockSymbols + 1;
  const int b = blockIdx.x;
  if (b >= nblocks) return;
  for (int i = threadIdx.x; i < kLCodes; i += blockDim.x) lfreq[i] = 0;
  if (threadIdx.x == 0) matches = 0;
  __syncthreads();
  const int64_t s0 = (int64_t)b * kBlockSymbols, s1 = min(s0 + kBlockSymbols, nsym);
  const uint16_t* sym = p.sym + g.data;
  for (int64_t k = s0 + threadIdx.x; k < s1; k += blockDim.x) {
    const int s = sym[k];
    if (s < 256) {
      atomicAdd(&lfreq[s], 1u);
    } else {
      atomicAdd(&lfreq[257 + length_code(s - 256)], 1u);
      atomicAdd(&matches, 1u);
    }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  DBlock& blk = p.blocks[g.blk + b];
  // the start of an empty final block is no symbol's, so emit_kernel did not write it
  const int64_t start = s0 < nsym ? blk.start : g.n;
  const int64_t end = s0 + kBlockSymbols < nsym ? p.blocks[g.blk + b + 1].start : g.n;
  if (s0 >= nsym) blk.start = start;
  lfreq[kEndBlock] = 1;
  int64_t opt = 0, stat = 0;
  // literal/length tree
  for (int n = 0; n < kLCodes; ++n) t.freq[n] = lfreq[n];
  const int lmax = build_tree(
      t, kLCodes, 15, true, [](int n) { return static_llen(n); },
      [](int n) { return n >= 257 ? (int)kExtraLBits[n - 257] : 0; }, &opt, &stat);
  for (int n = 0; n < kLCodes; ++n) llen[n] = t.len[n];
  // distance tree: only distance 1 (code 0, no extra bits) occurs
  for (int n = 0; n < kDCodes; ++n) t.freq[n] = n == 0 ? matches : 0;
  const int dmax = build_tree(
      t, kDCodes, 15, true, [](int) { return 5; }, [](int) { return 0; }, &opt, &stat);
  for (int n = 0; n < kDCodes; ++n) dlen[n] = t.len[n];
  // bit-length tree
  for (int n = 0; n < kBlCodes; ++n) t.freq[n] = 0;
  auto count_bl = [&](int s, int, int) { t.freq[s]++; };
  tree_runs(llen, lmax, count_bl);
  tree_runs(dlen, dmax, count_bl);
  build_tree(
      t, kBlCodes, 7, false, [](int) { return 0; },
      [](int n) { return (int)kExtraBlBits[n]; }, &opt, &stat);
  int max_blindex = kBlCodes - 1;
  while (max_blindex >= 3 && t.len[kBlOrder[max_blindex]] == 0) --max_blindex;
  const int64_t tree_bits = 14 + 3 * (max_blindex + 1);
  opt += tree_bits;
  // _tr_flush_block's choice
  const int64_t stored_len = end - start;
  const int64_t static_lenb = (stat + 3 + 7) >> 3;
  const int64_t opt_lenb = min((opt + 3 + 7) >> 3, static_lenb);
  blk.end = end;
  blk.lmax = (int16_t)lmax;
  blk.dmax = (int16_t)dmax;
  blk.max_blindex = (int16_t)max_blindex;
  if (stored_len + 4 <= opt_lenb) {
    blk.kind = kStored;
    blk.bits = -1;
    blk.head_bits = 3;
    return;
  }
  if (static_lenb == opt_lenb) {
    blk.kind = kStatic;
    blk.bits = 3 + stat;
    blk.head_bits = 3;
    for (int n = 0; n < kLCodes; ++n) llen[n] = (uint8_t)static_llen(n);
    for (int n = 0; n < kDCodes; ++n) dlen[n] = 5;
  } else {
    blk.kind = kDynamic;
    blk.bits = 3 + opt;
    // the header: 3 + 14 bits, 3 per bit-length code, then the coded lengths
    int64_t head = 3 + tree_bits;
    auto head_bits = [&](int s, int, int xb) { head += t.len[s] + xb; };
    tree_runs(llen, lmax, head_bits);
    tree_runs(dlen, dmax, head_bits);
    blk.head_bits = (int32_t)head;
    for (int n = 0; n < kBlCodes; ++n) blk.bl_len[n] = t.len[n];
    gen_codes(t, blk.bl_len, kBlCodes, blk.bl_code);
  }
  for (int n = 0; n < kLCodes; ++n) blk.len[n] = llen[n];
  for (int n = 0; n < kDCodes; ++n) blk.len[kLCodes + n] = dlen[n];
  if (blk.kind == kStatic) {
    for (int n = 0; n < kLCodes; ++n) blk.code[n] = (uint16_t)bit_reverse(static_lcode(n), llen[n]);
    for (int n = 0; n < kDCodes; ++n) blk.code[kLCodes + n] = (uint16_t)bit_reverse((uint32_t)n, 5);
  } else {
    gen_codes(t, blk.len, kLCodes, blk.code);
    gen_codes(t, blk.len + kLCodes, kDCodes, blk.code + kLCodes);
  }
}

// ---- bit writer --------------------------------------------------------------------------------------
// Bits LSB first into 32-bit little-endian words (stream bit j is bit j & 31 of word j >> 5), ORed in.
struct BitWriter {
  uint32_t* word;
  uint64_t acc;
  int n;                                // pending bits in acc, including the leading offset
  __device__ BitWriter(uint32_t* words, int64_t pos) : word(words + (pos >> 5)), acc(0), n((int)(pos & 31)) {}
  __device__ void put(uint32_t v, int len) {
    acc |= (uint64_t)v << n;
    n += len;
    if (n >= 32) {
      atomicOr(word++, (uint32_t)acc);
      acc >>= 32;
      n -= 32;
    }
  }
  __device__ void flush() {
    if (n > 0) atomicOr(word, (uint32_t)acc);
  }
};

__device__ __forceinline__ void put_byte(uint32_t* words, int64_t j, uint32_t v) {
  atomicOr(words + (j >> 2), v << (8 * (j & 3)));
}
__device__ __forceinline__ uint8_t get_byte(const uint32_t* words, int64_t j) {
  return (uint8_t)(words[j >> 2] >> (8 * (j & 3)));
}

// ---- 8. per-frame pass ----------------------------------------------------------------------------
// The zlib header libpng leaves for n bytes of image data (oracle.png.zlib_header).
__device__ uint32_t zlib_header(int64_t n) {
  int wbits = 15;
  if (n <= 16384) {
    int64_t half = 1 << 14;
    while (n + 262 <= half) {
      half >>= 1;
      --wbits;
    }
  }
  wbits = max(wbits, 9);
  uint32_t cmf = 8 | ((wbits - 8) << 4);
  uint32_t flg = 31 - (cmf << 8) % 31;
  if (n <= 16384) {                     // libpng's optimize_cmf
    int cinfo = (int)(cmf >> 4);
    int64_t half = (int64_t)1 << (cinfo + 7);
    if (n <= half) {
      do {
        half >>= 1;
        --cinfo;
      } while (cinfo > 0 && n <= half);
      cmf = 8 | (cinfo << 4);
      flg = (flg & 0xe0) + 31 - ((cmf << 8) + (flg & 0xe0)) % 31;
    }
  }
  return cmf | (flg << 8);
}

__global__ void __launch_bounds__(kFrameThreads) frame_kernel(const __grid_constant__ PngParams p) {
  __shared__ int64_t warp[32];
  const PngGeom& g = p.g[blockIdx.x];
  int64_t a1 = 0, a2 = 0;
  for (int i = threadIdx.x; i < g.segs; i += kFrameThreads) {
    a1 += p.adler[2 * (g.seg + i)];
    a2 += p.adler[2 * (g.seg + i) + 1];
  }
  int64_t t1, t2;
  block_exclusive_scan(a1 % 65521, warp, &t1);
  block_exclusive_scan(a2 % 65521, warp, &t2);
  if (threadIdx.x != 0) return;
  const uint32_t adler = (uint32_t)(((g.n % 65521 + t2) % 65521) << 16 | ((1 + t1) % 65521));
  const int64_t nsym = p.cnt[g.seg + g.segs];
  const int64_t nblocks = nsym / kBlockSymbols + 1;
  DBlock* blocks = p.blocks + g.blk;
  int64_t pos = 16;                     // after the zlib header
  for (int64_t b = 0; b < nblocks; ++b) {
    DBlock& d = blocks[b];
    d.pos = pos;
    if (d.kind == kStored) {
      pos += 3;
      pos += (-pos) & 7;
      pos += 32 + 8 * (d.end - d.start);
    } else {
      pos += d.bits;
    }
  }
  const int64_t body = (pos + 7) >> 3;
  const int64_t zbytes = body + 4;
  uint32_t* words = p.stream + g.words;
  const uint32_t head = zlib_header(g.n);
  put_byte(words, 0, head & 255);
  put_byte(words, 1, head >> 8);
  for (int k = 0; k < 4; ++k) put_byte(words, body + k, (adler >> (24 - 8 * k)) & 255);
  const int64_t chunks = (zbytes + kIdatBytes - 1) / kIdatBytes;
  const int64_t size = kFixedBytes + 12 * chunks + zbytes;
  FrameRec& r = p.rec[blockIdx.x];
  r.symbols = nsym;
  r.blocks = nblocks;
  r.zbytes = zbytes;
  r.size = size;
  *g.length = size <= p.cap ? size : -1;
}

// ---- 9. pack ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPackThreads) pack_kernel(const __grid_constant__ PngParams p) {
  __shared__ int64_t warp[32];
  __shared__ uint16_t code[kLCodes + kDCodes];
  __shared__ uint8_t len[kLCodes + kDCodes];
  const PngGeom& g = p.g[blockIdx.y];
  const FrameRec& r = p.rec[blockIdx.y];
  const int64_t b = blockIdx.x;
  if (b >= r.blocks) return;
  const DBlock& d = p.blocks[g.blk + b];
  uint32_t* words = p.stream + g.words;
  const int last = b == r.blocks - 1;
  if (d.kind == kStored) {
    // 3 header bits, zero bits to the byte, LEN and NLEN little-endian, the bytes
    const int64_t len_at = (d.pos + 3 + 7) >> 3;
    const int64_t stored_len = d.end - d.start;
    if (threadIdx.x == 0) {
      BitWriter w(words, d.pos);
      w.put(last, 3);
      w.flush();
      const uint32_t l = (uint32_t)stored_len;
      put_byte(words, len_at, l & 255);
      put_byte(words, len_at + 1, l >> 8);
      put_byte(words, len_at + 2, ~l & 255);
      put_byte(words, len_at + 3, (~l >> 8) & 255);
    }
    const int64_t at = len_at + 4;
    const uint8_t* src = p.data + g.data + d.start;
    const int64_t w0 = at >> 2, w1 = (at + stored_len - 1) >> 2;
    for (int64_t wi = w0 + threadIdx.x; wi <= w1; wi += kPackThreads) {
      uint32_t v = 0;
      for (int k = 0; k < 4; ++k) {
        const int64_t j = 4 * wi + k - at;
        if (j >= 0 && j < stored_len) v |= (uint32_t)src[j] << (8 * k);
      }
      atomicOr(words + wi, v);
    }
    return;
  }
  for (int i = threadIdx.x; i < kLCodes + kDCodes; i += kPackThreads) {
    code[i] = d.code[i];
    len[i] = d.len[i];
  }
  __syncthreads();
  const int64_t s0 = b * kBlockSymbols, s1 = min(s0 + kBlockSymbols, r.symbols);
  const int64_t first = s0 + (int64_t)threadIdx.x * kPackPerThread;
  const uint16_t* sym = p.sym + g.data;
  int bits = 0;
  for (int64_t k = first; k < min(first + kPackPerThread, s1); ++k) {
    const int s = sym[k];
    if (s < 256) {
      bits += len[s];
    } else {
      const int c = length_code(s - 256);
      bits += len[257 + c] + kExtraLBits[c] + len[kLCodes];
    }
  }
  int64_t total;
  const int64_t at = d.pos + d.head_bits + block_exclusive_scan(bits, warp, &total);
  BitWriter w(words, at);
  for (int64_t k = first; k < min(first + kPackPerThread, s1); ++k) {
    const int s = sym[k];
    if (s < 256) {
      w.put(code[s], len[s]);
    } else {
      const int lc = s - 256, c = length_code(lc);
      w.put(code[257 + c], len[257 + c]);
      if (kExtraLBits[c]) w.put((uint32_t)(lc - kBaseLength[c]), kExtraLBits[c]);
      w.put(code[kLCodes], len[kLCodes]);
    }
  }
  w.flush();
  if (threadIdx.x == 0) {
    BitWriter h(words, d.pos);
    h.put((d.kind == kStatic ? 2 : 4) + last, 3);
    if (d.kind == kDynamic) {
      h.put(d.lmax + 1 - 257, 5);
      h.put(d.dmax + 1 - 1, 5);
      h.put(d.max_blindex + 1 - 4, 4);
      for (int k = 0; k <= d.max_blindex; ++k) h.put(d.bl_len[kBlOrder[k]], 3);
      auto put = [&](int s, int xv, int xb) {
        h.put(d.bl_code[s], d.bl_len[s]);
        if (xb) h.put((uint32_t)xv, xb);
      };
      tree_runs(d.len, d.lmax, put);
      tree_runs(d.len + kLCodes, d.dmax, put);
    }
    h.flush();
    BitWriter e(words, d.pos + d.head_bits + total);
    e.put(code[kEndBlock], len[kEndBlock]);
    e.flush();
  }
}

// ---- 10. IDAT chunks, signature, IHDR, IEND ---------------------------------------------------------
__global__ void __launch_bounds__(kIdatThreads) idat_kernel(const __grid_constant__ PngParams p) {
  __shared__ uint32_t table[256];
  __shared__ int64_t warp[32];
  const PngGeom& g = p.g[blockIdx.y];
  const FrameRec& r = p.rec[blockIdx.y];
  if (r.size > p.cap) return;
  const int64_t chunks = (r.zbytes + kIdatBytes - 1) / kIdatBytes;
  const int64_t c = blockIdx.x;
  if (c >= chunks) return;
  for (int i = threadIdx.x; i < 256; i += kIdatThreads) table[i] = crc_byte((uint32_t)i);
  __syncthreads();
  const uint32_t* words = p.stream + g.words;
  const int64_t z0 = c * kIdatBytes;
  const int clen = (int)min((int64_t)kIdatBytes, r.zbytes - z0);
  uint8_t* o = g.out + 33 + c * (kIdatBytes + 12);
  // "IDAT" and the data: m bytes, CRC'd in pieces of kCrcPiece
  const int m = 4 + clen;
  auto byte_at = [&](int j) -> uint32_t {
    return j < 4 ? (uint32_t)("IDAT"[j]) : get_byte(words, z0 + j - 4);
  };
  uint32_t x = 0;
  for (int piece = threadIdx.x; piece * kCrcPiece < m; piece += kIdatThreads) {
    const int j0 = piece * kCrcPiece, j1 = min(j0 + kCrcPiece, m);
    uint32_t crc = 0xFFFFFFFFu;
    for (int j = j0; j < j1; ++j) {
      const uint32_t v = byte_at(j);
      crc = table[(crc ^ v) & 255] ^ (crc >> 8);
      o[4 + j] = (uint8_t)v;
    }
    x ^= mult_mod_p(x8n_mod_p(m - j1), ~crc);
  }
  // XOR over the CTA
#pragma unroll
  for (int s = 16; s; s >>= 1) x ^= __shfl_xor_sync(0xffffffffu, x, s);
  if ((threadIdx.x & 31) == 0) warp[threadIdx.x >> 5] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t crc = 0;
    for (int k = 0; k < kIdatThreads / 32; ++k) crc ^= (uint32_t)warp[k];
    const uint32_t be[2] = {(uint32_t)clen, crc};
    for (int k = 0; k < 4; ++k) {
      o[k] = (uint8_t)(be[0] >> (24 - 8 * k));
      o[8 + clen + k] = (uint8_t)(be[1] >> (24 - 8 * k));
    }
    if (c == 0) {
      // signature, IHDR
      uint8_t hdr[33] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n', 0, 0, 0, 13, 'I', 'H', 'D', 'R'};
      const uint32_t dims[2] = {(uint32_t)g.w, (uint32_t)g.h};
      for (int k = 0; k < 8; ++k) hdr[16 + k] = (uint8_t)(dims[k >> 2] >> (24 - 8 * (k & 3)));
      hdr[24] = 8;
      hdr[25] = 2;
      hdr[26] = hdr[27] = hdr[28] = 0;
      uint32_t hc = 0xFFFFFFFFu;
      for (int k = 12; k < 29; ++k) hc = table[(hc ^ hdr[k]) & 255] ^ (hc >> 8);
      hc = ~hc;
      for (int k = 0; k < 4; ++k) hdr[29 + k] = (uint8_t)(hc >> (24 - 8 * k));
      for (int k = 0; k < 33; ++k) g.out[k] = hdr[k];
    }
    if (c == chunks - 1) {
      const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
      for (int k = 0; k < 12; ++k) g.out[r.size - 12 + k] = iend[k];
    }
  }
}

// ---- host side --------------------------------------------------------------------------------------
// The worst case of an h x w image.  Each deflate block costs at most its static coding: 3 header
// bits, at most 9 bits per literal (a match, 18 bits at most, covers 3 or more bytes, so less per
// byte) and 7 for the end of block; a stored block is chosen only when its 8 (stored_len + 5) bits
// (header and padding at most 8, LEN and NLEN 32) are at most the static size + 18.  So n filtered
// bytes in B blocks take at most 9 n + 28 B bits, B <= n / 16383 + 1 (a block holds 16383 symbols
// of at least one byte each, the final block possibly none), plus 7 bits of final padding, the
// 2-byte zlib header and the 4-byte Adler-32; the file adds 12 bytes per 8192-byte IDAT chunk and
// the 45 bytes of signature, IHDR and IEND.
struct PngSizes {
  int64_t n, zmax, chunks;
  int segs, blocks;
};
PngSizes png_sizes(int h, int w) {
  PngSizes s;
  s.n = (int64_t)h * (3 * (int64_t)w + 1);
  s.blocks = (int)(s.n / kBlockSymbols + 1);
  s.zmax = 2 + (9 * s.n + 28 * (int64_t)s.blocks + 7 + 7) / 8 + 4;
  s.chunks = (s.zmax + kIdatBytes - 1) / kIdatBytes;
  s.segs = (int)((s.n + kSegBytes - 1) / kSegBytes);
  return s;
}

int64_t png_max_bytes(int h, int w) {
  const PngSizes s = png_sizes(h, w);
  return kFixedBytes + 12 * s.chunks + s.zmax;
}

// The scratch of the frames [first, first + count): filtered bytes, segment values (run starts,
// symbol counts, Adler-32 terms), symbols, deflate blocks, frame records, zlib streams.
struct GroupLayout {
  int64_t data, brk, cnt, adler, sym, blocks, rec, stream, total;
};
GroupLayout group_layout(const FrameSource* fr, int first, int count, PngGeom* g) {
  int64_t data = 0, segs = 0, blocks = 0, words = 0;
  for (int i = 0; i < count; ++i) {
    const FrameSource& s = fr[first + i];
    const PngSizes z = png_sizes(s.h, s.w);
    if (g) {
      g[i].h = s.h;
      g[i].w = s.w;
      g[i].n = z.n;
      g[i].segs = z.segs;
      g[i].max_blocks = z.blocks;
      g[i].max_chunks = (int)z.chunks;
      g[i].data = data;
      g[i].seg = segs;
      g[i].blk = blocks;
      g[i].words = words;
    }
    data += align256(z.n);
    segs += z.segs + 1;
    blocks += z.blocks;
    words += (z.zmax + 3) / 4 + 1;
  }
  GroupLayout L;
  L.data = 0;
  L.brk = L.data + align256(data);
  L.cnt = L.brk + align256(segs * 8);
  L.adler = L.cnt + align256(segs * 8);
  L.sym = L.adler + align256(segs * 16);
  L.blocks = L.sym + align256(data * 2);
  L.rec = L.blocks + align256(blocks * (int64_t)sizeof(DBlock));
  L.stream = L.rec + align256(count * (int64_t)sizeof(FrameRec));
  L.total = L.stream + align256(words * 4);
  return L;
}

template <int F>
int launch_group(const PixFormat& pf, const FrameSource* fr, int first, int count, uint8_t* out,
                 int64_t cap, int64_t* lengths, uint8_t* scratch, cudaStream_t stream) {
  FilterParams<F> fp;
  PngParams& p = fp.p;
  const GroupLayout L = group_layout(fr, first, count, p.g);
  int max_px = 0, max_segs = 0, max_blocks = 0, max_chunks = 0;
  for (int i = 0; i < count; ++i) {
    p.g[i].out = out + (int64_t)(first + i) * cap;
    p.g[i].length = lengths + first + i;
    fp.f[i] = frame_desc<kPlanes<F>>(pf, fr[first + i], fr[first + i].h, fr[first + i].w);
    max_px = std::max(max_px, (int)(((int64_t)p.g[i].h * p.g[i].w + kFilterPixels - 1) / kFilterPixels));
    max_segs = std::max(max_segs, p.g[i].segs);
    max_blocks = std::max(max_blocks, p.g[i].max_blocks);
    max_chunks = std::max(max_chunks, p.g[i].max_chunks);
  }
  p.data = scratch + L.data;
  p.brk = reinterpret_cast<int64_t*>(scratch + L.brk);
  p.cnt = reinterpret_cast<int64_t*>(scratch + L.cnt);
  p.adler = reinterpret_cast<int64_t*>(scratch + L.adler);
  p.sym = reinterpret_cast<uint16_t*>(scratch + L.sym);
  p.blocks = reinterpret_cast<DBlock*>(scratch + L.blocks);
  p.rec = reinterpret_cast<FrameRec*>(scratch + L.rec);
  p.stream = reinterpret_cast<uint32_t*>(scratch + L.stream);
  p.cap = cap;
  SQ_CUDA(cudaMemsetAsync(p.stream, 0, (size_t)(L.total - L.stream), stream));
  const unsigned n = (unsigned)count;
  filter_kernel<F><<<dim3((unsigned)max_px, n), kFilterThreads, 0, stream>>>(fp);
  SQ_CHECK_LAUNCH("png filter_kernel");
  const dim3 sgrid((unsigned)max_segs, n);
  mark_kernel<<<sgrid, kSegThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("png mark_kernel");
  seg_scan_kernel<ScanMax><<<n, 1024, 0, stream>>>(p, p.brk);
  SQ_CHECK_LAUNCH("png seg_scan_kernel");
  count_kernel<<<sgrid, kSegThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("png count_kernel");
  seg_scan_kernel<ScanSum><<<n, 1024, 0, stream>>>(p, p.cnt);
  SQ_CHECK_LAUNCH("png seg_scan_kernel");
  emit_kernel<<<sgrid, kSegThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("png emit_kernel");
  tree_kernel<<<dim3((unsigned)max_blocks, n), kTreeThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("png tree_kernel");
  frame_kernel<<<n, kFrameThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("png frame_kernel");
  pack_kernel<<<dim3((unsigned)max_blocks, n), kPackThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("png pack_kernel");
  idat_kernel<<<dim3((unsigned)max_chunks, n), kIdatThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("png idat_kernel");
  return SQDET_OK;
}

// The scratch the encode of the crops of `frames` needs.
int64_t png_scratch_bytes(const FrameSource* frames, int n) {
  int64_t most = 0;
  for_each_group(n, [&](int first, int count) {
    most = std::max(most, group_layout(frames, first, count, nullptr).total);
    return SQDET_OK;
  });
  return most;
}

int launch_encode_png(int format, const PixFormat& pf, const FrameSource* frames, int n, uint8_t* out,
                      int64_t cap, int64_t* lengths, void* scratch, cudaStream_t stream) {
  uint8_t* s = static_cast<uint8_t*>(scratch);
  return for_each_group(n, [&](int first, int count) {
    return dispatch_format(format, [&](auto f) {
      return launch_group<decltype(f)::value>(pf, frames, first, count, out, cap, lengths, s, stream);
    });
  });
}

}  // namespace
}  // namespace sqdet

using namespace sqdet;

int64_t sqdet_png_max_bytes(int h, int w) {
  if (h < 1 || w < 1 || h > kPngMaxSide || w > kPngMaxSide) {
    fail(SQDET_ERR_INVALID_ARG, "sqdet_png_max_bytes: h and w must be in [1, 1000000]");
    return -1;
  }
  return png_max_bytes(h, w);
}

int64_t sqdet_png_scratch_bytes(int n, const int32_t* heights, const int32_t* widths,
                                const int32_t* crops) {
  std::vector<FrameSource> fr;
  if (encode_crops(kPng.scratch_call, kPng, n, heights, widths, crops, fr)) return -1;
  return png_scratch_bytes(fr.data(), n);
}

int sqdet_encode_png(int n, int format, const uint8_t* const* planes, const int64_t* pitches,
                     const int32_t* heights, const int32_t* widths, const int32_t* crops,
                     uint8_t* out_dev, int64_t cap, int64_t* lengths_dev, void* scratch_dev,
                     int64_t scratch_bytes, void* stream) {
  auto settle = [&](const std::vector<FrameSource>& fr, int64_t& need) {
    need = png_scratch_bytes(fr.data(), n);
    return SQDET_OK;
  };
  auto launch = [&](const PixFormat& pf, const FrameSource* fr) {
    return launch_encode_png(format, pf, fr, n, out_dev, cap, lengths_dev, scratch_dev,
                             (cudaStream_t)stream);
  };
  return encode_frames(kPng, n, format, planes, pitches, heights, widths, crops, out_dev, cap,
                       lengths_dev, scratch_dev, scratch_bytes, settle, launch);
}
