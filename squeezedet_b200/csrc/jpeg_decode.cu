// Baseline / extended sequential JPEG decoding into BGR frames in device memory
// (sqdet_decode_jpeg): file i becomes exactly cv2.imdecode(file_i, cv2.IMREAD_COLOR), which is
// libjpeg-turbo's (SIMD) islow IDCT, fancy upsampling, fixed-point YCbCr->RGB and the EXIF orientation.
// With a scale_denom s of 2, 4 or 8 (sqdet_decode_jpeg_params) it is cv2.imdecode(file_i,
// IMREAD_REDUCED_COLOR_s): each component's scaled IDCT (8, 4, 2 or 1 samples a side, planned per
// component as libjpeg plans it), then that scale's upsampling.  With any_layout
// (sqdet_decode_jpeg_options) also CMYK, YCCK and RGB-coded files and every sampling libjpeg
// decodes: each component upsampled by its own factors, then its colour space converted as cv2
// reads it.  oracle/jpeg_decode.py restates the full-size decode in numpy,
// oracle/jpeg_decode_reduced.py the reduced one, oracle/jpeg_decode_layouts.py the other layouts.
//
// The host parses the headers, builds each file's Huffman lookup and quantization tables and
// packs them with the raw entropy-coded bytes into the caller's pinned staging; one copy takes
// them to the scratch.  Then, per call, on the stream:
//   1. destuff_count   per 4 KiB chunk of each file: its data bytes (stuffed 0x00 and markers
//                      dropped) and RSTn markers, packed in one int64; the first byte of the
//                      terminating marker (atomicMin)
//   2. scan            per file, the exclusive scan of the chunk sums
//   3. destuff_compact each chunk copies its data bytes to the file's clean stream and records
//                      where each restart interval starts, checking the RSTn numbering
//   4. intervals       per file: each interval's subsequences of kSubBits bits (at least one),
//                      scanned into the first subsequence of each interval
//   5. sync_tiles      the self-synchronising Huffman decode (Weissenberger & Schmidt): one
//                      thread per subsequence decodes from a guessed state (bit offset, block of
//                      the MCU, coefficient index) to its first symbol boundary past its end;
//                      rounds in shared memory re-run the subsequences whose entry state changed
//                      until every exit state matches its successor's entry (at most kTile rounds)
//   6. sync_chain      one CTA per file walks its tiles in order: a tile whose first entry
//                      differs from the previous tile's last exit re-runs the rounds of step 5
//   7. scan_counts     per file, the exclusive scan of each subsequence's completed blocks and
//                      per-component DC difference sums
//   8. decode_write    each subsequence decodes again from its final entry state, with its first
//                      block and DC predictors from the scan, and writes its coefficients
//   9. idct            per 8x8 block, the component's planned IDCT: jpeg_idct_islow, _4x4 or _2x2
//                      (as libjpeg-turbo's SIMD code computes them) or _1x1, into its plane
//  10. color           per output pixel: orientation, the planned upsampling (fancy or
//                      replicated), YCbCr->BGR; color_any for the other layouts (launched only
//                      when a call has one)
// All loops are bounded by host-known sizes; a corrupt entropy-coded segment sets a negative
// status for its file and nothing else.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"
#include "scan.cuh"

namespace sqdet {

namespace {

constexpr int kMaxFiles = 128;
constexpr int kMaxFileBytes = 1 << 28;   // bit offsets within a file fit int32
constexpr int kChunkThreads = 256;
constexpr int kChunkBytes = 16;          // raw bytes per destuffing thread
constexpr int kChunk = kChunkThreads * kChunkBytes;
constexpr int kScanThreads = 1024;
constexpr int kTile = 128;               // subsequences per sync CTA
constexpr int kDefaultSubBits = 1024;
constexpr int kFastBits = 9;
constexpr int kPixThreads = 256;

int g_sub_bits = kDefaultSubBits;

constexpr int kNatural[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5,
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t kNaturalDev[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5,
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// A Huffman table: codes of up to kFastBits bits by a lookup of the next kFastBits bits
// (length << 8 | symbol, 0 for longer or invalid codes); longer ones canonically, through the
// largest code of each length (-1: none) and the offset from a code to its symbol's index.
struct HuffTab {
  uint16_t fast[1 << kFastBits];
  int32_t maxcode[17];
  int32_t valoff[17];
  uint8_t vals[256];
};

constexpr int kMaxComps = 4;
constexpr int kMaxBlocks = 10;           // libjpeg's D_MAX_BLOCKS_IN_MCU

// libjpeg's colour space of a file, as default_decompress_parms decides it
enum Space : int8_t { kYcc = 0, kGray, kRgb, kCmyk, kYcck };

// Everything the kernels know of one file.  Offsets are bytes from the scratch's start.
struct DecFile {
  int32_t h, w, oh, ow, ncomp, orient;
  int32_t mcu_cols, mcus, bpm, restart, intervals;
  int32_t raw_len, chunks, blocks, sub_max;
  int32_t sub_bits;
  int8_t bcomp[kMaxBlocks], bdy[kMaxBlocks], bdx[kMaxBlocks];  // per block of an MCU: component,
                                                               // block row and column in it
  int8_t ch[kMaxComps], cv[kMaxComps];  // sampling factors
  int8_t isz[kMaxComps];               // IDCT size: samples a side per block (8 at full size)
  int8_t uh[kMaxComps], uv[kMaxComps];  // upsampling factors to the frame
  int8_t fancy;                        // fancy upsampling (off at 1/8)
  int8_t space;                        // Space
  int8_t general;                      // converted by color_any_kernel, not color_kernel
  int32_t pw[kMaxComps], ph[kMaxComps];  // padded plane width and height (whole blocks)
  int32_t cw[kMaxComps], chh[kMaxComps];  // component width and height in samples
  int16_t q[kMaxComps][64];            // dequantization, natural order (libjpeg's short multiplier)
  int32_t index;                       // the file's index in the call: where its status goes
  int64_t raw, clean, sums, term, ist, sbase, entry, exit_, counts, coef, plane[kMaxComps], tabs;
  int64_t counts3;                     // 4 components: component 3's DC sums beside counts
  uint8_t* out;
  int64_t pitch;
};

struct DecParams {
  DecFile* f;
  uint8_t* s;                           // the scratch
  int32_t* status;
};

__device__ __forceinline__ void fail_file(int32_t* status, const DecFile& f, int code) {
  status[f.index] = code;
}

// ---- 1. destuff counts ---------------------------------------------------------------------------
// Byte j of a file's entropy-coded segment is data unless it is the byte after a 0xFF that starts
// a marker or a stuffed 0x00, or a fill 0xFF before one.  A 0xFF followed by something other
// than 0x00, 0xFF or RSTn ends the segment (EOI, normally), as does a 0xFF that ends the file.
constexpr int64_t kRstOne = int64_t(1) << 40;   // chunk sums: RSTn count << 40 | data bytes

__device__ __forceinline__ int byte_at(const uint8_t* raw, int len, int j) {
  return j >= 0 && j < len ? raw[j] : -1;
}

// 0 data, 1 dropped, 2 RSTn (its 0xFF), 3 terminator (its 0xFF)
__device__ __forceinline__ int classify(const uint8_t* raw, int len, int j) {
  const int b = raw[j];
  if (b == 0xFF) {
    const int nx = byte_at(raw, len, j + 1);
    if (nx == 0x00) return 0;
    if (nx == 0xFF) return 1;
    if (nx >= 0xD0 && nx <= 0xD7) return 2;
    return 3;
  }
  return byte_at(raw, len, j - 1) == 0xFF ? 1 : 0;
}

__global__ void __launch_bounds__(kChunkThreads) destuff_count_kernel(DecParams p) {
  __shared__ int64_t warp[32];
  const DecFile& f = p.f[blockIdx.y];
  if ((int)blockIdx.x >= f.chunks) return;
  const uint8_t* raw = p.s + f.raw;
  const int first = blockIdx.x * kChunk + threadIdx.x * kChunkBytes;
  int64_t v = 0;
  int term = INT32_MAX;
  for (int j = first; j < first + kChunkBytes && j < f.raw_len; ++j) {
    const int c = classify(raw, f.raw_len, j);
    v += c == 0 ? 1 : c == 2 ? kRstOne : 0;
    if (c == 3 && term == INT32_MAX) term = j;
  }
  if (term != INT32_MAX) atomicMin(reinterpret_cast<uint32_t*>(p.s + f.term), (uint32_t)term);
  int64_t total;
  block_exclusive_scan(v, warp, &total);
  if (threadIdx.x == 0) reinterpret_cast<int64_t*>(p.s + f.sums)[blockIdx.x] = total;
}

// ---- 2. per-file exclusive scan of chunk sums ------------------------------------------------------
__global__ void __launch_bounds__(kScanThreads) scan_chunks_kernel(DecParams p) {
  __shared__ int64_t warp[32];
  const DecFile& f = p.f[blockIdx.x];
  int64_t* s = reinterpret_cast<int64_t*>(p.s + f.sums);
  int64_t carry = 0;
  for (int base = 0; base < f.chunks; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const int64_t v = i < f.chunks ? s[i] : 0;
    int64_t total;
    const int64_t ex = block_exclusive_scan(v, warp, &total);
    if (i < f.chunks) s[i] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) s[f.chunks] = carry;
}

// ---- 3. compact ------------------------------------------------------------------------------------
// ist[r] is the clean byte where interval r starts (ist[0] = 0, ist[intervals] = the end); the
// intervals kernel finds any left at -1.
__global__ void __launch_bounds__(kChunkThreads) destuff_compact_kernel(DecParams p) {
  __shared__ int64_t warp[32];
  const DecFile& f = p.f[blockIdx.y];
  if ((int)blockIdx.x >= f.chunks) return;
  const uint8_t* raw = p.s + f.raw;
  uint8_t* clean = p.s + f.clean;
  int32_t* ist = reinterpret_cast<int32_t*>(p.s + f.ist);
  const int term = (int)min(*reinterpret_cast<const uint32_t*>(p.s + f.term), (uint32_t)f.raw_len);
  const int first = blockIdx.x * kChunk + threadIdx.x * kChunkBytes;
  uint8_t cls[kChunkBytes];
  int64_t v = 0;
#pragma unroll
  for (int i = 0; i < kChunkBytes; ++i) {
    const int j = first + i;
    cls[i] = j < f.raw_len ? (uint8_t)classify(raw, f.raw_len, j) : 1;
    v += cls[i] == 0 ? 1 : cls[i] == 2 ? kRstOne : 0;
  }
  int64_t total;
  const int64_t at = reinterpret_cast<const int64_t*>(p.s + f.sums)[blockIdx.x] + block_exclusive_scan(v, warp, &total);
  int64_t o = at & (kRstOne - 1);
  int r = (int)(at >> 40);
  for (int i = 0; i < kChunkBytes; ++i) {
    const int j = first + i;
    if (j >= term) {
      if (j == term) ist[f.intervals] = (int32_t)o;
      break;
    }
    if (cls[i] == 0) {
      clean[o++] = raw[j];
    } else if (cls[i] == 2) {
      // the r-th marker ends interval r and must be RST(r mod 8); markers after the last
      // interval's are skipped, as libjpeg skips them
      if (r + 1 < f.intervals) {
        if (raw[j + 1] != 0xD0 + (r & 7)) fail_file(p.status, f, -2);
        ist[r + 1] = (int32_t)o;
      }
      ++r;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    ist[0] = 0;
    if (term >= f.raw_len) {                            // no terminator: the data runs to the end
      ist[f.intervals] = (int32_t)(reinterpret_cast<const int64_t*>(p.s + f.sums)[f.chunks] & (kRstOne - 1));
    }
  }
}

// ---- 4. intervals -> subsequences ------------------------------------------------------------------
// sbase[r] is the first subsequence of interval r, sbase[intervals] their count (<= sub_max).
__global__ void __launch_bounds__(kScanThreads) intervals_kernel(DecParams p) {
  __shared__ int32_t warp[32];
  const int i = blockIdx.x;
  const DecFile& f = p.f[i];
  const int32_t* ist = reinterpret_cast<const int32_t*>(p.s + f.ist);
  int32_t* sbase = reinterpret_cast<int32_t*>(p.s + f.sbase);
  int32_t carry = 0;
  bool bad = false;
  for (int base = 0; base < f.intervals; base += kScanThreads) {
    const int r = base + threadIdx.x;
    int32_t v = 0;
    if (r < f.intervals) {
      const int a = ist[r], b = ist[r + 1];
      if (a < 0 || b < a) {
        bad = true;
        v = 1;
      } else {
        v = max(1, (int)(((int64_t)(b - a) * 8 + f.sub_bits - 1) / f.sub_bits));
      }
    }
    int32_t total;
    const int32_t ex = block_exclusive_scan(v, warp, &total);
    if (r < f.intervals) sbase[r] = carry + ex;
    carry += total;
  }
  if (bad) fail_file(p.status, f, -3);
  if (threadIdx.x == 0) sbase[f.intervals] = min(carry, f.sub_max);
}

// ---- the Huffman decoder ---------------------------------------------------------------------------
// The 32 bits of the clean stream from bit p on (MSB first); words past the end are padding.
__device__ __forceinline__ uint32_t peek32(const uint8_t* clean, int p) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(clean) + (p >> 5);
  const uint32_t a = __byte_perm(w[0], 0, 0x0123), b = __byte_perm(w[1], 0, 0x0123);
  return __funnelshift_l(b, a, p & 31);
}

// One decoder state at a symbol boundary: bit offset, block of the MCU, next coefficient (0: DC).
struct State {
  int p, uk;                             // uk = u << 8 | k
  __device__ bool operator==(const State& o) const { return p == o.p && uk == o.uk; }
};

// The symbol and code length at the front of `bits`, length 0 for an invalid code.
__device__ __forceinline__ int huff_decode(const HuffTab& t, uint32_t bits, int& len) {
  const int e = t.fast[bits >> (32 - kFastBits)];
  if (e) {
    len = e >> 8;
    return e & 255;
  }
  int l = kFastBits + 1;
  int code = (int)(bits >> (32 - l));
#pragma unroll 1
  for (; l <= 16 && code > t.maxcode[l]; ++l) code = (int)(bits >> (32 - (l + 1)));
  if (l > 16) {
    len = 0;
    return 0;
  }
  len = l;
  return t.vals[(t.valoff[l] + code) & 255];
}

__device__ __forceinline__ int extend(uint32_t v, int s) {
  return s && v < (1u << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v;
}

struct Counts {
  int blocks, dc[kMaxComps];
};

// Decodes from state st while st.p < end and fewer than block_limit blocks are complete.  kWrite:
// writes the block's coefficients (JCOEF, natural order) to coef + 64 * (block0 + blocks), with
// the DC predictors in c.dc, and reports corrupt data through the return value (negative);
// otherwise c.dc sums the DC differences and corrupt data decodes on deterministically.
template <bool kWrite>
__device__ int decode_run(const DecFile& f, const HuffTab* tabs, const uint8_t* clean, State& st,
                          int end, int block_limit, Counts& c, int16_t* coef, int64_t block0,
                          int max_iter) {
  int p = st.p, u = st.uk >> 8, k = st.uk & 255;
#pragma unroll 1
  for (int it = 0; it < max_iter && p < end && c.blocks < block_limit; ++it) {
    const int comp = f.bcomp[u];
    const uint32_t bits = peek32(clean, p);
    int len;
    const int sym = huff_decode(tabs[2 * comp + (k ? 1 : 0)], bits, len);
    if (!len) {
      if (kWrite) return -4;
      ++p;                                // speculative: step one bit
      continue;
    }
    const int s = sym & 15, run = sym >> 4;
    const uint32_t extra = s ? (bits << len) >> (32 - s) : 0;
    p += len + s;
    if (k == 0) {
      if (sym > 15) {
        if (kWrite) return -4;
      }
      c.dc[comp] += extend(extra, s);
      if (kWrite) coef[(block0 + c.blocks) * 64] = (int16_t)c.dc[comp];
      k = 1;
    } else if (s) {
      k += run;
      if (k > 63) {
        if (kWrite) return -5;
        k = 64;
      } else {
        if (kWrite) coef[(block0 + c.blocks) * 64 + kNaturalDev[k]] = (int16_t)extend(extra, s);
        ++k;
      }
    } else if (run == 15) {
      k += 16;
      if (k > 64) {
        if (kWrite) return -5;
        k = 64;
      }
    } else {
      k = 64;
    }
    if (k >= 64) {
      ++c.blocks;
      k = 0;
      u = u + 1 == f.bpm ? 0 : u + 1;
    }
  }
  st.p = p;
  st.uk = u << 8 | k;
  return 0;
}

// Subsequence g of a file: its interval r, its first bit and the end of its range.
struct Sub {
  int r, j, start, end, nsub;
};
__device__ Sub locate(const DecFile& f, const int32_t* ist, const int32_t* sbase, int g) {
  int lo = 0, hi = f.intervals - 1;           // the last r with sbase[r] <= g
#pragma unroll 1
  for (int it = 0; it < 32 && lo < hi; ++it) {
    const int mid = (lo + hi + 1) >> 1;
    if (sbase[mid] <= g) lo = mid; else hi = mid - 1;
  }
  Sub s;
  s.r = lo;
  s.j = g - sbase[lo];
  s.nsub = sbase[lo + 1] - sbase[lo];
  const int a = max(ist[lo], 0), b = max(ist[lo + 1], a);
  s.start = a * 8 + s.j * f.sub_bits;
  s.end = min(s.start + f.sub_bits, b * 8);
  return s;
}

// The rounds of the synchronisation within one tile of kTile subsequences from g0: entries whose
// `dirty` flag is set are decoded again, and each exit that differs from its successor's entry
// (unless that successor starts an interval) becomes that entry.  Each round makes at least one
// more entry final, so kTile rounds suffice.
__device__ void sync_rounds(const DecFile& f, const HuffTab* tabs, const uint8_t* clean,
                            const Sub& sub, bool valid, bool dirty0, State* entry, State* exit_,
                            Counts& cnt, int* starts_interval) {
  const int t = threadIdx.x;
  bool dirty = dirty0;
  starts_interval[t] = !valid || sub.j == 0;
  __syncthreads();
#pragma unroll 1
  for (int round = 0; round < kTile; ++round) {
    if (dirty && valid) {
      State st = entry[t];
      cnt = Counts{0, {0, 0, 0, 0}};
      decode_run<false>(f, tabs, clean, st, sub.end, INT32_MAX, cnt, nullptr, 0, f.sub_bits + 64);
      exit_[t] = st;
    }
    dirty = false;
    __syncthreads();
    bool changed = false;
    if (t > 0 && valid && !starts_interval[t] && !(exit_[t - 1] == entry[t])) {
      changed = true;
    }
    const State prev = t > 0 ? exit_[t - 1] : State{0, 0};
    __syncthreads();
    if (changed) {
      entry[t] = prev;
      dirty = true;
    }
    if (!__syncthreads_or(changed)) break;
  }
}

// ---- 5. sync within tiles ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kTile) sync_tiles_kernel(DecParams p) {
  __shared__ State entry[kTile], exit_[kTile];
  __shared__ int starts[kTile];
  const DecFile& f = p.f[blockIdx.y];
  const int32_t* sbase = reinterpret_cast<const int32_t*>(p.s + f.sbase);
  const int nsub = sbase[f.intervals];
  const int g0 = blockIdx.x * kTile;
  if (g0 >= nsub) return;
  const int32_t* ist = reinterpret_cast<const int32_t*>(p.s + f.ist);
  const HuffTab* tabs = reinterpret_cast<const HuffTab*>(p.s + f.tabs);
  const uint8_t* clean = p.s + f.clean;
  const int g = g0 + threadIdx.x;
  const bool valid = g < nsub;
  const Sub sub = valid ? locate(f, ist, sbase, g) : Sub{0, 0, 0, 0, 0};
  entry[threadIdx.x] = State{sub.start, 0};
  Counts cnt{0, {0, 0, 0, 0}};
  sync_rounds(f, tabs, clean, sub, valid, true, entry, exit_, cnt, starts);
  if (valid) {
    reinterpret_cast<State*>(p.s + f.entry)[g] = entry[threadIdx.x];
    reinterpret_cast<State*>(p.s + f.exit_)[g] = exit_[threadIdx.x];
    reinterpret_cast<int4*>(p.s + f.counts)[g] = make_int4(cnt.blocks, cnt.dc[0], cnt.dc[1], cnt.dc[2]);
    if (f.ncomp == 4) reinterpret_cast<int32_t*>(p.s + f.counts3)[g] = cnt.dc[3];
  }
}

// ---- 6. sync across tiles ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kTile) sync_chain_kernel(DecParams p) {
  __shared__ State entry[kTile], exit_[kTile];
  __shared__ int starts[kTile];
  const DecFile& f = p.f[blockIdx.x];
  const int32_t* sbase = reinterpret_cast<const int32_t*>(p.s + f.sbase);
  const int nsub = sbase[f.intervals];
  const int32_t* ist = reinterpret_cast<const int32_t*>(p.s + f.ist);
  const HuffTab* tabs = reinterpret_cast<const HuffTab*>(p.s + f.tabs);
  const uint8_t* clean = p.s + f.clean;
  State* gentry = reinterpret_cast<State*>(p.s + f.entry);
  State* gexit = reinterpret_cast<State*>(p.s + f.exit_);
  int4* gcounts = reinterpret_cast<int4*>(p.s + f.counts);
  int32_t* gcounts3 = reinterpret_cast<int32_t*>(p.s + f.counts3);
  const int tiles = (f.sub_max + kTile - 1) / kTile;
#pragma unroll 1
  for (int tile = 1; tile < tiles; ++tile) {
    const int g0 = tile * kTile;
    if (g0 >= nsub) break;
    const int g = g0 + threadIdx.x;
    const bool valid = g < nsub;
    // the tile's first entry is final once the previous tile's last exit is
    const Sub first = locate(f, ist, sbase, g0);
    const State want = gexit[g0 - 1];
    const bool stale = first.j != 0 && !(gentry[g0] == want);
    if (!stale) continue;                  // uniform across the CTA
    const Sub sub = valid ? locate(f, ist, sbase, g) : Sub{0, 0, 0, 0, 0};
    if (valid) {
      entry[threadIdx.x] = threadIdx.x == 0 ? want : gentry[g];
      exit_[threadIdx.x] = gexit[g];
    }
    const int4 c4 = valid ? gcounts[g] : make_int4(0, 0, 0, 0);
    Counts cnt{c4.x, {c4.y, c4.z, c4.w, valid && f.ncomp == 4 ? gcounts3[g] : 0}};
    __syncthreads();
    sync_rounds(f, tabs, clean, sub, valid, threadIdx.x == 0, entry, exit_, cnt, starts);
    if (valid) {
      gentry[g] = entry[threadIdx.x];
      gexit[g] = exit_[threadIdx.x];
      gcounts[g] = make_int4(cnt.blocks, cnt.dc[0], cnt.dc[1], cnt.dc[2]);
      if (f.ncomp == 4) gcounts3[g] = cnt.dc[3];
    }
    __syncthreads();
  }
}

// ---- 7. per-file exclusive scan of the counts ---------------------------------------------------------
__global__ void __launch_bounds__(kScanThreads) scan_counts_kernel(DecParams p) {
  __shared__ int32_t warp[32];
  const DecFile& f = p.f[blockIdx.x];
  const int nsub = reinterpret_cast<const int32_t*>(p.s + f.sbase)[f.intervals];
  int4* c = reinterpret_cast<int4*>(p.s + f.counts);
  int4 carry = make_int4(0, 0, 0, 0);
  for (int base = 0; base < nsub; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const int4 v = i < nsub ? c[i] : make_int4(0, 0, 0, 0);
    int4 ex, tot;
    ex.x = block_exclusive_scan(v.x, warp, &tot.x);
    ex.y = block_exclusive_scan(v.y, warp, &tot.y);
    ex.z = block_exclusive_scan(v.z, warp, &tot.z);
    ex.w = block_exclusive_scan(v.w, warp, &tot.w);
    if (i < nsub) c[i] = make_int4(carry.x + ex.x, carry.y + ex.y, carry.z + ex.z, carry.w + ex.w);
    carry = make_int4(carry.x + tot.x, carry.y + tot.y, carry.z + tot.z, carry.w + tot.w);
  }
  if (f.ncomp != 4) return;                // uniform: one file per CTA
  int32_t* c3 = reinterpret_cast<int32_t*>(p.s + f.counts3);
  int32_t carry3 = 0;
  for (int base = 0; base < nsub; base += kScanThreads) {
    const int i = base + threadIdx.x;
    int32_t tot;
    const int32_t ex = block_exclusive_scan(i < nsub ? c3[i] : 0, warp, &tot);
    if (i < nsub) c3[i] = carry3 + ex;
    carry3 += tot;
  }
}

// ---- 8. decode and write coefficients -----------------------------------------------------------------
__global__ void __launch_bounds__(kTile) decode_write_kernel(DecParams p) {
  const DecFile& f = p.f[blockIdx.y];
  const int32_t* sbase = reinterpret_cast<const int32_t*>(p.s + f.sbase);
  const int nsub = sbase[f.intervals];
  const int g = blockIdx.x * kTile + threadIdx.x;
  if (g >= nsub) return;
  const int32_t* ist = reinterpret_cast<const int32_t*>(p.s + f.ist);
  const HuffTab* tabs = reinterpret_cast<const HuffTab*>(p.s + f.tabs);
  const int4* counts = reinterpret_cast<const int4*>(p.s + f.counts);
  const Sub sub = locate(f, ist, sbase, g);
  const int4 mine = counts[g], base = counts[sbase[sub.r]];
  const int interval_blocks = min(f.restart, f.mcus - sub.r * f.restart) * f.bpm;
  const int32_t* counts3 = reinterpret_cast<const int32_t*>(p.s + f.counts3);
  Counts c{mine.x - base.x, {mine.y - base.y, mine.z - base.z, mine.w - base.w,
                             f.ncomp == 4 ? counts3[g] - counts3[sbase[sub.r]] : 0}};
  const int b0 = c.blocks;
  if (b0 < 0) {
    fail_file(p.status, f, -6);
    return;
  }
  State st = reinterpret_cast<const State*>(p.s + f.entry)[g];
  // every block of the interval lies in [first block of the interval, + interval_blocks)
  c.blocks = 0;
  int16_t* coef = reinterpret_cast<int16_t*>(p.s + f.coef);
  const int64_t block0 = (int64_t)sub.r * f.restart * f.bpm + b0;
  const int limit = interval_blocks - b0;
  const int rc = limit > 0 ? decode_run<true>(f, tabs, p.s + f.clean, st, sub.end, limit, c, coef,
                                              block0, f.sub_bits + 64)
                           : 0;
  const int end_bits = max(ist[sub.r + 1], 0) * 8;
  if (rc) {
    fail_file(p.status, f, rc);
  } else if (st.p > end_bits) {
    fail_file(p.status, f, -7);                          // ran off the interval's data
  } else if (sub.j == sub.nsub - 1 && b0 + c.blocks < interval_blocks) {
    fail_file(p.status, f, -8);                          // too few blocks in the interval
  }
  // data after an interval's last block is skipped, as libjpeg skips it before the next marker
}

// ---- 9. IDCT ----------------------------------------------------------------------------------------
constexpr int F0_298 = 2446, F0_390 = 3196, F0_541 = 4433, F0_765 = 6270, F0_899 = 7373,
              F1_175 = 9633, F1_501 = 12299, F1_847 = 15137, F1_961 = 16069, F2_053 = 16819,
              F2_562 = 20995, F3_072 = 25172;

__device__ __forceinline__ int w16(int x) { return (int)(int16_t)x; }   // a 16-bit SIMD add
__device__ __forceinline__ int s16(int x) { return min(max(x, -32768), 32767); }   // packssdw

// One 1-D pass of jpeg_idct_islow over d[0], d[stride], ... d[7 stride], descaled by `shift`, as
// libjpeg-turbo's SIMD islow computes it (cv2 runs that code): products and their sums in 32 bits,
// in0 +- in4, in7 + in3 and in5 + in1 in 16 bits.  For coefficients an 8-bit encoder writes this
// is jidctint.c's arithmetic; it differs only where those sums overflow 16 bits.
__device__ __forceinline__ void idct8(int* d, int stride, int shift) {
  int z2 = d[2 * stride], z3 = d[6 * stride];
  int z1 = (z2 + z3) * F0_541;
  const int tmp2 = z1 - z3 * F1_847, tmp3 = z1 + z2 * F0_765;
  const int tmp0 = w16(d[0] + d[4 * stride]) << 13, tmp1 = w16(d[0] - d[4 * stride]) << 13;
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int a0 = d[7 * stride], a1 = d[5 * stride], a2 = d[3 * stride], a3 = d[stride];
  z1 = a0 + a3;
  z2 = a1 + a2;
  z3 = w16(a0 + a2);
  int z4 = w16(a1 + a3);
  const int z5 = (z3 + z4) * F1_175;
  a0 *= F0_298;
  a1 *= F2_053;
  a2 *= F3_072;
  a3 *= F1_501;
  z1 *= -F0_899;
  z2 *= -F2_562;
  z3 = z3 * -F1_961 + z5;
  z4 = z4 * -F0_390 + z5;
  a0 += z1 + z3;
  a1 += z2 + z4;
  a2 += z2 + z3;
  a3 += z1 + z4;
  const int rnd = 1 << (shift - 1);
  d[0] = (t10 + a3 + rnd) >> shift;
  d[7 * stride] = (t10 - a3 + rnd) >> shift;
  d[stride] = (t11 + a2 + rnd) >> shift;
  d[6 * stride] = (t11 - a2 + rnd) >> shift;
  d[2 * stride] = (t12 + a1 + rnd) >> shift;
  d[5 * stride] = (t12 - a1 + rnd) >> shift;
  d[3 * stride] = (t13 + a0 + rnd) >> shift;
  d[4 * stride] = (t13 - a0 + rnd) >> shift;
}

// jidctred.c's constants, 13 fraction bits
constexpr int F0_211 = 1730, F0_509 = 4176, F0_601 = 4926, F0_720 = 5906, F0_850 = 6967,
              F1_061 = 8697, F1_272 = 10426, F1_451 = 11893, F2_172 = 17799, F3_624 = 29692;

// 32-bit sums that wrap as the SIMD code's paddd does (they can pass 2^31 on 16-bit tables)
__device__ __forceinline__ int wadd(int a, int b) { return (int)((unsigned)a + (unsigned)b); }
__device__ __forceinline__ int wsub(int a, int b) { return (int)((unsigned)a - (unsigned)b); }
__device__ __forceinline__ int wshl(int a, int s) { return (int)((unsigned)a << s); }

// One 1-D pass of jpeg_idct_4x4 over d[0], d[stride], ... d[7 stride] (d[4 stride] unused), as
// jsimd_idct_4x4_sse2 computes it: pmaddwd products of 16-bit inputs summed in 32 bits -> the
// four outputs, descaled by `shift`.
__device__ __forceinline__ void red4(const int* d, int stride, int shift, int* o) {
  const int tmp0 = wshl(d[0], 14);
  const int tmp2 = wsub(d[2 * stride] * F1_847, d[6 * stride] * F0_765);
  const int t10 = wadd(tmp0, tmp2), t12 = wsub(tmp0, tmp2);
  const int z1 = d[7 * stride], z2 = d[5 * stride], z3 = d[3 * stride], z4 = d[stride];
  const int odd0 = wadd(wadd(z1 * -F0_211, z2 * F1_451), wadd(z3 * -F2_172, z4 * F1_061));
  const int odd2 = wadd(wadd(z1 * -F0_509, z2 * -F0_601), wadd(z3 * F0_899, z4 * F2_562));
  const int rnd = 1 << (shift - 1);
  o[0] = wadd(wadd(t10, odd2), rnd) >> shift;
  o[1] = wadd(wadd(t12, odd0), rnd) >> shift;
  o[2] = wadd(wsub(t12, odd0), rnd) >> shift;
  o[3] = wadd(wsub(t10, odd2), rnd) >> shift;
}

// jpeg_idct_2x2's odd part over d[stride], d[3 stride], d[5 stride], d[7 stride].
__device__ __forceinline__ int red2_odd(const int* d, int stride) {
  return wadd(wsub(d[stride] * F3_624, d[3 * stride] * F1_272),
              wsub(d[5 * stride] * F0_850, d[7 * stride] * F0_720));
}

__device__ __forceinline__ uint32_t clamp_sample(int v) { return (uint32_t)(min(max(v, -128), 127) + 128); }

// jpeg_idct_4x4 (jsimd_idct_4x4_sse2) of dequantized d[64] into a 4x4 block of the plane: a block
// whose coefficient rows 1, 2, 3, 5, 6 and 7 are all zero takes row 0 << 2 (16-bit) as its column
// pass, the others the column pass saturated to 16 bits; the row pass saturates to 8 bits.
__device__ __forceinline__ void idct_4x4(int* d, bool ac, uint8_t* out, int pw) {
  int ws[32];
#pragma unroll
  for (int col = 0; col < 8; ++col) {
    int o[4];
    if (ac) {
      red4(d + col, 8, 12, o);
#pragma unroll
      for (int r = 0; r < 4; ++r) o[r] = s16(o[r]);
    } else {
#pragma unroll
      for (int r = 0; r < 4; ++r) o[r] = w16(d[col] << 2);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) ws[8 * r + col] = o[r];
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    int o[4];
    red4(ws + 8 * r, 1, 19, o);
    uint32_t w = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) w |= clamp_sample(o[k]) << (8 * k);
    *reinterpret_cast<uint32_t*>(out + (int64_t)r * pw) = w;
  }
}

// jpeg_idct_2x2 (jsimd_idct_2x2_sse2) of dequantized d[64] into a 2x2 block: no zero test; the
// column pass keeps column 0 in 32 bits and saturates columns 1, 3, 5 and 7 to 16; the row pass
// shifts column 0 left in 32 bits (it wraps) and saturates the output to 8 bits.
__device__ __forceinline__ void idct_2x2(const int* d, uint8_t* out, int pw) {
  int ws[2][8];
#pragma unroll
  for (int col = 0; col < 8; ++col) {
    if (col == 2 || col == 4 || col == 6) continue;
    const int t10 = wshl(d[col], 15), t0 = red2_odd(d + col, 8);
    const int a = wadd(wadd(t10, t0), 1 << 12) >> 13, b = wadd(wsub(t10, t0), 1 << 12) >> 13;
    ws[0][col] = col ? s16(a) : a;
    ws[1][col] = col ? s16(b) : b;
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int t10 = wshl(ws[r][0], 15), t0 = red2_odd(ws[r], 1);
    const uint32_t lo = clamp_sample(wadd(wadd(t10, t0), 1 << 19) >> 20);
    const uint32_t hi = clamp_sample(wadd(wsub(t10, t0), 1 << 19) >> 20);
    *reinterpret_cast<uint16_t*>(out + (int64_t)r * pw) = (uint16_t)(lo | hi << 8);
  }
}

// jpeg_idct_1x1 (C: libjpeg-turbo has no SIMD one): the DC times its quantizer (16-bit signed,
// product exact), descaled by 3, through jidctred.c's range_limit[x & 1023].
__device__ __forceinline__ uint8_t idct_1x1(int dc, int q) {
  const int x = ((dc * q + 4) >> 3) & 1023;
  return (uint8_t)(x < 128 ? x + 128 : x < 512 ? 255 : x < 896 ? 0 : x - 896);
}

// Each block through its component's planned IDCT.  8: the SIMD islow's block, dequantization by a
// 16-bit multiply; the column pass saturated to 16 bits, or, when every AC coefficient is zero,
// the DC << 2 in 16 bits; the output clamped.  4, 2, 1: the reduced ones above, which only the
// kScaled instance has, so that a full-size decode keeps islow's registers and occupancy.
template <bool kScaled>
__global__ void __launch_bounds__(kPixThreads) idct_kernel(DecParams p) {
  const DecFile& f = p.f[blockIdx.y];
  const int b = blockIdx.x * kPixThreads + threadIdx.x;
  if (b >= f.blocks) return;
  const int m = b / f.bpm, u = b - m * f.bpm;
  const int c = f.bcomp[u];
  int by, bx;
  if (f.ncomp == 1) {
    by = m / f.mcu_cols;
    bx = m - by * f.mcu_cols;
  } else {
    const int my = m / f.mcu_cols, mx = m - my * f.mcu_cols;
    by = my * f.cv[c] + f.bdy[u];
    bx = mx * f.ch[c] + f.bdx[u];
  }
  const int4* src = reinterpret_cast<const int4*>(p.s + f.coef) + (int64_t)b * 8;
  const int n = kScaled ? f.isz[c] : 8;
  uint8_t* plane = p.s + f.plane[c];
  const int pw = f.pw[c];
  if (kScaled && n == 1) {
    plane[(int64_t)by * pw + bx] = idct_1x1(reinterpret_cast<const int16_t*>(src)[0], f.q[c][0]);
    return;
  }
  int d[64];
  int ac = 0, ac4 = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int4 v = src[i];
    if (i) ac |= v.x | v.y | v.z | v.w;
    if (kScaled && i && i != 4) ac4 |= v.x | v.y | v.z | v.w;
    const int16_t* h = reinterpret_cast<const int16_t*>(&v);
#pragma unroll
    for (int e = 0; e < 8; ++e) d[8 * i + e] = w16((int)h[e] * (int)f.q[c][8 * i + e]);
  }
  if (kScaled && n == 4) {
    idct_4x4(d, ac4 != 0, plane + (int64_t)by * 4 * pw + bx * 4, pw);
    return;
  }
  if (kScaled && n == 2) {
    idct_2x2(d, plane + (int64_t)by * 2 * pw + bx * 2, pw);
    return;
  }
  if (ac) {
#pragma unroll
    for (int col = 0; col < 8; ++col) idct8(d + col, 8, 11);
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = s16(d[i]);
  } else {
#pragma unroll
    for (int i = 63; i >= 0; --i) d[i] = w16(d[i & 7] << 2);   // row 0 last: the others read it
  }
#pragma unroll
  for (int row = 0; row < 8; ++row) idct8(d + 8 * row, 1, 18);
#pragma unroll
  for (int row = 0; row < 8; ++row) {
    uint32_t w[2] = {0, 0};
#pragma unroll
    for (int col = 0; col < 8; ++col) {
      const int v = min(max(s16(d[8 * row + col]), -128), 127) + 128;
      w[col >> 2] |= (uint32_t)v << (8 * (col & 3));
    }
    *reinterpret_cast<uint2*>(plane + (int64_t)(by * 8 + row) * pw + bx * 8) = make_uint2(w[0], w[1]);
  }
}

// ---- 10. upsample, convert, orient ----------------------------------------------------------------------
// Chroma of frame pixel (y, x) from plane c (cw x chh samples) upsampled by (fh, fv): with `fancy`,
// libjpeg's triangle filters where it has them (h2v1 and h2v2 on planes wider than 2 samples,
// h1v2 always), replication otherwise.
__device__ __forceinline__ int chroma_at(const uint8_t* pl, int pw, int cw, int chh, int fh, int fv,
                                         bool fancy, int y, int x) {
  const bool fancy_h = fancy && fh == 2 && cw > 2;
  if (fh == 1 && fv == 1) return pl[(int64_t)y * pw + x];
  if (fancy && fv == 2 && (fh == 1 || fancy_h)) {
    const int r = y >> 1, rn = (y & 1) ? min(r + 1, chh - 1) : max(r - 1, 0);
    if (fh == 1) return (3 * pl[(int64_t)r * pw + x] + pl[(int64_t)rn * pw + x] + 1 + (y & 1)) >> 2;
    const int cx = x >> 1, xn = (x & 1) ? min(cx + 1, cw - 1) : max(cx - 1, 0);
    const int near = 3 * pl[(int64_t)r * pw + cx] + pl[(int64_t)rn * pw + cx];
    const int far = 3 * pl[(int64_t)r * pw + xn] + pl[(int64_t)rn * pw + xn];
    return (3 * near + far + 8 - (x & 1)) >> 4;
  }
  if (fv == 1 && fancy_h) {
    const int cx = x >> 1, xn = (x & 1) ? min(cx + 1, cw - 1) : max(cx - 1, 0);
    const uint8_t* row = pl + (int64_t)y * pw;
    return (3 * row[cx] + row[xn] + 1 + (x & 1)) >> 2;
  }
  return pl[(int64_t)(y / fv) * pw + x / fh];
}

// The decoded pixel (sy, sx) that output pixel (oy, ox) shows under the EXIF orientation.
__device__ __forceinline__ void oriented_source(const DecFile& f, int oy, int ox, int& sy, int& sx) {
  sy = oy;
  sx = ox;
  switch (f.orient) {
    case 2: sx = f.w - 1 - ox; break;
    case 3: sy = f.h - 1 - oy; sx = f.w - 1 - ox; break;
    case 4: sy = f.h - 1 - oy; break;
    case 5: sy = ox; sx = oy; break;
    case 6: sy = f.h - 1 - ox; sx = oy; break;
    case 7: sy = f.h - 1 - ox; sx = f.w - 1 - oy; break;
    case 8: sy = ox; sx = f.w - 1 - oy; break;
    default: break;
  }
}

// jdcolor.c's ycc_rgb_convert (tables FIX(x) = x * 2^16 rounded), cb and cr centred, clamped.
__device__ __forceinline__ void ycc_rgb(int y, int cb, int cr, int& r, int& g, int& b) {
  r = y + ((91881 * cr + 32768) >> 16);
  b = y + ((116130 * cb + 32768) >> 16);
  g = y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  r = min(max(r, 0), 255);
  g = min(max(g, 0), 255);
  b = min(max(b, 0), 255);
}

// Gray files and YCbCr files whose luma is not upsampled and whose two chroma planes share their
// factors: every file the plain decoder takes.
__global__ void __launch_bounds__(kPixThreads) color_kernel(DecParams p) {
  const DecFile& f = p.f[blockIdx.y];
  const int64_t i = (int64_t)blockIdx.x * kPixThreads + threadIdx.x;
  if (f.general || i >= (int64_t)f.oh * f.ow) return;
  const int oy = (int)(i / f.ow), ox = (int)(i - (int64_t)oy * f.ow);
  int sy, sx;
  oriented_source(f, oy, ox, sy, sx);
  const int y = p.s[f.plane[0] + (int64_t)sy * f.pw[0] + sx];
  int b = y, g = y, r = y;
  if (f.ncomp == 3) {
    const int fh = f.uh[1], fv = f.uv[1];
    const int cb = chroma_at(p.s + f.plane[1], f.pw[1], f.cw[1], f.chh[1], fh, fv, f.fancy, sy, sx) - 128;
    const int cr = chroma_at(p.s + f.plane[2], f.pw[2], f.cw[2], f.chh[2], fh, fv, f.fancy, sy, sx) - 128;
    ycc_rgb(y, cb, cr, r, g, b);
  }
  uint8_t* o = f.out + (int64_t)oy * f.pitch + 3 * (int64_t)ox;
  o[0] = (uint8_t)b;
  o[1] = (uint8_t)g;
  o[2] = (uint8_t)r;
}

// The other files (f.general): each component upsampled by its own factors (jinit_upsampler's
// rule, chroma_at), then its colour space to BGR as cv2 reads it.  RGB: the planes as they are.
// YCbCr: as above.  CMYK and YCCK: libjpeg's CMYK output (YCCK through ycck_cmyk_convert: C, M, Y
// = 255 - the clamped YCbCr->RGB, K unchanged), then cv2's icvCvt_CMYK2BGR: B = K - ((255 - Y) *
// K >> 8), and so on.
__global__ void __launch_bounds__(kPixThreads) color_any_kernel(DecParams p) {
  const DecFile& f = p.f[blockIdx.y];
  const int64_t i = (int64_t)blockIdx.x * kPixThreads + threadIdx.x;
  if (!f.general || i >= (int64_t)f.oh * f.ow) return;
  const int oy = (int)(i / f.ow), ox = (int)(i - (int64_t)oy * f.ow);
  int sy, sx;
  oriented_source(f, oy, ox, sy, sx);
  int v[kMaxComps] = {0, 0, 0, 0};
#pragma unroll
  for (int c = 0; c < kMaxComps; ++c)
    if (c < f.ncomp)
      v[c] = chroma_at(p.s + f.plane[c], f.pw[c], f.cw[c], f.chh[c], f.uh[c], f.uv[c], f.fancy, sy, sx);
  int r = v[0], g = v[1], b = v[2];
  if (f.space == kYcc || f.space == kYcck) ycc_rgb(v[0], v[1] - 128, v[2] - 128, r, g, b);
  if (f.space == kCmyk || f.space == kYcck) {
    const int k = v[3];
    const int cc = f.space == kCmyk ? v[0] : 255 - r, m = f.space == kCmyk ? v[1] : 255 - g,
              yy = f.space == kCmyk ? v[2] : 255 - b;
    r = k - ((255 - cc) * k >> 8);
    g = k - ((255 - m) * k >> 8);
    b = k - ((255 - yy) * k >> 8);
  }
  uint8_t* o = f.out + (int64_t)oy * f.pitch + 3 * (int64_t)ox;
  o[0] = (uint8_t)b;
  o[1] = (uint8_t)g;
  o[2] = (uint8_t)r;
}

// ---- host: parsing -----------------------------------------------------------------------------------
struct Comp {
  int id, h, v, tq, td, ta;
};
struct Parsed {
  sqdet_jpeg_info info;
  Comp comp[kMaxComps];
  int hmax, vmax;                      // the largest sampling factors (1 for gray)
  Space space;
  uint16_t qt[4][64];                  // natural order
  bool have_q[4], have_dc[4], have_ac[4];
  uint8_t dc_bits[4][16], ac_bits[4][16];
  uint8_t dc_vals[4][256], ac_vals[4][256];
  bool progressive;                    // SOF2 (parse with progressive = true only)
  int64_t first_sos;                   // SOF2: the first SOS marker's offset
  bool wide_mcu;                       // SOF2: more than 10 blocks in the frame's MCU
  int reduce;                          // the scale it decodes at: 1 / reduce
};

int u16(const uint8_t* b, int64_t i) { return (b[i] << 8) | b[i + 1]; }

// As cv2 reads it: the first Orientation (0x0112) entry of IFD0, its u16 at entry offset 8 in the
// TIFF byte order whatever the entry's type and count, with only the entry's bytes [0, 10) needed
// inside the segment; a value outside 1..8 means 1.
int exif_orientation(const uint8_t* s, int64_t n) {
  if (n < 14 || memcmp(s, "Exif\0\0", 6) != 0) return 1;
  const uint8_t* t = s + 6;
  const int64_t tn = n - 6;
  bool le;
  if (t[0] == 'I' && t[1] == 'I') le = true;
  else if (t[0] == 'M' && t[1] == 'M') le = false;
  else return 1;
  auto rd = [&](int64_t i, int k) -> int64_t {
    if (i < 0 || i + k > tn) return -1;
    int64_t v = 0;
    for (int j = 0; j < k; ++j) v |= (int64_t)t[i + (le ? j : k - 1 - j)] << (8 * j);
    return v;
  };
  if (rd(2, 2) != 42) return 1;
  const int64_t ifd = rd(4, 4);
  const int64_t count = rd(ifd, 2);
  if (ifd < 0 || count < 0) return 1;
  for (int64_t e = 0; e < count; ++e) {
    const int64_t q = ifd + 2 + 12 * e;
    if (q + 10 > tn) break;
    if (rd(q, 2) == 0x0112) {
      const int64_t o = rd(q + 8, 2);
      return o >= 1 && o <= 8 ? (int)o : 1;
    }
  }
  return 1;
}

// jpeg.jpeg_info reports these words; the oracles' REASONS are tested equal to them
const char* kReasons[] = {"ok", "malformed or truncated header", "progressive", "arithmetic coding",
                          "lossless", "not 8-bit samples", "not 1 or 3 components",
                          "RGB-coded", "unsupported sampling",
                          "zero height or width", "larger than cv2 decodes",
                          "scan script libjpeg rejects", "scan script libjpeg warns on or overwrites",
                          "block-smoothed by libjpeg", "more than 256 scans",
                          "more than 2^30 coded pixels, which cv2 decodes at this scale",
                          "sampling libjpeg rejects"};

// The largest file cv2.imdecode decodes: libjpeg's JPEG_MAX_DIMENSION per side, and cv2's default
// CV_IO_MAX_IMAGE_PIXELS (it raises above that many pixels).
constexpr int kMaxSide = 65500;
constexpr int64_t kMaxPixels = int64_t{1} << 30;

// libjpeg's checks of a Huffman table a scan uses: no length's codes run past its all-ones code,
// and a DC table's symbols are categories 0..15.
bool huff_ok(const uint8_t* bits, const uint8_t* vals, bool dc) {
  int code = 0, count = 0;
  for (int l = 1; l <= 16; ++l) {
    code += bits[l - 1];
    count += bits[l - 1];
    if (code >= (1 << l)) return false;
    code <<= 1;
  }
  for (int k = 0; dc && k < count; ++k)
    if (vals[k] > 15) return false;
  return true;
}

// One marker segment: its marker, where the marker starts and its body.
struct Segment {
  int m;
  int64_t at;
  const uint8_t* body;
  int bn;
};

// Reads the marker segment at i, after any fill bytes, and moves i past it; the reason
// (SQDET_JPEG_*).  A standalone marker (SOI, EOI, RSTn, TEM) or a length past the end is malformed.
// With `eoi_ends`, the end of the data or an EOI there is not: it reads as s.m = EOI.
int next_segment(const uint8_t* b, int64_t n, int64_t& i, bool eoi_ends, Segment& s) {
  while (i + 1 < n && b[i] == 0xFF && b[i + 1] == 0xFF) ++i;
  if (eoi_ends && i >= n) {
    s.m = 0xD9;
    return SQDET_JPEG_OK;
  }
  if (i + 2 > n || b[i] != 0xFF) return SQDET_JPEG_MALFORMED;
  s.at = i;
  s.m = b[i + 1];
  i += 2;
  if (eoi_ends && s.m == 0xD9) return SQDET_JPEG_OK;
  if (s.m == 0xD8 || s.m == 0xD9 || (s.m >= 0xD0 && s.m <= 0xD7) || s.m == 0x01) return SQDET_JPEG_MALFORMED;
  if (i + 2 > n) return SQDET_JPEG_MALFORMED;
  const int len = u16(b, i);
  if (len < 2 || i + len > n) return SQDET_JPEG_MALFORMED;
  s.body = b + i + 2;
  s.bn = len - 2;
  i += len;
  return SQDET_JPEG_OK;
}

// A DQT or DHT segment's tables into P; the reason.  Other segments are the caller's.
int read_tables(const Segment& s, Parsed& P) {
  const uint8_t* body = s.body;
  const int bn = s.bn;
  if (s.m == 0xDB) {
    for (int j = 0; j < bn;) {
      const int pq = body[j] >> 4, tq = body[j] & 15, size = pq ? 128 : 64;
      if (pq > 1 || tq > 3 || j + 1 + size > bn) return SQDET_JPEG_MALFORMED;
      for (int k = 0; k < 64; ++k)
        P.qt[tq][kNatural[k]] = pq ? (uint16_t)u16(body, j + 1 + 2 * k) : body[j + 1 + k];
      P.have_q[tq] = true;
      j += 1 + size;
    }
  } else if (s.m == 0xC4) {
    for (int j = 0; j < bn;) {
      if (j + 17 > bn) return SQDET_JPEG_MALFORMED;
      const int tc = body[j] >> 4, th = body[j] & 15;
      int cnt = 0;
      for (int l = 0; l < 16; ++l) cnt += body[j + 1 + l];
      if (tc > 1 || th > 3 || cnt > 256 || j + 17 + cnt > bn) return SQDET_JPEG_MALFORMED;
      memcpy(tc ? P.ac_bits[th] : P.dc_bits[th], body + j + 1, 16);
      memcpy(tc ? P.ac_vals[th] : P.dc_vals[th], body + j + 17, (size_t)cnt);
      (tc ? P.have_ac : P.have_dc)[th] = true;
      j += 17 + cnt;
    }
  }
  return SQDET_JPEG_OK;
}

// The headers up to the first SOS, for a decode at scale 1 / reduce; the reason (SQDET_JPEG_*) and
// what was read.  With `progressive`, an SOF2 frame is read as SOF0's is and the first SOS is left
// to parse_scans.  With `any_layout`, 4 components, the RGB, CMYK and YCCK colour spaces and every
// sampling libjpeg decodes are read too; the other sampling is SQDET_JPEG_BAD_SAMPLING.
int parse(const uint8_t* b, int64_t n, Parsed& P, bool progressive, int reduce, bool any_layout) {
  memset(&P, 0, sizeof(P));
  P.reduce = reduce;
  sqdet_jpeg_info& I = P.info;
  I.orientation = 1;
  if (n < 4 || b[0] != 0xFF || b[1] != 0xD8) return SQDET_JPEG_MALFORMED;
  int adobe = -1, ncomp = 0;
  bool frame = false, exif = false, jfif = false;
  int64_t i = 2;
  for (;;) {
    Segment s;
    if (const int r = next_segment(b, n, i, false, s)) return r;
    if (const int r = read_tables(s, P)) return r;
    const int m = s.m, bn = s.bn;
    const uint8_t* body = s.body;
    if ((m == 0xC2 && !progressive) || m == 0xC6 || m == 0xCA || m == 0xCE) return SQDET_JPEG_PROGRESSIVE;
    if (m == 0xC9 || m == 0xCB || m == 0xCD || m == 0xCF) return SQDET_JPEG_ARITHMETIC;
    if (m == 0xC3 || m == 0xC7) return SQDET_JPEG_LOSSLESS;
    if (m == 0xC5) return SQDET_JPEG_PROGRESSIVE;
    if (m == 0xC0 || m == 0xC1 || m == 0xC2) {
      if (frame || bn < 6) return SQDET_JPEG_MALFORMED;
      P.progressive = m == 0xC2;
      I.coded_height = u16(body, 1);
      I.coded_width = u16(body, 3);
      ncomp = body[5];
      if (body[0] != 8) return SQDET_JPEG_PRECISION;
      if (bn != 6 + 3 * ncomp) return SQDET_JPEG_MALFORMED;
      if (ncomp != 1 && ncomp != 3 && !(any_layout && ncomp == 4)) return SQDET_JPEG_COMPONENTS;
      I.components = ncomp;
      for (int k = 0; k < ncomp; ++k) {
        Comp& c = P.comp[k];
        c.id = body[6 + 3 * k];
        c.h = body[7 + 3 * k] >> 4;
        c.v = body[7 + 3 * k] & 15;
        c.tq = body[8 + 3 * k];
        if (c.tq > 3 || c.h < 1 || c.h > 4 || c.v < 1 || c.v > 4) return SQDET_JPEG_MALFORMED;
      }
      if (I.coded_height == 0 || I.coded_width == 0) return SQDET_JPEG_SIZE;
      // libjpeg's side limit holds at every scale; cv2's pixel limit is on the reduced size, but
      // more coded pixels than that is refused before anything is sized from them
      if (I.coded_height > kMaxSide || I.coded_width > kMaxSide) return SQDET_JPEG_TOO_LARGE;
      if ((int64_t)I.coded_height * I.coded_width > kMaxPixels)
        return (int64_t)((I.coded_height + reduce - 1) / reduce) * ((I.coded_width + reduce - 1) / reduce) > kMaxPixels
                   ? SQDET_JPEG_TOO_LARGE : SQDET_JPEG_CODED_TOO_LARGE;
      P.hmax = P.vmax = 1;
      int mcu_blocks = 0;
      for (int k = 0; ncomp > 1 && k < ncomp; ++k) {
        P.hmax = std::max(P.hmax, P.comp[k].h);
        P.vmax = std::max(P.vmax, P.comp[k].v);
        mcu_blocks += P.comp[k].h * P.comp[k].v;
      }
      if (ncomp > 1 && any_layout) {
        // jinit_upsampler takes integral ratios only; a sequential file's one scan is
        // interleaved, and jdinput.c's per_scan_setup allows 10 blocks per MCU
        for (int k = 0; k < ncomp; ++k)
          if (P.hmax % P.comp[k].h || P.vmax % P.comp[k].v) return SQDET_JPEG_BAD_SAMPLING;
        // a progressive frame's MCU may be wider, if no interleaved scan is: parse_scans decides
        if (m != 0xC2 && mcu_blocks > kMaxBlocks) return SQDET_JPEG_BAD_SAMPLING;
        P.wide_mcu = mcu_blocks > kMaxBlocks;
      } else if (ncomp == 3) {
        const int h = P.comp[0].h, v = P.comp[0].v;
        const bool luma_ok = (h == 1 && v == 1) || (h == 2 && v == 1) || (h == 1 && v == 2) ||
                             (h == 2 && v == 2) || (h == 4 && v == 1);
        for (int k = 1; k < 3; ++k)
          if (P.comp[k].h != 1 || P.comp[k].v != 1) return SQDET_JPEG_SAMPLING;
        if (!luma_ok) return SQDET_JPEG_SAMPLING;
      }
      frame = true;
    } else if (m == 0xDD) {
      if (bn != 2) return SQDET_JPEG_MALFORMED;
      I.restart_interval = u16(body, 0);
    } else if (m == 0xE1 && !exif && bn >= 6 && memcmp(body, "Exif\0\0", 6) == 0) {
      exif = true;
      I.orientation = exif_orientation(body, bn);
    } else if (m == 0xE0 && bn >= 14 && memcmp(body, "JFIF\0", 5) == 0) {
      jfif = true;
    } else if (m == 0xEE && bn >= 12 && memcmp(body, "Adobe", 5) == 0) {
      adobe = body[11];
    } else if (m == 0xDA) {
      if (!frame || bn < 1) return SQDET_JPEG_MALFORMED;
      if (!P.progressive) {                 // the one scan of a sequential file
        const int ns = body[0];
        if (bn != 4 + 2 * ns) return SQDET_JPEG_MALFORMED;
        if (ns != ncomp) return SQDET_JPEG_SAMPLING;
        for (int k = 0; k < ns; ++k) {
          Comp& c = P.comp[k];
          if (body[1 + 2 * k] != c.id) return SQDET_JPEG_SAMPLING;
          c.td = body[2 + 2 * k] >> 4;
          c.ta = body[2 + 2 * k] & 15;
          if (c.td > 3 || c.ta > 3 || !P.have_dc[c.td] || !P.have_ac[c.ta] || !P.have_q[c.tq])
            return SQDET_JPEG_MALFORMED;
          if (!huff_ok(P.dc_bits[c.td], P.dc_vals[c.td], true) || !huff_ok(P.ac_bits[c.ta], P.ac_vals[c.ta], false))
            return SQDET_JPEG_MALFORMED;
        }
        if (body[1 + 2 * ns] != 0 || body[2 + 2 * ns] != 63 || body[3 + 2 * ns] != 0)
          return SQDET_JPEG_MALFORMED;
      }
      // libjpeg's colour space of 3 components: YCbCr after a JFIF APP0; else as an Adobe APP14's
      // transform says (0: RGB); else RGB for component ids 'R', 'G', 'B'.  Of 4: as an Adobe
      // APP14's transform says (0: CMYK, anything else YCCK), CMYK without one
      if (ncomp == 3 && !jfif &&
          (adobe >= 0 ? adobe == 0
                      : P.comp[0].id == 'R' && P.comp[1].id == 'G' && P.comp[2].id == 'B')) {
        if (!any_layout) return SQDET_JPEG_COLOR_TRANSFORM;
        P.space = kRgb;
      } else {
        P.space = ncomp == 1 ? kGray : ncomp == 3 ? kYcc : adobe > 0 ? kYcck : kCmyk;
      }
      if (P.progressive) P.first_sos = s.at;
      else I.scan_offset = i;
      I.h_samp = ncomp == 1 ? 1 : P.comp[0].h;
      I.v_samp = ncomp == 1 ? 1 : P.comp[0].v;
      const bool swap = I.orientation >= 5;
      const int rh = (I.coded_height + reduce - 1) / reduce, rw = (I.coded_width + reduce - 1) / reduce;
      I.height = swap ? rw : rh;
      I.width = swap ? rh : rw;
      I.supported = 1;
      return SQDET_JPEG_OK;
    }
  }
}

void build_tab(const uint8_t* bits, const uint8_t* vals, HuffTab& t) {
  memset(&t, 0, sizeof(t));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    t.maxcode[l] = -1;
    const int first_k = k, first_code = code;
    for (int j = 0; j < bits[l - 1]; ++j) {
      if (code < (1 << l)) {
        if (l <= kFastBits) {
          const int lo = code << (kFastBits - l), hi = (code + 1) << (kFastBits - l);
          for (int e = lo; e < hi; ++e) t.fast[e] = (uint16_t)(l << 8 | vals[k]);
        }
        t.maxcode[l] = code;
      }
      ++code;
      ++k;
    }
    t.valoff[l] = first_k - first_code;
    code <<= 1;
  }
  memcpy(t.vals, vals, 256);
}

// One file's layout: sizes that follow from its headers alone.  isz, uh and uv are each
// component's IDCT size and upsampling factors at the file's scale; pw and ph its plane's.
struct Layout {
  int mcu_cols, mcu_rows, mcus, bpm, restart, intervals, chunks, blocks, sub_max;
  int isz[kMaxComps], uh[kMaxComps], uv[kMaxComps];
  int pw[kMaxComps], ph[kMaxComps];
  int64_t raw_len;
};

Layout layout(const Parsed& P, int64_t file_len, int sub_bits) {
  const sqdet_jpeg_info& I = P.info;
  Layout L{};
  const int H = I.coded_height, W = I.coded_width;
  const bool gray = I.components == 1;
  const int hmax = P.hmax, vmax = P.vmax;
  L.mcu_cols = (W + 8 * hmax - 1) / (8 * hmax);
  L.mcu_rows = (H + 8 * vmax - 1) / (8 * vmax);
  L.bpm = 0;
  for (int c = 0; c < I.components; ++c) L.bpm += gray ? 1 : P.comp[c].h * P.comp[c].v;
  // jpeg_calc_output_dimensions: luma's IDCT is m = 8 / reduce; another component's doubles
  // from m while below 8 and both divisibility conditions hold (4:2:0 chroma: 2m, the others m)
  const int m = 8 / P.reduce;
  for (int c = 0; c < I.components; ++c) {
    const int h = gray ? 1 : P.comp[c].h, v = gray ? 1 : P.comp[c].v;
    int n = m;
    while (n < 8 && (hmax * m) % (h * n * 2) == 0 && (vmax * m) % (v * n * 2) == 0) n *= 2;
    L.isz[c] = n;
    L.uh[c] = hmax * m / (h * n);
    L.uv[c] = vmax * m / (v * n);
    L.pw[c] = L.mcu_cols * h * n;
    L.ph[c] = L.mcu_rows * v * n;
  }
  L.mcus = L.mcu_cols * L.mcu_rows;
  L.blocks = L.mcus * L.bpm;
  L.restart = I.restart_interval ? std::min(I.restart_interval, L.mcus) : L.mcus;
  L.intervals = (L.mcus + L.restart - 1) / L.restart;
  L.raw_len = file_len - I.scan_offset;
  L.chunks = (int)std::max<int64_t>(1, (L.raw_len + kChunk - 1) / kChunk);
  L.sub_max = (int)((L.raw_len * 8 + sub_bits - 1) / sub_bits) + L.intervals;
  return L;
}

// Whether color_any_kernel converts the file: anything but gray and YCbCr with luma at the frame's
// size and both chroma planes upsampled alike.
bool general_layout(const Parsed& P, const Layout& L) {
  return !(P.space == kGray || (P.space == kYcc && L.uh[0] == 1 && L.uv[0] == 1 &&
                                L.uh[1] == L.uh[2] && L.uv[1] == L.uv[2]));
}

// The fields of a file's descriptor that follow from its frame header, its quantization tables
// (as the components name them) included.
void describe(const Parsed& P, const Layout& L, DecFile& f) {
  const sqdet_jpeg_info& I = P.info;
  f.h = (I.coded_height + P.reduce - 1) / P.reduce;
  f.w = (I.coded_width + P.reduce - 1) / P.reduce;
  f.oh = I.height;
  f.ow = I.width;
  f.ncomp = I.components;
  f.orient = I.orientation;
  f.mcu_cols = L.mcu_cols;
  f.mcus = L.mcus;
  f.bpm = L.bpm;
  f.restart = L.restart;
  f.intervals = L.intervals;
  f.raw_len = (int32_t)L.raw_len;
  f.chunks = L.chunks;
  f.blocks = L.blocks;
  f.sub_max = L.sub_max;
  f.sub_bits = g_sub_bits;
  f.fancy = P.reduce < 8;              // jinit_upsampler: fancy only while luma's IDCT is above 1
  f.space = P.space;
  f.general = general_layout(P, L);
  int u = 0;
  for (int c = 0; c < I.components; ++c) {
    const Comp& cp = P.comp[c];
    const int hc = I.components == 1 ? 1 : cp.h, vc = I.components == 1 ? 1 : cp.v;
    f.ch[c] = (int8_t)hc;
    f.cv[c] = (int8_t)vc;
    for (int by = 0; by < vc; ++by)
      for (int bx = 0; bx < hc; ++bx, ++u) {
        f.bcomp[u] = (int8_t)c;
        f.bdy[u] = (int8_t)by;
        f.bdx[u] = (int8_t)bx;
      }
    f.isz[c] = (int8_t)L.isz[c];
    f.uh[c] = (int8_t)L.uh[c];
    f.uv[c] = (int8_t)L.uv[c];
    f.pw[c] = L.pw[c];
    f.ph[c] = L.ph[c];
    // libjpeg's downsampled_width / _height at this scale
    const int hmax = P.hmax, vmax = P.vmax;
    f.cw[c] = (int)(((int64_t)I.coded_width * hc * L.isz[c] + 8 * hmax - 1) / (8 * hmax));
    f.chh[c] = (int)(((int64_t)I.coded_height * vc * L.isz[c] + 8 * vmax - 1) / (8 * vmax));
    for (int k = 0; k < 64; ++k) f.q[c][k] = (int16_t)P.qt[cp.tq][k];
  }
}

// The decode calls' checks of everything but the files, in their order; info[i] is file i's.
int check_decode_args(const std::string& name, int n, const sqdet_jpeg_info* const* info,
                      uint8_t* const* out_planes, const int64_t* out_pitches, void* staging_pinned,
                      int64_t staging_bytes, int64_t staging_need, void* scratch_dev,
                      int64_t scratch_bytes, int64_t scratch_need, int32_t* status_dev,
                      const std::string& staging_fn, const std::string& scratch_fn) {
  if ((uintptr_t)scratch_dev % 256) return fail(SQDET_ERR_INVALID_ARG, name + ": scratch_dev must be 256-byte aligned");
  if ((uintptr_t)status_dev % alignof(int32_t))
    return fail(SQDET_ERR_INVALID_ARG, name + ": status_dev must be 4-byte aligned");
  if (staging_bytes < staging_need)
    return fail(SQDET_ERR_INVALID_ARG, name + ": staging_bytes is below " + staging_fn);
  if (scratch_bytes < scratch_need)
    return fail(SQDET_ERR_INVALID_ARG, name + ": scratch_bytes is below " + scratch_fn);
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, staging_pinned) != cudaSuccess || attr.type != cudaMemoryTypeHost) {
    (void)cudaGetLastError();
    return fail(SQDET_ERR_INVALID_ARG, name + ": staging_pinned is not page-locked host memory");
  }
  if (!out_planes[0]) return fail(SQDET_ERR_INVALID_ARG, name + ": output 0 is null");
  const int device = pointer_device(out_planes[0]);
  if (device < 0) return fail(SQDET_ERR_INVALID_ARG, name + ": output 0 is not device memory");
  for (int i = 0; i < n; ++i) {
    const sqdet_jpeg_info& I = *info[i];
    const std::string which = name + ": output " + std::to_string(i);
    if (!out_planes[i]) return fail(SQDET_ERR_INVALID_ARG, which + " is null");
    if (out_pitches[i] < 3 * (int64_t)I.width) return fail(SQDET_ERR_INVALID_ARG, which + ": pitch below 3 * width");
    const int64_t bytes = (int64_t)(I.height - 1) * out_pitches[i] + 3 * (int64_t)I.width;
    if (!device_range_ok(out_planes[i], bytes, device))
      return fail(SQDET_ERR_INVALID_ARG, which + " is not inside one device allocation on output 0's device");
  }
  if (!device_range_ok(status_dev, (int64_t)n * 4, device) ||
      !device_range_ok(scratch_dev, scratch_bytes, device))
    return fail(SQDET_ERR_INVALID_ARG, name + ": status_dev or scratch_dev is not inside one device "
                                              "allocation on output 0's device");
  return SQDET_OK;
}

// ==== progressive (SOF2) files ============================================================
// libjpeg reads every scan into a whole-image coefficient buffer and runs its output pass once
// the file has ended, so a progressive file decodes to what a sequential file of the final
// coefficients decodes to; idct_kernel and color_kernel run unchanged.  The host parses every
// SOS with the tables in force at that point, removes the stuffing and splits each scan's data
// at its RSTn markers, and packs it all into the staging.  Then, on the stream:
//   1. prog_seq (first)  every first scan (Ah = 0, DC and AC) of every file: one warp per
//                        (scan, restart interval) decodes it in order; first scans write disjoint
//                        (component, coefficient) sets and read none, so they are independent
//   2. prog_dc_refine    every DC refinement scan: one thread per block ORs bit Al into its DC
//   3. prog_seq (refine) AC refinements, one launch per depth of the longest chain: the d-th
//                        refinement scan of each component of each file, one warp per
//                        (scan, interval), which keeps each block's nonzero coefficients as a
//                        mask so a run and the correction bits it passes are found with
//                        popcount and bit scans
// then idct and color.  Every loop is bounded by host-known sizes; corrupt data sets a negative
// status for its file only.
constexpr int kMaxScans = 256;
// one (scan, interval) per CTA of one warp, decoded by its first lane: items that shared a warp
// would run their divergent walks one after another
constexpr int kProgThreads = 32;
constexpr int kScanPad = 32;          // zero bytes after each scan's clean data

struct ProgScan {
  int32_t file, ss, se, ah, al;
  int32_t nb;                         // blocks per unit: the MCU's of the scan's components, or 1
  int32_t units, per, intervals;      // units in the scan and per restart interval
  int32_t cols;                       // one-component scans: the component's block columns
  int32_t single, bad;                // one-component scan; an RSTn out of sequence or missing
  int8_t bc[10], bu[10], bt[10];      // per block of a unit: component, block of the MCU, table
  int64_t tabs, clean, ist;
};

struct ProgParams {
  DecFile* f;
  const ProgScan* sc;
  const int2* items;                  // (scan, interval) or, for prog_dc_refine, (scan, 0)
  int nitems;
  uint8_t* s;
  int32_t* status;
};

// The coefficient block of block j of unit u of scan S.
__device__ __forceinline__ int64_t unit_block(const DecFile& f, const ProgScan& S, int u, int j) {
  if (!S.single) return (int64_t)u * f.bpm + S.bu[j];
  const int by = u / S.cols, bx = u - by * S.cols;
  if (f.ncomp == 1) return (int64_t)by * f.mcu_cols + bx;
  const int c = S.bc[0], h = f.ch[c], v = f.cv[c];
  return ((int64_t)(by / v) * f.mcu_cols + bx / h) * f.bpm + S.bu[0] + (by % v) * h + bx % h;
}

__device__ __forceinline__ int16_t jcoef(int v) { return (int16_t)v; }

// Reads one correction bit for each set bit of `corr` (zigzag positions, in order) and applies
// it as decode_mcu_AC_refine does.
__device__ __forceinline__ int corrections(const uint8_t* clean, int p, int16_t* blk, uint64_t corr,
                                           int p1, int m1) {
#pragma unroll 1
  while (corr) {
    const int take = min(__popcll(corr), 32);
    const uint32_t w = peek32(clean, p);
    p += take;
#pragma unroll 1
    for (int i = 0; i < take; ++i) {
      const int k = __ffsll((long long)corr) - 1;
      corr &= corr - 1;
      if ((w >> (31 - i)) & 1) {
        int16_t& c = blk[kNaturalDev[k]];
        if ((c & p1) == 0) c = jcoef(c + (c >= 0 ? p1 : m1));
      }
    }
  }
  return p;
}

// One restart interval of a Huffman-coded scan; 0 or a negative status.
__device__ int prog_interval(const DecFile& f, const ProgScan& S, const uint8_t* clean,
                             const HuffTab* tabs, int16_t* coef, int u0, int u1, int p, int end) {
  if (S.ss == 0) {                                       // DC first
    int dc[kMaxComps] = {0, 0, 0, 0};
#pragma unroll 1
    for (int u = u0; u < u1; ++u) {
#pragma unroll 1
      for (int j = 0; j < S.nb; ++j) {
        const uint32_t bits = peek32(clean, p);
        int len;
        const int s = huff_decode(tabs[S.bt[j]], bits, len);
        if (!len) return -4;
        const uint32_t extra = s ? (bits << len) >> (32 - s) : 0;
        p += len + s;
        const int c = S.bc[j];
        dc[c] += extend(extra, s);
        coef[unit_block(f, S, u, j) * 64] = jcoef((int)((unsigned)dc[c] << S.al));
        if (p > end) return -7;
      }
    }
    return 0;
  }
  const HuffTab& t = tabs[0];
  int eobrun = 0;
  if (S.ah == 0) {                                       // AC first
#pragma unroll 1
    for (int u = u0; u < u1; ++u) {
      if (eobrun) {
        --eobrun;
        continue;
      }
      int16_t* blk = coef + unit_block(f, S, u, 0) * 64;
#pragma unroll 1
      for (int k = S.ss; k <= S.se;) {
        const uint32_t bits = peek32(clean, p);
        int len;
        const int sym = huff_decode(t, bits, len);
        if (!len) return -4;
        const int r = sym >> 4, s = sym & 15;
        if (s) {
          k += r;
          if (k > S.se) return -5;
          blk[kNaturalDev[k]] = jcoef((int)((unsigned)extend((bits << len) >> (32 - s), s) << S.al));
          p += len + s;
          ++k;
        } else if (r == 15) {
          p += len;
          k += 16;
          if (k > S.se + 1) return -5;
        } else {
          eobrun = (1 << r) + (r ? (int)((bits << len) >> (32 - r)) : 0) - 1;
          p += len + r;
          break;
        }
        if (p > end) return -7;
      }
      if (p > end) return -7;
    }
    return eobrun ? -9 : 0;
  }
  // AC refinement
  const int p1 = 1 << S.al, m1 = (int)(~0u << S.al);
  const uint64_t band = (~0ull >> (63 - S.se)) & (~0ull << S.ss);
#pragma unroll 1
  for (int u = u0; u < u1; ++u) {
    int16_t* blk = coef + unit_block(f, S, u, 0) * 64;
    uint64_t nat = 0;                                    // nonzero coefficients, natural order
    const int4* src = reinterpret_cast<const int4*>(blk);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int4 v = src[i];
      const int32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        nat |= (uint64_t)((w[e] & 0xFFFF) != 0) << (8 * i + 2 * e);
        nat |= (uint64_t)((w[e] >> 16) != 0) << (8 * i + 2 * e + 1);
      }
    }
    uint64_t nz = 0;                                     // the same in zigzag order, in the band
#pragma unroll 1
    for (int k = S.ss; k <= S.se; ++k) nz |= ((nat >> kNaturalDev[k]) & 1) << k;
    int k = S.ss;
    if (eobrun == 0) {
#pragma unroll 1
      while (k <= S.se) {
        const uint32_t bits = peek32(clean, p);
        int len;
        const int sym = huff_decode(t, bits, len);
        if (!len) return -4;
        int r = sym >> 4;
        const int s = sym & 15;
        p += len;
        int val = 0;
        if (s) {
          if (s != 1) return -10;
          val = (bits << len) >> 31 ? p1 : m1;
          p += 1;
        } else if (r != 15) {
          eobrun = (1 << r) + (r ? (int)((bits << len) >> (32 - r)) : 0);
          p += r;
          break;
        }
        // the target is the (r + 1)-th coefficient still zero from k on; the nonzero ones
        // before it take a correction bit each
        uint64_t zeros = ~nz & band & (~0ull << k);
        if (__popcll(zeros) <= r) return -5;
#pragma unroll 1
        for (; r > 0; --r) zeros &= zeros - 1;
        const int target = __ffsll((long long)zeros) - 1;
        p = corrections(clean, p, blk, nz & (~0ull << k) & ((1ull << target) - 1), p1, m1);
        if (val) blk[kNaturalDev[target]] = jcoef(val);
        k = target + 1;
        if (p > end) return -7;
      }
    }
    if (eobrun > 0) {
      p = corrections(clean, p, blk, k < 64 ? nz & (~0ull << k) : 0, p1, m1);
      --eobrun;
    }
    if (p > end) return -7;
  }
  return eobrun ? -9 : 0;
}

__global__ void __launch_bounds__(kProgThreads) prog_seq_kernel(ProgParams p) {
  const int t = blockIdx.x;
  if (threadIdx.x || t >= p.nitems) return;
  const int2 it = p.items[t];
  const ProgScan& S = p.sc[it.x];
  const DecFile& f = p.f[S.file];
  const int32_t* ist = reinterpret_cast<const int32_t*>(p.s + S.ist);
  const int r = it.y, u0 = r * S.per, u1 = min(S.units, u0 + S.per);
  const int rc = S.bad ? -2
                       : prog_interval(f, S, p.s + S.clean, reinterpret_cast<const HuffTab*>(p.s + S.tabs),
                                       reinterpret_cast<int16_t*>(p.s + f.coef), u0, u1, ist[r] * 8,
                                       ist[r + 1] * 8);
  // p.f[S.file] rather than f: with f here, ptxas gives the kernel 70 registers instead of 55
  if (rc) fail_file(p.status, p.f[S.file], rc);
}

// DC refinement: block g of the scan is bit g - (its interval's first block) of its interval.
__global__ void __launch_bounds__(kPixThreads) prog_dc_refine_kernel(ProgParams p) {
  const ProgScan& S = p.sc[p.items[blockIdx.y].x];
  const DecFile& f = p.f[S.file];
  const int g = blockIdx.x * kPixThreads + threadIdx.x;
  if (g >= S.units * S.nb) return;
  if (S.bad) {                       // its intervals past the markers present have no ist
    fail_file(p.status, f, -2);
    return;
  }
  const int u = g / S.nb, j = g - u * S.nb, r = u / S.per;
  const int32_t* ist = reinterpret_cast<const int32_t*>(p.s + S.ist);
  const int64_t bit = (int64_t)ist[r] * 8 + (int64_t)(g - r * S.per * S.nb);
  if (bit >= (int64_t)ist[r + 1] * 8) {
    fail_file(p.status, f, -7);
    return;
  }
  if ((p.s[S.clean + (bit >> 3)] >> (7 - (bit & 7))) & 1) {
    // two refinement scans of one DC may run at once: OR into the word that holds it
    int16_t* dc = reinterpret_cast<int16_t*>(p.s + f.coef) + unit_block(f, S, u, j) * 64;
    atomicOr(reinterpret_cast<unsigned int*>(dc), (unsigned)(1 << S.al));
  }
}

// ---- host: every scan -------------------------------------------------------------------------
struct PScan {
  int ncomp, comp[kMaxComps], ss, se, ah, al, restart;
  uint8_t bits[kMaxComps][16], vals[kMaxComps][256];   // the tables in force at the scan
  int64_t start, end;                  // its entropy-coded bytes
  int64_t markers;                     // the RSTn markers among them
};
struct Prog {
  std::vector<PScan> scans;
  bool latched[kMaxComps];
  uint16_t q[kMaxComps][64];
};

// The first byte at or after j that starts a marker other than RSTn (or n), and the RSTn markers
// before it.
int64_t data_end(const uint8_t* b, int64_t n, int64_t j, int64_t& markers) {
  markers = 0;
  for (; j < n; ++j) {
    if (b[j] != 0xFF) continue;
    if (j + 1 >= n) return j;
    const int nx = b[j + 1];
    if (nx >= 0xD0 && nx <= 0xD7) ++markers;
    else if (!(nx == 0x00 || nx == 0xFF)) return j;
  }
  return n;
}

// jdcoefct.c's smoothing_ok at the output pass: whether libjpeg block-smooths the file.
bool smoothed(int ncomp, const Prog& G, const int (*cbits)[64]) {
  static const int kQ[10] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24};
  bool useful = false;
  for (int c = 0; c < ncomp; ++c) {
    if (!G.latched[c] || cbits[c][0] < 0) return false;
    for (int k : kQ)
      if (G.q[c][k] == 0) return false;
    for (int k = 1; k < 10; ++k) useful = useful || cbits[c][k] != 0;
  }
  return useful;
}

// The scans of an SOF2 file from its first SOS on (oracle/jpeg_decode_progressive.py restates
// it): the reason (SQDET_JPEG_*) and every scan.
int parse_scans(const uint8_t* b, int64_t n, Parsed& P, Prog& G) {
  G.scans.clear();
  memset(G.latched, 0, sizeof(G.latched));
  memset(G.q, 0, sizeof(G.q));
  const int ncomp = P.info.components;
  int cbits[kMaxComps][64];
  for (auto& row : cbits)
    for (int& x : row) x = -1;
  bool bogus = false, too_many = false;
  int restart = P.info.restart_interval;
  int64_t i = P.first_sos;
  for (;;) {
    Segment s;
    if (const int r = next_segment(b, n, i, !G.scans.empty(), s)) return r;
    if (s.m == 0xD9) break;                              // EOI, or no EOI: the image ends there
    if (const int r = read_tables(s, P)) return r;
    const int m = s.m, bn = s.bn;
    const uint8_t* body = s.body;
    if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) return SQDET_JPEG_MALFORMED;
    if (m == 0xDD) {
      if (bn != 2) return SQDET_JPEG_MALFORMED;
      restart = u16(body, 0);
    } else if (m == 0xDA) {
      if (bn < 1) return SQDET_JPEG_MALFORMED;
      const int ns = body[0];
      if (bn != 4 + 2 * ns || ns < 1 || ns > 4) return SQDET_JPEG_MALFORMED;
      PScan S{};
      S.ncomp = ns;
      int prev = -1;
      for (int k = 0; k < ns; ++k) {
        int c = 0;
        while (c < ncomp && P.comp[c].id != body[1 + 2 * k]) ++c;
        if (c == ncomp) return SQDET_JPEG_MALFORMED;
        if (c <= prev) return SQDET_JPEG_SAMPLING;       // out of the frame's order, or repeated
        prev = S.comp[k] = c;
      }
      // jdinput.c's per_scan_setup: an interleaved scan's MCU is at most 10 blocks
      int scan_blocks = 0;
      for (int k = 0; ns > 1 && k < ns; ++k) scan_blocks += P.comp[S.comp[k]].h * P.comp[S.comp[k]].v;
      if (scan_blocks > kMaxBlocks) return SQDET_JPEG_BAD_SAMPLING;
      S.ss = body[1 + 2 * ns];
      S.se = body[2 + 2 * ns];
      S.ah = body[3 + 2 * ns] >> 4;
      S.al = body[3 + 2 * ns] & 15;
      S.restart = restart;
      for (int k = 0; k < ns; ++k) {                    // latch_quant_tables
        const int c = S.comp[k];
        if (G.latched[c]) continue;
        if (!P.have_q[P.comp[c].tq]) return SQDET_JPEG_MALFORMED;
        memcpy(G.q[c], P.qt[P.comp[c].tq], sizeof(G.q[c]));
        G.latched[c] = true;
      }
      const bool dc_band = S.ss == 0;
      const bool bad = dc_band ? S.se != 0 : (S.ss > S.se || S.se > 63 || ns != 1);
      if ((S.ah != 0 && S.al != S.ah - 1) || S.al > 13 || bad) return SQDET_JPEG_BAD_PROGRESSION;
      for (int k = 0; k < ns; ++k) {
        int* cb = cbits[S.comp[k]];
        if (!dc_band && cb[0] < 0) bogus = true;
        for (int q = S.ss; q <= S.se; ++q) {
          if (S.ah != std::max(cb[q], 0) || (S.ah == 0 && cb[q] >= 0)) bogus = true;
          cb[q] = S.al;
        }
      }
      for (int k = 0; k < ns; ++k) {
        const int td = body[2 + 2 * k] >> 4, ta = body[2 + 2 * k] & 15;
        if (dc_band && S.ah == 0) {
          if (td > 3 || !P.have_dc[td] || !huff_ok(P.dc_bits[td], P.dc_vals[td], true))
            return SQDET_JPEG_MALFORMED;
          memcpy(S.bits[k], P.dc_bits[td], 16);
          memcpy(S.vals[k], P.dc_vals[td], 256);
        } else if (!dc_band) {
          if (ta > 3 || !P.have_ac[ta] || !huff_ok(P.ac_bits[ta], P.ac_vals[ta], false))
            return SQDET_JPEG_MALFORMED;
          memcpy(S.bits[k], P.ac_bits[ta], 16);
          memcpy(S.vals[k], P.ac_vals[ta], 256);
        }
      }
      S.start = i;
      S.end = data_end(b, n, i, S.markers);
      i = S.end;
      // past the cap the scans are still checked, so that a later one libjpeg rejects is
      // reported as libjpeg reports it
      if ((int)G.scans.size() == kMaxScans) too_many = true;
      else G.scans.push_back(S);
    }
    // APPn, COM and anything else: skipped
  }
  if (too_many) return SQDET_JPEG_TOO_MANY_SCANS;
  if (bogus) return SQDET_JPEG_BOGUS_PROGRESSION;
  if (smoothed(ncomp, G, cbits)) return SQDET_JPEG_SMOOTHED;
  // the coefficients are laid out in the frame's MCUs, of at most 10 blocks here; libjpeg decodes
  // such a file, so it goes to cv2
  if (P.wide_mcu) return SQDET_JPEG_SAMPLING;
  P.info.scan_offset = G.scans[0].start;
  return SQDET_JPEG_OK;
}

// How a call decodes: SOF2 files too or not, and at which scale (1 / reduce).
struct Mode {
  bool progressive;
  int reduce;
  bool any_layout;
  const char* suffix;                  // of the entry points' names in messages
};

// A file as the entry points read it: with `progressive`, SOF2 files too, with their scans.
int parse_file(const uint8_t* b, int64_t n, const Mode& mode, Parsed& P, Prog& G) {
  const int reason = parse(b, n, P, mode.progressive, mode.reduce, mode.any_layout);
  if (reason || !P.progressive) return reason;
  return parse_scans(b, n, P, G);
}

// The scan's geometry: its units, blocks per unit and restart interval in units.
void scan_geometry(const Parsed& P, const Layout& L, const PScan& S, ProgScan& D) {
  const int ncomp = P.info.components;
  D.ss = S.ss;
  D.se = S.se;
  D.ah = S.ah;
  D.al = S.al;
  D.single = S.ncomp == 1;
  int uoff[kMaxComps] = {0, 0, 0, 0};
  for (int c = 1; c < ncomp; ++c) uoff[c] = uoff[c - 1] + P.comp[c - 1].h * P.comp[c - 1].v;
  if (D.single) {
    const int c = S.comp[0];
    const int hc = ncomp == 1 ? 1 : P.comp[c].h, vc = ncomp == 1 ? 1 : P.comp[c].v;
    const int hmax = P.hmax, vmax = P.vmax;
    const int64_t cw = ((int64_t)P.info.coded_width * hc + hmax - 1) / hmax;
    const int64_t chh = ((int64_t)P.info.coded_height * vc + vmax - 1) / vmax;
    D.cols = (int)((cw + 7) / 8);
    D.units = D.cols * (int)((chh + 7) / 8);
    D.nb = 1;
    D.bc[0] = (int8_t)c;
    D.bu[0] = (int8_t)(ncomp == 1 ? 0 : uoff[c]);
    D.bt[0] = 0;
  } else {
    D.units = L.mcus;
    D.cols = L.mcu_cols;
    int j = 0;
    for (int k = 0; k < S.ncomp; ++k) {
      const int c = S.comp[k];
      for (int q = 0; q < P.comp[c].h * P.comp[c].v; ++q, ++j) {
        D.bc[j] = (int8_t)c;
        D.bu[j] = (int8_t)(uoff[c] + q);
        D.bt[j] = (int8_t)k;
      }
    }
    D.nb = j;
  }
  D.per = S.restart ? std::min(S.restart, D.units) : D.units;
  // only the intervals the scan's markers delimit are placed, so that the staging follows the
  // file's bytes and not its DRI; a scan with fewer markers than intervals is corrupt
  const int64_t need = (D.units + D.per - 1) / D.per;
  D.intervals = (int)std::min<int64_t>(need, S.markers + 1);
  D.bad = D.intervals < need;
}

// Removes the stuffing of a scan's bytes and splits them at its RSTn markers into clean (ist[r]:
// where interval r starts); whether the markers are in sequence and none is missing.  Markers
// after the last interval's are skipped, as libjpeg skips them.
bool destuff_scan(const uint8_t* b, int64_t start, int64_t end, int intervals, uint8_t* clean,
                  int32_t* ist) {
  int64_t o = 0;
  int r = 0;
  bool ok = true;
  ist[0] = 0;
  for (int64_t j = start; j < end; ++j) {
    if (b[j] != 0xFF) {
      clean[o++] = b[j];
      continue;
    }
    const int nx = j + 1 < end ? b[j + 1] : -1;
    if (nx == 0x00) {
      clean[o++] = 0xFF;
      ++j;
    } else if (nx >= 0xD0 && nx <= 0xD7) {
      if (r + 1 < intervals) {
        ok = ok && nx == 0xD0 + (r & 7);
        ist[r + 1] = (int32_t)o;
      }
      ++r;
      ++j;
    }
  }
  for (int k = std::min(r + 1, intervals); k <= intervals; ++k) ist[k] = (int32_t)o;
  return ok && r + 1 >= intervals;
}

// ---- host: one call ------------------------------------------------------------------------------
// One file of a call: its headers, its layout, its scans (progressive files) and its index in the
// call.
struct Input {
  Parsed P;
  Layout L;
  Prog G;
  int index;
};

// The whole call.  Its sequential files come first, so that the sequential stages' grids run over
// the first nseq descriptors; the progressive stages reach theirs through the work items.
struct Plan {
  std::vector<Input> in;               // the sequential files, then the progressive ones
  int nseq = 0;
  std::vector<DecFile> files;          // in's descriptors, their regions placed
  std::vector<ProgScan> scans;         // every scan of every progressive file, in order
  std::vector<int2> items;             // first-scan items, then DC refinements, then each depth's
  int first = 0, dc_refine = 0;
  std::vector<int> depth;              // AC refinement items per depth
  int reduce = 1;                      // every file's scale: 1 / reduce
  bool general = false;                // some file needs color_any_kernel
  int64_t scan_off = 0, item_off = 0, staging = 0, scratch = 0;
  int64_t marks = 0, marks_bytes = 0, coef = 0, coef_bytes = 0;
};

// Places every region of the call.  The staging holds the file descriptors, the scan descriptors
// and the work items, then each sequential file's Huffman tables and raw bytes (+16 zero bytes of
// padding), then each scan's tables, interval starts and clean data; it is copied to the scratch's
// start.  After it in the scratch come the sequential files' marks (a terminator, then ist), every
// file's coefficients, and then per file: a sequential file's chunk sums, clean stream (padded),
// sbase, entry, exit and counts, and every file's planes.
void place(Plan& plan) {
  const size_t n = plan.in.size(), ns = (size_t)plan.nseq;
  std::vector<DecFile>& fd = plan.files;
  fd.assign(n, DecFile{});
  Carver c;
  c.next((int64_t)sizeof(DecFile) * (int64_t)n);
  plan.scan_off = c.next((int64_t)sizeof(ProgScan) * (int64_t)plan.scans.size());
  plan.item_off = c.next((int64_t)sizeof(int2) * (int64_t)plan.items.size());
  for (size_t i = 0; i < ns; ++i) {
    fd[i].tabs = c.next((int64_t)sizeof(HuffTab) * 2 * std::max(3, plan.in[i].P.info.components));
    fd[i].raw = c.next(plan.in[i].L.raw_len + 16);
  }
  size_t si = 0;
  for (size_t i = ns; i < n; ++i)
    for (const PScan& S : plan.in[i].G.scans) {
      ProgScan& D = plan.scans[si++];
      D.tabs = c.next((int64_t)sizeof(HuffTab) * S.ncomp);
      D.ist = c.next((int64_t)(D.intervals + 1) * 4);
      D.clean = c.next(S.end - S.start + kScanPad);
    }
  plan.staging = plan.marks = c.offset;
  for (size_t i = 0; i < ns; ++i) {
    fd[i].term = c.next(256);
    fd[i].ist = c.next((int64_t)(plan.in[i].L.intervals + 1) * 4);
  }
  plan.coef = c.offset;
  plan.marks_bytes = plan.coef - plan.marks;
  for (size_t i = 0; i < n; ++i) fd[i].coef = c.next((int64_t)plan.in[i].L.blocks * 128);
  plan.coef_bytes = c.offset - plan.coef;
  for (size_t i = 0; i < n; ++i) {
    const Layout& L = plan.in[i].L;
    if (i < ns) {
      fd[i].sums = c.next((int64_t)(L.chunks + 1) * 8);
      fd[i].clean = c.next(L.raw_len + 16);
      fd[i].sbase = c.next((int64_t)(L.intervals + 1) * 4);
      fd[i].entry = c.next((int64_t)L.sub_max * 8);
      fd[i].exit_ = c.next((int64_t)L.sub_max * 8);
      fd[i].counts = c.next((int64_t)L.sub_max * 16);
      if (plan.in[i].P.info.components == 4) fd[i].counts3 = c.next((int64_t)L.sub_max * 4);
    }
    for (int k = 0; k < plan.in[i].P.info.components; ++k)
      fd[i].plane[k] = c.next((int64_t)L.pw[k] * L.ph[k]);
  }
  plan.scratch = c.offset;
}

// Parses every file, SOF2 files too with `progressive`, and places every region; a refusal names
// the first file refused.
int make_plan(const std::string& name, int n, const uint8_t* const* files, const int64_t* lengths,
              const Mode& mode, Plan& plan) {
  if (!files || !lengths) return fail(SQDET_ERR_INVALID_ARG, name + ": null argument");
  if (n < 1 || n > kMaxFiles)
    return fail(SQDET_ERR_INVALID_ARG, name + ": n must be in [1, " + std::to_string(kMaxFiles) + "]");
  plan.in.resize((size_t)n);
  plan.reduce = mode.reduce;
  for (int i = 0; i < n; ++i) {
    if (!files[i]) return fail(SQDET_ERR_INVALID_ARG, name + ": file " + std::to_string(i) + " is null");
    if (lengths[i] < 4 || lengths[i] > kMaxFileBytes)
      return fail(SQDET_ERR_INVALID_ARG, name + ": file " + std::to_string(i) + ": length must be in [4, 2^28]");
    Input& in = plan.in[(size_t)i];
    const int reason = parse_file(files[i], lengths[i], mode, in.P, in.G);
    if (reason)
      return fail(SQDET_ERR_UNSUPPORTED, name + ": file " + std::to_string(i) + " is not supported: " +
                                             kReasons[reason]);
    in.L = layout(in.P, lengths[i], g_sub_bits);
    in.index = i;
    plan.general = plan.general || general_layout(in.P, in.L);
  }
  const auto prog = std::stable_partition(plan.in.begin(), plan.in.end(),
                                          [](const Input& in) { return !in.P.progressive; });
  plan.nseq = (int)(prog - plan.in.begin());
  // work items: first scans, DC refinements, then AC refinements by their depth in their
  // component's chain
  std::vector<std::vector<int2>> depth_items;
  std::vector<int2> dcref;
  for (size_t i = (size_t)plan.nseq; i < plan.in.size(); ++i) {
    int chain[kMaxComps] = {0, 0, 0, 0};
    for (const PScan& S : plan.in[i].G.scans) {
      ProgScan D{};
      D.file = (int)i;
      scan_geometry(plan.in[i].P, plan.in[i].L, S, D);
      const int si = (int)plan.scans.size();
      plan.scans.push_back(D);
      if (S.ah == 0) {
        for (int r = 0; r < D.intervals; ++r) plan.items.push_back(make_int2(si, r));
      } else if (S.ss == 0) {
        dcref.push_back(make_int2(si, 0));
      } else {
        const int d = chain[S.comp[0]]++;
        if ((int)depth_items.size() <= d) depth_items.resize((size_t)d + 1);
        for (int r = 0; r < D.intervals; ++r) depth_items[(size_t)d].push_back(make_int2(si, r));
      }
    }
  }
  plan.first = (int)plan.items.size();
  plan.items.insert(plan.items.end(), dcref.begin(), dcref.end());
  plan.dc_refine = (int)dcref.size();
  for (const auto& v : depth_items) {
    plan.items.insert(plan.items.end(), v.begin(), v.end());
    plan.depth.push_back((int)v.size());
  }
  place(plan);
  return SQDET_OK;
}

// Fills the staging (descriptors, tables, raw bytes, scans, work items) for outputs out/pitch.
void fill_staging(const Plan& plan, const uint8_t* const* files, uint8_t* const* out,
                  const int64_t* pitch, uint8_t* stage) {
  DecFile* fd = reinterpret_cast<DecFile*>(stage);
  ProgScan* sc = reinterpret_cast<ProgScan*>(stage + plan.scan_off);
  size_t si = 0;
  for (size_t j = 0; j < plan.in.size(); ++j) {
    const Input& in = plan.in[j];
    const Parsed& P = in.P;
    const uint8_t* file = files[in.index];
    DecFile f = plan.files[j];
    describe(P, in.L, f);
    f.index = in.index;
    f.out = out[in.index];
    f.pitch = pitch[in.index];
    if (!P.progressive) {
      HuffTab* tabs = reinterpret_cast<HuffTab*>(stage + f.tabs);
      for (int c = 0; c < P.info.components; ++c) {
        build_tab(P.dc_bits[P.comp[c].td], P.dc_vals[P.comp[c].td], tabs[2 * c]);
        build_tab(P.ac_bits[P.comp[c].ta], P.ac_vals[P.comp[c].ta], tabs[2 * c + 1]);
      }
      memcpy(stage + f.raw, file + P.info.scan_offset, (size_t)in.L.raw_len);
      memset(stage + f.raw + in.L.raw_len, 0, 16);
    }
    for (int c = 0; P.progressive && c < P.info.components; ++c)   // latched at the first scans
      for (int q = 0; q < 64; ++q) f.q[c][q] = in.G.latched[c] ? (int16_t)in.G.q[c][q] : 0;
    fd[j] = f;
    for (const PScan& S : in.G.scans) {
      ProgScan D = plan.scans[si];
      HuffTab* tabs = reinterpret_cast<HuffTab*>(stage + D.tabs);
      const bool coded = S.ss != 0 || S.ah == 0;
      for (int t = 0; coded && t < (S.ss ? 1 : S.ncomp); ++t) build_tab(S.bits[t], S.vals[t], tabs[t]);
      uint8_t* clean = stage + D.clean;
      const bool ok = destuff_scan(file, S.start, S.end, D.intervals, clean,
                                   reinterpret_cast<int32_t*>(stage + D.ist));
      D.bad = D.bad || !ok;
      const int32_t len = reinterpret_cast<int32_t*>(stage + D.ist)[D.intervals];
      memset(clean + len, 0, (size_t)(S.end - S.start - len + kScanPad));
      sc[si++] = D;
    }
  }
  std::copy(plan.items.begin(), plan.items.end(), reinterpret_cast<int2*>(stage + plan.item_off));
}

// The call's launches: the sequential stages over the sequential files, the progressive stages
// over the progressive files' scans, then the IDCT and colour over every file.
int launch_decode(const Plan& plan, uint8_t* stage, uint8_t* scratch, int32_t* status,
                  cudaStream_t stream) {
  const int n = (int)plan.in.size(), ns = plan.nseq;
  int max_chunks = 0, max_tiles = 0, max_blocks = 0;
  int64_t max_pix = 0;
  for (int i = 0; i < n; ++i) {
    const Layout& L = plan.in[(size_t)i].L;
    const sqdet_jpeg_info& I = plan.in[(size_t)i].P.info;
    if (i < ns) {
      max_chunks = std::max(max_chunks, L.chunks);
      max_tiles = std::max(max_tiles, (L.sub_max + kTile - 1) / kTile);
    }
    max_blocks = std::max(max_blocks, L.blocks);
    max_pix = std::max(max_pix, (int64_t)I.height * I.width);
  }
  SQ_CUDA(cudaMemcpyAsync(scratch, stage, (size_t)plan.staging, cudaMemcpyHostToDevice, stream));
  SQ_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * (size_t)n, stream));
  if (ns) SQ_CUDA(cudaMemsetAsync(scratch + plan.marks, 0xFF, (size_t)plan.marks_bytes, stream));
  SQ_CUDA(cudaMemsetAsync(scratch + plan.coef, 0, (size_t)plan.coef_bytes, stream));
  const DecParams p{reinterpret_cast<DecFile*>(scratch), scratch, status};
  if (ns) {
    const unsigned un = (unsigned)ns;
    destuff_count_kernel<<<dim3((unsigned)max_chunks, un), kChunkThreads, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg destuff_count_kernel");
    scan_chunks_kernel<<<un, kScanThreads, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg scan_chunks_kernel");
    destuff_compact_kernel<<<dim3((unsigned)max_chunks, un), kChunkThreads, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg destuff_compact_kernel");
    intervals_kernel<<<un, kScanThreads, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg intervals_kernel");
    sync_tiles_kernel<<<dim3((unsigned)max_tiles, un), kTile, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg sync_tiles_kernel");
    sync_chain_kernel<<<un, kTile, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg sync_chain_kernel");
    scan_counts_kernel<<<un, kScanThreads, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg scan_counts_kernel");
    decode_write_kernel<<<dim3((unsigned)max_tiles, un), kTile, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg decode_write_kernel");
  }
  const ProgParams pp{p.f, reinterpret_cast<const ProgScan*>(scratch + plan.scan_off),
                      reinterpret_cast<const int2*>(scratch + plan.item_off), plan.first, scratch, status};
  if (plan.first) {
    prog_seq_kernel<<<(unsigned)plan.first, kProgThreads, 0, stream>>>(pp);
    SQ_CHECK_LAUNCH("jpeg prog_seq_kernel (first scans)");
  }
  int at = plan.first;
  if (plan.dc_refine) {
    int dc_blocks = 0;
    for (int k = 0; k < plan.dc_refine; ++k) {
      const ProgScan& S = plan.scans[(size_t)plan.items[(size_t)(at + k)].x];
      dc_blocks = std::max(dc_blocks, S.units * S.nb);
    }
    ProgParams q = pp;
    q.items += at;
    q.nitems = plan.dc_refine;
    prog_dc_refine_kernel<<<dim3((unsigned)((dc_blocks + kPixThreads - 1) / kPixThreads), (unsigned)plan.dc_refine),
                            kPixThreads, 0, stream>>>(q);
    SQ_CHECK_LAUNCH("jpeg prog_dc_refine_kernel");
    at += plan.dc_refine;
  }
  for (int d : plan.depth) {
    ProgParams q = pp;
    q.items += at;
    q.nitems = d;
    prog_seq_kernel<<<(unsigned)d, kProgThreads, 0, stream>>>(q);
    SQ_CHECK_LAUNCH("jpeg prog_seq_kernel (AC refinements)");
    at += d;
  }
  const dim3 idct_grid((unsigned)((max_blocks + kPixThreads - 1) / kPixThreads), (unsigned)n);
  if (plan.reduce > 1) idct_kernel<true><<<idct_grid, kPixThreads, 0, stream>>>(p);
  else idct_kernel<false><<<idct_grid, kPixThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg idct_kernel");
  const dim3 pix_grid((unsigned)((max_pix + kPixThreads - 1) / kPixThreads), (unsigned)n);
  color_kernel<<<pix_grid, kPixThreads, 0, stream>>>(p);
  SQ_CHECK_LAUNCH("jpeg color_kernel");
  if (plan.general) {
    color_any_kernel<<<pix_grid, kPixThreads, 0, stream>>>(p);
    SQ_CHECK_LAUNCH("jpeg color_any_kernel");
  }
  return SQDET_OK;
}

// ---- entry points: the plain ones, their _progressive siblings and the _params ones -------------------
std::string entry_name(const char* plain, const Mode& mode) { return std::string(plain) + mode.suffix; }

int parse_entry(const uint8_t* file, int64_t len, sqdet_jpeg_info* out, const Mode& mode) {
  const std::string name = entry_name("sqdet_jpeg_parse", mode);
  if (!file || !out || len < 0) return fail(SQDET_ERR_INVALID_ARG, name + ": bad argument");
  Parsed P;
  Prog G;
  const int reason = parse_file(file, len, mode, P, G);
  P.info.reason = reason;
  if (reason) P.info.supported = 0;
  *out = P.info;
  if (reason) return fail(SQDET_ERR_UNSUPPORTED, name + ": not supported: " + kReasons[reason]);
  return SQDET_OK;
}

int64_t staging_bytes_entry(int n, const uint8_t* const* files, const int64_t* lengths, const Mode& mode) {
  Plan plan;
  if (make_plan(entry_name("sqdet_jpeg_decode_staging_bytes", mode), n, files, lengths, mode, plan))
    return -1;
  return plan.staging;
}

int64_t scratch_bytes_entry(int n, const uint8_t* const* files, const int64_t* lengths, const Mode& mode) {
  Plan plan;
  if (make_plan(entry_name("sqdet_jpeg_decode_scratch_bytes", mode), n, files, lengths, mode, plan))
    return -1;
  return plan.scratch;
}

int decode_entry(int n, const uint8_t* const* files_host, const int64_t* lengths, uint8_t* const* out_planes,
                 const int64_t* out_pitches, void* staging_pinned, int64_t staging_bytes, void* scratch_dev,
                 int64_t scratch_bytes, int32_t* status_dev, void* stream, const Mode& mode) {
  const std::string name = entry_name("sqdet_decode_jpeg", mode);
  if (!out_planes || !out_pitches || !staging_pinned || !scratch_dev || !status_dev)
    return fail(SQDET_ERR_INVALID_ARG, name + ": null argument");
  Plan plan;
  int rc = make_plan(name, n, files_host, lengths, mode, plan);
  if (rc) return rc;
  std::vector<const sqdet_jpeg_info*> info((size_t)n);
  for (const Input& in : plan.in) info[(size_t)in.index] = &in.P.info;
  rc = check_decode_args(name, n, info.data(), out_planes, out_pitches, staging_pinned, staging_bytes,
                         plan.staging, scratch_dev, scratch_bytes, plan.scratch, status_dev,
                         entry_name("sqdet_jpeg_decode_staging_bytes", mode),
                         entry_name("sqdet_jpeg_decode_scratch_bytes", mode));
  if (rc) return rc;
  fill_staging(plan, files_host, out_planes, out_pitches, static_cast<uint8_t*>(staging_pinned));
  DeviceGuard guard(pointer_device(out_planes[0]));
  if (!guard.ok) return fail(SQDET_ERR_CUDA, "cannot select output 0's device");
  return launch_decode(plan, static_cast<uint8_t*>(staging_pinned), static_cast<uint8_t*>(scratch_dev),
                       status_dev, (cudaStream_t)stream);
}

constexpr Mode kPlain{false, 1, false, ""}, kProgressive{true, 1, false, "_progressive"};

// A sqdet_jpeg_decode_options as a Mode, its functions named with `suffix` in messages; false
// (with the error set) when it is not one.
bool options_mode(const char* plain, const char* suffix, const sqdet_jpeg_decode_options* o, Mode& mode) {
  const std::string name = std::string(plain) + suffix;
  if (!o) return fail(SQDET_ERR_INVALID_ARG, name + ": options is null"), false;
  const int s = o->scale_denom;
  if (o->progressive != 0 && o->progressive != 1)
    return fail(SQDET_ERR_INVALID_ARG, name + ": progressive must be 0 or 1"), false;
  if (s != 1 && s != 2 && s != 4 && s != 8)
    return fail(SQDET_ERR_INVALID_ARG, name + ": scale_denom must be 1, 2, 4 or 8"), false;
  if (o->any_layout != 0 && o->any_layout != 1)
    return fail(SQDET_ERR_INVALID_ARG, name + ": any_layout must be 0 or 1"), false;
  for (const int32_t r : o->reserved)
    if (r) return fail(SQDET_ERR_INVALID_ARG, name + ": reserved must be 0"), false;
  mode = Mode{o->progressive == 1, s, o->any_layout == 1, suffix};
  return true;
}

// A sqdet_jpeg_decode_params as a Mode: the options {progressive, scale_denom, any_layout = 0}.
bool params_mode(const char* plain, const sqdet_jpeg_decode_params* params, Mode& mode) {
  if (!params) return fail(SQDET_ERR_INVALID_ARG, std::string(plain) + "_params: params is null"), false;
  sqdet_jpeg_decode_options o{};
  o.progressive = params->progressive;
  o.scale_denom = params->scale_denom;
  o.reserved[0] = params->reserved[0] | params->reserved[1];
  return options_mode(plain, "_params", &o, mode);
}
}  // namespace
}  // namespace sqdet

using namespace sqdet;

int sqdet_jpeg_parse(const uint8_t* file, int64_t len, sqdet_jpeg_info* out) {
  return parse_entry(file, len, out, kPlain);
}

int64_t sqdet_jpeg_decode_staging_bytes(int n, const uint8_t* const* files_host, const int64_t* lengths) {
  return staging_bytes_entry(n, files_host, lengths, kPlain);
}

int64_t sqdet_jpeg_decode_scratch_bytes(int n, const uint8_t* const* files_host, const int64_t* lengths) {
  return scratch_bytes_entry(n, files_host, lengths, kPlain);
}

int sqdet_jpeg_decode_set_subsequence_bits(int bits) {
  if (bits == 0) bits = kDefaultSubBits;
  if (bits < 32 || bits > 8192 || bits % 32)
    return fail(SQDET_ERR_INVALID_ARG, "sqdet_jpeg_decode_set_subsequence_bits: bits must be a multiple of 32 in [32, 8192]");
  g_sub_bits = bits;
  return SQDET_OK;
}

int sqdet_decode_jpeg(int n, const uint8_t* const* files_host, const int64_t* lengths,
                      uint8_t* const* out_planes, const int64_t* out_pitches, void* staging_pinned,
                      int64_t staging_bytes, void* scratch_dev, int64_t scratch_bytes,
                      int32_t* status_dev, void* stream) {
  return decode_entry(n, files_host, lengths, out_planes, out_pitches, staging_pinned, staging_bytes,
                      scratch_dev, scratch_bytes, status_dev, stream, kPlain);
}

int sqdet_jpeg_parse_progressive(const uint8_t* file, int64_t len, sqdet_jpeg_info* out) {
  return parse_entry(file, len, out, kProgressive);
}

int64_t sqdet_jpeg_decode_staging_bytes_progressive(int n, const uint8_t* const* files_host,
                                                    const int64_t* lengths) {
  return staging_bytes_entry(n, files_host, lengths, kProgressive);
}

int64_t sqdet_jpeg_decode_scratch_bytes_progressive(int n, const uint8_t* const* files_host,
                                                    const int64_t* lengths) {
  return scratch_bytes_entry(n, files_host, lengths, kProgressive);
}

int sqdet_decode_jpeg_progressive(int n, const uint8_t* const* files_host, const int64_t* lengths,
                                  uint8_t* const* out_planes, const int64_t* out_pitches,
                                  void* staging_pinned, int64_t staging_bytes, void* scratch_dev,
                                  int64_t scratch_bytes, int32_t* status_dev, void* stream) {
  return decode_entry(n, files_host, lengths, out_planes, out_pitches, staging_pinned, staging_bytes,
                      scratch_dev, scratch_bytes, status_dev, stream, kProgressive);
}

int sqdet_jpeg_parse_params(const uint8_t* file, int64_t len, const sqdet_jpeg_decode_params* params,
                            sqdet_jpeg_info* out) {
  Mode mode;
  if (!params_mode("sqdet_jpeg_parse", params, mode)) return SQDET_ERR_INVALID_ARG;
  return parse_entry(file, len, out, mode);
}

int64_t sqdet_jpeg_decode_staging_bytes_params(int n, const uint8_t* const* files_host,
                                               const int64_t* lengths,
                                               const sqdet_jpeg_decode_params* params) {
  Mode mode;
  if (!params_mode("sqdet_jpeg_decode_staging_bytes", params, mode)) return -1;
  return staging_bytes_entry(n, files_host, lengths, mode);
}

int64_t sqdet_jpeg_decode_scratch_bytes_params(int n, const uint8_t* const* files_host,
                                               const int64_t* lengths,
                                               const sqdet_jpeg_decode_params* params) {
  Mode mode;
  if (!params_mode("sqdet_jpeg_decode_scratch_bytes", params, mode)) return -1;
  return scratch_bytes_entry(n, files_host, lengths, mode);
}

int sqdet_decode_jpeg_params(int n, const uint8_t* const* files_host, const int64_t* lengths,
                             const sqdet_jpeg_decode_params* params, uint8_t* const* out_planes,
                             const int64_t* out_pitches, void* staging_pinned, int64_t staging_bytes,
                             void* scratch_dev, int64_t scratch_bytes, int32_t* status_dev,
                             void* stream) {
  Mode mode;
  if (!params_mode("sqdet_decode_jpeg", params, mode)) return SQDET_ERR_INVALID_ARG;
  return decode_entry(n, files_host, lengths, out_planes, out_pitches, staging_pinned, staging_bytes,
                      scratch_dev, scratch_bytes, status_dev, stream, mode);
}

int sqdet_jpeg_parse_options(const uint8_t* file, int64_t len, const sqdet_jpeg_decode_options* options,
                             sqdet_jpeg_info* out) {
  Mode mode;
  if (!options_mode("sqdet_jpeg_parse", "_options", options, mode)) return SQDET_ERR_INVALID_ARG;
  return parse_entry(file, len, out, mode);
}

int64_t sqdet_jpeg_decode_staging_bytes_options(int n, const uint8_t* const* files_host,
                                                const int64_t* lengths,
                                                const sqdet_jpeg_decode_options* options) {
  Mode mode;
  if (!options_mode("sqdet_jpeg_decode_staging_bytes", "_options", options, mode)) return -1;
  return staging_bytes_entry(n, files_host, lengths, mode);
}

int64_t sqdet_jpeg_decode_scratch_bytes_options(int n, const uint8_t* const* files_host,
                                                const int64_t* lengths,
                                                const sqdet_jpeg_decode_options* options) {
  Mode mode;
  if (!options_mode("sqdet_jpeg_decode_scratch_bytes", "_options", options, mode)) return -1;
  return scratch_bytes_entry(n, files_host, lengths, mode);
}

int sqdet_decode_jpeg_options(int n, const uint8_t* const* files_host, const int64_t* lengths,
                              const sqdet_jpeg_decode_options* options, uint8_t* const* out_planes,
                              const int64_t* out_pitches, void* staging_pinned, int64_t staging_bytes,
                              void* scratch_dev, int64_t scratch_bytes, int32_t* status_dev,
                              void* stream) {
  Mode mode;
  if (!options_mode("sqdet_decode_jpeg", "_options", options, mode)) return SQDET_ERR_INVALID_ARG;
  return decode_entry(n, files_host, lengths, out_planes, out_pitches, staging_pinned, staging_bytes,
                      scratch_dev, scratch_bytes, status_dev, stream, mode);
}
