// Baseline Huffman JPEG -> RGB on the device, byte for byte equal to Pillow's `Image.open(f).convert("RGB")` with its
// libjpeg-turbo backend (the arithmetic is restated in oracle/jpeg_ref.py and pinned against Pillow there).
//
// The host parses each header (markers SOI .. SOS), decides eligibility, derives the Huffman tables exactly as
// libjpeg does and uploads every photo's tables and layout in one copy.  The device then runs, for the whole batch:
//   segment   seg_count / seg_scan / seg_write: one pass over the entropy-coded bytes that removes the 0xFF00
//             stuffing, finds the RSTn markers and checks their order; the restart intervals become independent
//             bitstreams (the whole scan is one interval without restart markers).
//   entropy   Weissenberger & Schmidt's self-synchronising decoding (ICPP 2018): every interval is cut into
//             subsequences of `subseq_bits`; a thread decodes one subsequence from a state (bit position, block of
//             the MCU, coefficient index) and records the state it ends in.  huff_sync_kernel starts every
//             subsequence from a guess and repeats passes, each starting subsequence j from j-1's last end state,
//             until no start state changes.  The first subsequence of an interval starts from its exact state, so
//             the fixed point is the sequential decode however many passes it takes.  A scan of the per-subsequence
//             block counts and DC-difference sums (reset per interval) then places every block and gives its DC
//             prediction, and huff_write_kernel decodes once more, writing 16-bit coefficients (libjpeg's JCOEF).
//   idct      jpeg_idct_islow with libjpeg's constants, passes and descaling, 64-bit where libjpeg's JLONG is.
//   colour    fancy h2v1 / h2v2 upsampling (box for a component at most 2 samples wide), YCbCr -> RGB with libjpeg's
//             16-bit fixed-point tables, gray replicated; HWC uint8 at the caller's pitch.
// Any anomaly of the entropy data, or an IDCT block where libjpeg-turbo's SIMD and C IDCTs disagree, sets a bit of
// the photo's status instead of guessing at libjpeg's recovery; the caller decodes such a photo on the host.
//
// Memory safety for any content of the compressed bytes: every address below comes from the validated header or from
// a counter checked against it.  Segment kernels read only [0, ecs_len) of their photo's bytes and write a kept byte
// at (kept bytes before it) < ecs_len of the photo's destuffed buffer; a marker's interval slot is written only for
// marker index < intervals - 1.  The bit reader clamps its word index into the photo's destuffed buffer.  The
// entropy kernels write a coefficient only for block index < the interval's block count (so the MCU, and the block's
// plane row and column, are inside the header's MCU grid) and coefficient index <= 63; Huffman value lookups clamp to
// the 256-entry table.  IDCT and colour kernels index planes and outputs from header sizes only.
#include "common.cuh"

#include <cooperative_groups.h>

#include <algorithm>
#include <cstring>
#include <vector>

using namespace mhmr;
namespace cg = cooperative_groups;

namespace {

// status bits (oracle/jpeg_ref.py has the same values)
constexpr int kBadCode = 1, kBadSize = 2, kBadRun = 4, kShortData = 8, kBadRst = 16, kIdctRange = 32;
constexpr int kChunk = 4096;         // segment kernels: bytes per CTA (256 threads x 16)
constexpr int kSlack = 32;           // zero bytes after each destuffed stream (the bit reader's look-ahead)
constexpr int kDefaultSubseqBits = 1024;
constexpr int kMaxBytes = 1 << 28;   // per file: bit positions stay int32

constexpr uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t c_zigzag[64];

struct JHuff {             // libjpeg's derived decoding table plus a 9-bit first-level lookup
  uint16_t lut[512];       // (length << 8 | value) of the code that prefixes a 9-bit window, 0 if longer than 9 bits
  int32_t maxcode[18];     // largest code of each length, -1 if none
  int32_t valoff[17];
  uint8_t vals[256];
};

struct JTables {
  JHuff dc[3], ac[3];
  int32_t qt[3][64];       // natural order
};

struct JPhoto {
  const uint8_t* ecs;      // entropy-coded segment (device), ecs_len bytes
  int ecs_len;
  int chunk0, nchunk;      // segment chunks
  int iv0, niv;            // restart intervals
  uint8_t* dst;            // destuffed stream, ecs_len + kSlack bytes
  int W, H, ncomp, hm, vm;
  int hs[3], vs[3];
  int bpm, mcux, mcuy, per;          // blocks per MCU, MCU grid, MCUs per interval
  int blk_comp[6], blk_x[6], blk_y[6];
  int bw[3], bh[3];                  // coefficient / sample planes in blocks
  int16_t* coef[3];
  uint8_t* plane[3];
  uint8_t* out;
  int64_t pitch;
};

struct JIv {
  int photo, first_mcu, mcus;
  int start, end;          // destuffed byte range
  int sub0, nsub;
};

struct Ctx {
  const JPhoto* ph;
  const JTables* tab;
  JIv* iv;
  int niv;
  int subseq_bits;
  int max_sub;             // host bound on the subsequence count
  int* nsub;               // device: actual count
  int* sub_iv;             // [max_sub]
  int2* start;             // [max_sub]: (bit position, block-of-MCU * 64 + coefficient index)
  int2* endst;             // [2][max_sub]
  int* cnt;                // [max_sub] DC symbols (blocks started)
  uint32_t* dcs;           // [max_sub][3] DC-difference sums
  int* cntx;               // exclusive scans of the above
  uint32_t* dcx;
  uint32_t* part;          // [4][nparts] per-tile totals, then their exclusive scans
  int nparts;              // 1024-subsequence tiles of max_sub
  int* done;               // [niv] the interval's last block completed inside its data
  int* flags;              // [3] sync-pass change flags
  int* passes;             // device out (nullable)
  int32_t* status;
};

// ---- small block-wide scans -------------------------------------------------------------------------------------
template <int NT>
__device__ int block_excl_scan(int v, int* total) {
  __shared__ int warp_sums[NT / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[w] = x;
  __syncthreads();
  if (w == 0) {
    int s = lane < NT / 32 ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < NT / 32) warp_sums[lane] = s;
  }
  __syncthreads();
  const int r = x - v + (w > 0 ? warp_sums[w - 1] : 0);
  *total = warp_sums[NT / 32 - 1];
  __syncthreads();
  return r;
}

// ---- segment: destuffing and restart markers ----------------------------------------------------------------------
// Byte i of a segment is kept unless it follows a 0xFF (the 0x00 of a stuffed 0xFF, or a marker's code byte) or is
// a 0xFF that starts a marker (followed by anything but 0x00).  The host checked that a 0xFF inside the segment is
// followed by 0x00 or RST0..7; the kernels stay inside [0, ecs_len) whatever the bytes are.
__device__ __forceinline__ void classify(const uint8_t* b, int L, int i, bool* keep, bool* marker) {
  const uint8_t c = __ldg(b + i);
  const bool after_ff = i > 0 && __ldg(b + i - 1) == 0xFF;
  const bool ff_marker = c == 0xFF && (i + 1 >= L || __ldg(b + i + 1) != 0x00);
  *keep = !after_ff && !ff_marker;
  *marker = !after_ff && ff_marker;
}

struct Chunk {
  int photo, off;
};

__global__ void __launch_bounds__(256) seg_count_kernel(const JPhoto* __restrict__ ph, const Chunk* __restrict__ ch,
                                                        int* kept, int* marks) {
  const Chunk c = ch[blockIdx.x];
  const JPhoto& p = ph[c.photo];
  const int i0 = c.off + threadIdx.x * (kChunk / 256), i1 = min(i0 + kChunk / 256, p.ecs_len);
  int k = 0, m = 0;
  for (int i = i0; i < i1; ++i) {
    bool keep, marker;
    classify(p.ecs, p.ecs_len, i, &keep, &marker);
    k += keep;
    m += marker;
  }
  int tk, tm;
  block_excl_scan<256>(k, &tk);
  block_excl_scan<256>(m, &tm);
  if (threadIdx.x == 0) {
    kept[blockIdx.x] = tk;
    marks[blockIdx.x] = tm;
  }
}

// One CTA per photo: chunk offsets (exclusive scans of the counts, in place), the destuffed length, and the marker
// count check (exactly intervals - 1 markers).
__global__ void __launch_bounds__(1024) seg_scan_kernel(const JPhoto* __restrict__ ph, JIv* iv, int* kept, int* marks,
                                                        int32_t* status) {
  const JPhoto& p = ph[blockIdx.x];
  int kbase = 0, mbase = 0;
  for (int t0 = 0; t0 < p.nchunk; t0 += 1024) {
    const int t = t0 + threadIdx.x;
    const int k = t < p.nchunk ? kept[p.chunk0 + t] : 0, m = t < p.nchunk ? marks[p.chunk0 + t] : 0;
    int tk, tm;
    const int ek = block_excl_scan<1024>(k, &tk), em = block_excl_scan<1024>(m, &tm);
    if (t < p.nchunk) {
      kept[p.chunk0 + t] = kbase + ek;
      marks[p.chunk0 + t] = mbase + em;
    }
    kbase += tk;
    mbase += tm;
  }
  if (threadIdx.x == 0) {
    if (mbase != p.niv - 1) atomicOr(status + blockIdx.x, kBadRst);
    iv[p.iv0].start = 0;
    iv[p.iv0 + p.niv - 1].end = kbase;
  }
}

__global__ void __launch_bounds__(256) seg_write_kernel(const JPhoto* __restrict__ ph, const Chunk* __restrict__ ch,
                                                        const int* __restrict__ kept, const int* __restrict__ marks,
                                                        JIv* iv, int32_t* status) {
  const Chunk c = ch[blockIdx.x];
  const JPhoto& p = ph[c.photo];
  const int i0 = c.off + threadIdx.x * (kChunk / 256), i1 = min(i0 + kChunk / 256, p.ecs_len);
  int k = 0, m = 0;
  for (int i = i0; i < i1; ++i) {
    bool keep, marker;
    classify(p.ecs, p.ecs_len, i, &keep, &marker);
    k += keep;
    m += marker;
  }
  int tk, tm;
  int kpos = kept[blockIdx.x] + block_excl_scan<256>(k, &tk);
  int mpos = marks[blockIdx.x] + block_excl_scan<256>(m, &tm);
  for (int i = i0; i < i1; ++i) {
    bool keep, marker;
    classify(p.ecs, p.ecs_len, i, &keep, &marker);
    if (keep) {
      p.dst[kpos++] = __ldg(p.ecs + i);   // kpos < number of kept bytes <= ecs_len
    } else if (marker) {
      const int code = i + 1 < p.ecs_len ? __ldg(p.ecs + i + 1) : -1;
      if (mpos < p.niv - 1) {
        iv[p.iv0 + mpos].end = kpos;
        iv[p.iv0 + mpos + 1].start = kpos;
        if (code != 0xD0 + (mpos & 7)) atomicOr(status + c.photo, kBadRst);
      }
      ++mpos;
    }
  }
}

// Subsequences per interval (at least one) and their global numbering; sub_map_kernel then fills the subsequence ->
// interval map in parallel.
__global__ void __launch_bounds__(1024) plan_kernel(Ctx ctx) {
  int base = 0;
  for (int t0 = 0; t0 < ctx.niv; t0 += 1024) {
    const int t = t0 + threadIdx.x;
    int n = 0;
    if (t < ctx.niv) {
      const JIv& v = ctx.iv[t];
      const int64_t bits = 8ll * max(v.end - v.start, 0);
      n = static_cast<int>((bits + ctx.subseq_bits - 1) / ctx.subseq_bits);
      n = n > 0 ? n : 1;
    }
    int tot;
    const int e = block_excl_scan<1024>(n, &tot);
    if (t < ctx.niv) {
      ctx.iv[t].sub0 = base + e;
      ctx.iv[t].nsub = n;
    }
    base += tot;
  }
  if (threadIdx.x == 0) *ctx.nsub = min(base, ctx.max_sub);   // base <= max_sub by the host's bound
}

// One thread per subsequence: the interval whose first subsequence is the last one at or before j (the sub0 are
// strictly increasing, every interval having at least one subsequence).
__global__ void __launch_bounds__(256) sub_map_kernel(Ctx ctx) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= *ctx.nsub) return;
  int lo = 0, hi = ctx.niv - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (ctx.iv[mid].sub0 <= j) lo = mid; else hi = mid - 1;
  }
  ctx.sub_iv[j] = lo;
}

// ---- entropy decoding -------------------------------------------------------------------------------------------
// 32 bits of the destuffed stream from bit p, read as two big-endian words.  The word index is clamped into the
// photo's buffer (ecs_len + kSlack bytes), so no read leaves it whatever p is.
__device__ __forceinline__ uint32_t peek32(const uint8_t* buf, int nwords, int p) {
  const int w = min(p >> 5, nwords - 2);
  const uint32_t* wp = reinterpret_cast<const uint32_t*>(buf);
  const uint64_t hi = __byte_perm(__ldg(wp + w), 0, 0x0123), lo = __byte_perm(__ldg(wp + w + 1), 0, 0x0123);
  return static_cast<uint32_t>(((hi << 32) | lo) << (p & 31) >> 32);
}

// One Huffman symbol from the window `bits`: its value, and its code length (0 for a code with no table entry).
__device__ __forceinline__ int huff_decode(const JHuff& t, uint32_t bits, int* len) {
  const uint32_t e = t.lut[bits >> 23];
  if (e) {
    *len = e >> 8;
    return e & 255;
  }
  int l = 10;
  int code = static_cast<int>(bits >> 22);
  while (l <= 16 && code > t.maxcode[l]) {
    ++l;
    code = static_cast<int>(bits >> (32 - l));
  }
  if (l > 16) {
    *len = 0;
    return 0;
  }
  *len = l;
  return t.vals[min(max(code + t.valoff[l], 0), 255)];
}

__device__ __forceinline__ int extend(uint32_t v, int s) {
  return s && v < (1u << (s - 1)) ? static_cast<int>(v) - (1 << s) + 1 : static_cast<int>(v);
}

// Decodes subsequence j from state `st` up to the first symbol boundary at or past its end and returns that state.
// Counting (WRITE false): blocks started and DC-difference sums per component.  Writing: coefficients, DC
// predictions, anomalies of real blocks, and the interval's completion.  An anomaly ends the block (after the bits
// of its code), a deterministic rule that keeps the sync passes well defined for any guessed state.
template <bool WRITE>
__device__ int2 decode_subseq(const Ctx& ctx, int j, int2 st, int* n_dc, uint32_t dsum[3]) {
  const JIv& v = ctx.iv[ctx.sub_iv[j]];
  const JPhoto& p = ctx.ph[v.photo];
  const JTables& tab = ctx.tab[v.photo];
  const int nwords = (p.ecs_len + kSlack) >> 2;
  const int ivbit0 = 8 * v.start, ivbit1 = 8 * max(v.end, v.start);
  const int q = j - v.sub0;
  const int64_t rel = static_cast<int64_t>(q + 1) * ctx.subseq_bits;
  const int seq_end = rel < ivbit1 - ivbit0 ? ivbit0 + static_cast<int>(rel) : ivbit1;
  const int needed = v.mcus * p.bpm;
  int pos = st.x, blk = st.y >> 6, k = st.y & 63;
  if (blk >= p.bpm) blk = 0;
  int bidx = 0;
  uint32_t pred[3] = {0, 0, 0};
  if (WRITE) {
    bidx = ctx.cntx[j] - ctx.cntx[v.sub0] - 1;  // the block in progress at the start
    for (int c = 0; c < 3; ++c) pred[c] = ctx.dcx[3 * j + c] - ctx.dcx[3 * v.sub0 + c];
  }
  int ndc = 0;
  while (pos < seq_end) {
    const int comp = p.blk_comp[blk];
    int bad = 0;
    if (k == 0) {
      int len;
      const int s = huff_decode(tab.dc[comp], peek32(p.dst, nwords, pos), &len);
      ++ndc;
      if (WRITE) ++bidx;
      if (len == 0) {
        bad = kBadCode;
        pos += 16;
      } else if (s > 11) {
        bad = kBadSize;
        pos += len;
      } else {
        pos += len;
        const int d = s ? extend(peek32(p.dst, nwords, pos) >> (32 - s), s) : 0;
        pos += s;
        dsum[comp] += static_cast<uint32_t>(d);
        if (WRITE && bidx < needed) {
          pred[comp] += static_cast<uint32_t>(d);
          const int m = v.first_mcu + bidx / p.bpm;
          const int bx = (m % p.mcux) * p.hs[comp] + p.blk_x[blk], by = (m / p.mcux) * p.vs[comp] + p.blk_y[blk];
          p.coef[comp][(static_cast<int64_t>(by) * p.bw[comp] + bx) * 64] = static_cast<int16_t>(pred[comp]);
        }
        k = 1;
      }
    } else {
      int len;
      const int rs = huff_decode(tab.ac[comp], peek32(p.dst, nwords, pos), &len);
      const int r = rs >> 4, s = rs & 15;
      if (len == 0) {
        bad = kBadCode;
        pos += 16;
      } else if (s == 0) {
        pos += len;
        if (r != 15) {
          k = 64;
        } else if (k + 15 > 63) {
          bad = kBadRun;
        } else {
          k += 16;
        }
      } else if (s > 10) {
        bad = kBadSize;
        pos += len;
      } else if (k + r > 63) {
        bad = kBadRun;
        pos += len;
      } else {
        pos += len;
        k += r;
        const int val = extend(peek32(p.dst, nwords, pos) >> (32 - s), s);
        pos += s;
        if (WRITE && bidx >= 0 && bidx < needed) {
          const int m = v.first_mcu + bidx / p.bpm;
          const int bx = (m % p.mcux) * p.hs[comp] + p.blk_x[blk], by = (m / p.mcux) * p.vs[comp] + p.blk_y[blk];
          p.coef[comp][(static_cast<int64_t>(by) * p.bw[comp] + bx) * 64 + c_zigzag[k]] = static_cast<int16_t>(val);
        }
        ++k;
      }
    }
    if (bad) {
      if (WRITE && bidx >= 0 && bidx < needed) atomicOr(ctx.status + v.photo, bad);
      k = 64;
    }
    if (k >= 64) {
      if (WRITE && bidx == needed - 1 && !bad && pos <= ivbit1) ctx.done[ctx.sub_iv[j]] = 1;
      k = 0;
      blk = blk + 1 == p.bpm ? 0 : blk + 1;
      if (WRITE && bidx >= needed - 1) break;    // past the interval's blocks: the rest is padding
    }
  }
  *n_dc = ndc;
  return make_int2(pos, blk * 64 + k);
}

__device__ __forceinline__ int2 first_state(const Ctx& ctx, int j, bool* exact) {
  const JIv& v = ctx.iv[ctx.sub_iv[j]];
  *exact = j == v.sub0;
  return make_int2(8 * v.start + (j - v.sub0) * ctx.subseq_bits, 0);
}

// Cooperative: every pass covers all subsequences (grid-stride), then the grid synchronises and stops when no start
// state changed.  End states are double-buffered by pass parity; three change flags let a pass reset the flag of
// the next one while stragglers still read the current one.
__global__ void __launch_bounds__(256) huff_sync_kernel(Ctx ctx) {
  cg::grid_group g = cg::this_grid();
  const int n = *ctx.nsub;
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    bool exact;
    const int2 s = first_state(ctx, j, &exact);
    uint32_t ds[3] = {0, 0, 0};
    int c;
    ctx.start[j] = s;
    ctx.endst[j] = decode_subseq<false>(ctx, j, s, &c, ds);
    ctx.cnt[j] = c;
    for (int q = 0; q < 3; ++q) ctx.dcs[3 * j + q] = ds[q];
  }
  g.sync();
  int pass = 1;
  for (;; ++pass) {
    if (g.thread_rank() == 0) ctx.flags[(pass + 1) % 3] = 0;
    const int2* prev = ctx.endst + static_cast<int64_t>((pass - 1) & 1) * ctx.max_sub;
    int2* cur = ctx.endst + static_cast<int64_t>(pass & 1) * ctx.max_sub;
    bool changed = false;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
      const bool first = j == ctx.iv[ctx.sub_iv[j]].sub0;
      const int2 s = first ? ctx.start[j] : prev[j - 1];
      const int2 old = ctx.start[j];
      if (s.x == old.x && s.y == old.y) {
        cur[j] = prev[j];
        continue;
      }
      changed = true;
      uint32_t ds[3] = {0, 0, 0};
      int c;
      ctx.start[j] = s;
      cur[j] = decode_subseq<false>(ctx, j, s, &c, ds);
      ctx.cnt[j] = c;
      for (int q = 0; q < 3; ++q) ctx.dcs[3 * j + q] = ds[q];
    }
    if (changed) ctx.flags[pass % 3] = 1;
    g.sync();
    if (ctx.flags[pass % 3] == 0) break;
  }
  if (g.thread_rank() == 0 && ctx.passes != nullptr) *ctx.passes = pass;
}

// Exclusive scans over all subsequences of the block counts and the per-component DC sums, in two levels: the totals
// of each 1024-subsequence tile, a scan of those totals (one CTA over max_sub / 1024 values), then each tile's own
// scan.  An interval's offsets are differences against its first subsequence, so the scans need no segments; the DC
// sums wrap around, scanned as int with the same bits as uint32 arithmetic.
__device__ __forceinline__ int sub_value(const Ctx& ctx, int t, int n, int q) {
  if (t >= n) return 0;
  return q == 0 ? ctx.cnt[t] : static_cast<int>(ctx.dcs[3 * t + q - 1]);
}

__global__ void __launch_bounds__(1024) sub_tile_sum_kernel(Ctx ctx) {
  const int n = *ctx.nsub;
  if (blockIdx.x * 1024 >= n) return;   // uniform over the CTA
  const int t = blockIdx.x * 1024 + threadIdx.x;
  for (int q = 0; q < 4; ++q) {
    int tot;
    block_excl_scan<1024>(sub_value(ctx, t, n, q), &tot);
    if (threadIdx.x == 0) ctx.part[q * ctx.nparts + blockIdx.x] = static_cast<uint32_t>(tot);
  }
}

__global__ void __launch_bounds__(1024) sub_tile_scan_kernel(Ctx ctx) {
  const int nt = (*ctx.nsub + 1023) / 1024;
  for (int q = 0; q < 4; ++q) {
    uint32_t base = 0;
    for (int t0 = 0; t0 < nt; t0 += 1024) {
      const int t = t0 + threadIdx.x;
      uint32_t* row = ctx.part + q * ctx.nparts;
      int tot;
      const int e = block_excl_scan<1024>(t < nt ? static_cast<int>(row[t]) : 0, &tot);
      if (t < nt) row[t] = base + static_cast<uint32_t>(e);
      base += static_cast<uint32_t>(tot);
    }
  }
}

__global__ void __launch_bounds__(1024) sub_scan_kernel(Ctx ctx) {
  const int n = *ctx.nsub;
  if (blockIdx.x * 1024 >= n) return;
  const int t = blockIdx.x * 1024 + threadIdx.x;
  for (int q = 0; q < 4; ++q) {
    int tot;
    const uint32_t e = static_cast<uint32_t>(block_excl_scan<1024>(sub_value(ctx, t, n, q), &tot)) +
                       ctx.part[q * ctx.nparts + blockIdx.x];
    if (t < n) {
      if (q == 0) ctx.cntx[t] = static_cast<int>(e);
      else ctx.dcx[3 * t + q - 1] = e;
    }
  }
}

__global__ void __launch_bounds__(256) huff_write_kernel(Ctx ctx) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= *ctx.nsub) return;
  uint32_t ds[3] = {0, 0, 0};
  int c;
  decode_subseq<true>(ctx, j, ctx.start[j], &c, ds);
}

__global__ void check_done_kernel(Ctx ctx) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < ctx.niv && !ctx.done[t]) atomicOr(ctx.status + ctx.iv[t].photo, kShortData);
}

// ---- IDCT -------------------------------------------------------------------------------------------------------
constexpr int kF0298 = 2446, kF0390 = 3196, kF0541 = 4433, kF0765 = 6270, kF0899 = 7373, kF1175 = 9633,
              kF1501 = 12299, kF1847 = 15137, kF1961 = 16069, kF2053 = 16819, kF2562 = 20995, kF3072 = 25172;

// One islow butterfly: x[0..7] in, the 8 undescaled sums out (libjpeg's JLONG arithmetic).
__device__ __forceinline__ void idct_1d(const int64_t x[8], int64_t o[8]) {
  int64_t z2 = x[2], z3 = x[6];
  int64_t z1 = (z2 + z3) * kF0541;
  const int64_t tmp2 = z1 + z3 * -kF1847, tmp3 = z1 + z2 * kF0765;
  const int64_t tmp0 = (x[0] + x[4]) * (1 << 13), tmp1 = (x[0] - x[4]) * (1 << 13);
  const int64_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int64_t a0 = x[7], a1 = x[5], a2 = x[3], a3 = x[1];
  z1 = a0 + a3;
  z2 = a1 + a2;
  z3 = a0 + a2;
  int64_t z4 = a1 + a3;
  const int64_t z5 = (z3 + z4) * kF1175;
  a0 *= kF0298;
  a1 *= kF2053;
  a2 *= kF3072;
  a3 *= kF1501;
  z1 *= -kF0899;
  z2 *= -kF2562;
  z3 = z3 * -kF1961 + z5;
  z4 = z4 * -kF0390 + z5;
  a0 += z1 + z3;
  a1 += z2 + z4;
  a2 += z2 + z3;
  a3 += z1 + z4;
  o[0] = t10 + a3; o[7] = t10 - a3;
  o[1] = t11 + a2; o[6] = t11 - a2;
  o[2] = t12 + a1; o[5] = t12 - a1;
  o[3] = t13 + a0; o[4] = t13 - a0;
}

struct PlaneRef {
  int photo, comp, block0;   // first block of this plane in the launch's numbering
};

// 8 threads per block: column pass then row pass through shared memory.  Flags a block whose dequantised
// coefficients or pass-1 values leave int16 or whose outputs leave [-512, 512): libjpeg-turbo's 16-bit SIMD IDCT
// saturates there while its C IDCT wraps.
__global__ void __launch_bounds__(256) idct_kernel(const JPhoto* __restrict__ ph, const JTables* __restrict__ tab,
                                                   const PlaneRef* __restrict__ planes, int nplanes, int nblocks,
                                                   int32_t* status) {
  __shared__ int32_t ws[32][64];
  const int lb = threadIdx.x >> 3, col = threadIdx.x & 7;
  const int b = blockIdx.x * 32 + lb;
  const bool live = b < nblocks;
  int lo = 0, hi = nplanes - 1;
  while (lo < hi) {   // the plane holding block b
    const int mid = (lo + hi + 1) >> 1;
    if (planes[mid].block0 <= (live ? b : 0)) lo = mid; else hi = mid - 1;
  }
  const PlaneRef pr = planes[lo];
  const JPhoto& p = ph[pr.photo];
  const int c = pr.comp;
  const int local = live ? b - pr.block0 : 0;
  bool bad = false;
  if (live) {
    const int16_t* cf = p.coef[c] + static_cast<int64_t>(local) * 64;
    const int32_t* q = tab[pr.photo].qt[c];
    int64_t x[8], o[8];
    for (int r = 0; r < 8; ++r) {
      x[r] = static_cast<int64_t>(cf[r * 8 + col]) * q[r * 8 + col];
      bad |= x[r] > 32767 || x[r] < -32767;
    }
    idct_1d(x, o);
    for (int r = 0; r < 8; ++r) {
      const int32_t w = static_cast<int32_t>((o[r] + (1 << 10)) >> 11);   // (int)DESCALE(.., CONST_BITS - PASS1_BITS)
      bad |= w > 32767 || w < -32767;
      ws[lb][r * 8 + col] = w;
    }
  }
  __syncthreads();
  if (!live) return;
  int64_t x[8], o[8];
  for (int i = 0; i < 8; ++i) x[i] = ws[lb][col * 8 + i];
  idct_1d(x, o);
  const int bw = p.bw[c];
  const int bx = local % bw, by = local / bw;
  uint8_t* dst = p.plane[c] + (static_cast<int64_t>(by) * 8 + col) * (bw * 8) + bx * 8;
  uint8_t px[8];
  for (int i = 0; i < 8; ++i) {
    const int64_t vv = (o[i] + (1 << 17)) >> 18;   // DESCALE(.., CONST_BITS + PASS1_BITS + 3)
    bad |= vv < -512 || vv > 511;
    const int w = static_cast<int>(((vv + 512) & 1023) - 512);   // the range-limit table's wrap-around
    px[i] = static_cast<uint8_t>(min(max(w + 128, 0), 255));
  }
  *reinterpret_cast<uint2*>(dst) = make_uint2(px[0] | px[1] << 8 | px[2] << 16 | static_cast<uint32_t>(px[3]) << 24,
                                              px[4] | px[5] << 8 | px[6] << 16 | static_cast<uint32_t>(px[7]) << 24);
  if (bad) atomicOr(status + pr.photo, kIdctRange);
}

// ---- upsampling and colour --------------------------------------------------------------------------------------
__device__ __forceinline__ int sample(const JPhoto& p, int c, int x, int y) {
  return p.plane[c][static_cast<int64_t>(y) * (p.bw[c] * 8) + x];
}

// Chroma sample of component c at output pixel (x, y): libjpeg-turbo's fancy h2v1 / h2v2 filters over the
// component's real size dw x dh with replicated edges, or box upsampling for a component at most 2 samples wide.
__device__ __forceinline__ int chroma(const JPhoto& p, int c, int x, int y) {
  const int hf = p.hm / p.hs[c], vf = p.vm / p.vs[c];
  if (hf == 1 && vf == 1) return sample(p, c, x, y);
  const int dw = (p.W * p.hs[c] + p.hm - 1) / p.hm, dh = (p.H * p.vs[c] + p.vm - 1) / p.vm;
  if (dw <= 2) return sample(p, c, x / hf, y / vf);
  const int i = x >> 1;
  const bool odd = x & 1;
  if (vf == 1) {   // h2v1
    const int s = sample(p, c, i, y);
    if (!odd) return i == 0 ? s : (3 * s + sample(p, c, i - 1, y) + 1) >> 2;
    return i == dw - 1 ? s : (3 * s + sample(p, c, i + 1, y) + 2) >> 2;
  }
  const int r = y >> 1, nb = (y & 1) ? min(r + 1, dh - 1) : max(r - 1, 0);   // h2v2
  const int cs = 3 * sample(p, c, i, r) + sample(p, c, i, nb);
  if (!odd) return i == 0 ? (4 * cs + 8) >> 4 : (3 * cs + 3 * sample(p, c, i - 1, r) + sample(p, c, i - 1, nb) + 8) >> 4;
  return i == dw - 1 ? (4 * cs + 7) >> 4 : (3 * cs + 3 * sample(p, c, i + 1, r) + sample(p, c, i + 1, nb) + 7) >> 4;
}

__global__ void __launch_bounds__(256) color_kernel(const JPhoto* __restrict__ ph) {
  const JPhoto& p = ph[blockIdx.z];
  const int x = blockIdx.x * 256 + threadIdx.x;
  if (x >= p.W) return;
  for (int y = blockIdx.y; y < p.H; y += gridDim.y) {
    uint8_t* o = p.out + static_cast<int64_t>(y) * p.pitch + 3 * x;
    const int Y = sample(p, 0, x, y);
    if (p.ncomp == 1) {
      o[0] = o[1] = o[2] = static_cast<uint8_t>(Y);
      continue;
    }
    const int cb = chroma(p, 1, x, y) - 128, cr = chroma(p, 2, x, y) - 128;
    // libjpeg's build_ycc_rgb_table: FIX(1.40200), FIX(1.77200), FIX(0.71414), FIX(0.34414) with 16 fraction bits
    const int R = Y + ((91881 * cr + 32768) >> 16);
    const int G = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
    const int B = Y + ((116130 * cb + 32768) >> 16);
    o[0] = static_cast<uint8_t>(min(max(R, 0), 255));
    o[1] = static_cast<uint8_t>(min(max(G, 0), 255));
    o[2] = static_cast<uint8_t>(min(max(B, 0), 255));
  }
}

// ---- host: header parsing ---------------------------------------------------------------------------------------
struct Header {
  int W = 0, H = 0, ncomp = 0, hs[3] = {1, 1, 1}, vs[3] = {1, 1, 1};
  int restart = 0;
  int64_t ecs0 = 0, ecs1 = 0;
  JTables tab;
};

int be16(const uint8_t* d) { return d[0] << 8 | d[1]; }

// libjpeg's jpeg_make_d_derived_tbl (a table with an all-ones code is bogus; DC symbols above 15 too) plus the LUT.
bool derive(const uint8_t* counts, const uint8_t* vals, int nvals, bool is_dc, JHuff* t) {
  std::memset(t, 0, sizeof(JHuff));
  int codes[256], sizes[256], p = 0;
  for (int l = 1; l <= 16; ++l)
    for (int i = 0; i < counts[l - 1]; ++i) sizes[p++] = l;
  if (p != nvals || p > 256) return false;
  int code = 0, q = 0;
  for (int si = 1; si <= 16; ++si) {
    while (q < p && sizes[q] == si) codes[q++] = code++;
    if (code >= (1 << si)) return false;
    code <<= 1;
  }
  q = 0;
  for (int l = 1; l <= 16; ++l) {
    t->maxcode[l] = -1;
    if (counts[l - 1]) {
      t->valoff[l] = q - codes[q];
      q += counts[l - 1];
      t->maxcode[l] = codes[q - 1];
    }
  }
  t->maxcode[17] = 0xFFFFF;
  for (int i = 0; i < p; ++i) {
    if (is_dc && vals[i] > 15) return false;
    t->vals[i] = vals[i];
    if (sizes[i] <= 9) {
      const int shift = 9 - sizes[i];
      for (int f = 0; f < (1 << shift); ++f) t->lut[(codes[i] << shift) | f] = static_cast<uint16_t>(sizes[i] << 8 | vals[i]);
    }
  }
  return true;
}

// The header of a file the device decodes (see oracle/jpeg_ref.py `parse`, which states the same rules); false for
// any other file.
bool parse(const uint8_t* d, int64_t n, Header* h) {
  if (n < 4 || n > kMaxBytes || d[0] != 0xFF || d[1] != 0xD8) return false;
  int64_t pos = 2;
  bool sof = false, jfif = false;
  int adobe = -1;
  int ids[3] = {0, 0, 0}, tq[3] = {0, 0, 0};
  bool have_q[4] = {}, have_h[2][4] = {};
  uint8_t hcounts[2][4][16], hvals[2][4][256];
  int hn[2][4] = {};
  int32_t qtab[4][64];
  const uint8_t* seg = nullptr;
  int seglen = 0;
  for (;;) {
    if (pos + 4 > n || d[pos] != 0xFF) return false;
    const int m = d[pos + 1];
    if (m == 0xFF || m == 0x01 || (m >= 0xD0 && m <= 0xD9)) return false;
    const int length = be16(d + pos + 2);
    if (length < 2 || pos + 2 + length > n) return false;
    seg = d + pos + 4;
    seglen = length - 2;
    pos += 2 + length;
    if (m == 0xC0 || m == 0xC1) {
      if (sof || seglen < 6) return false;
      const int prec = seg[0], nf = seg[5];
      h->H = be16(seg + 1);
      h->W = be16(seg + 3);
      if (prec != 8 || h->H == 0 || h->W == 0 || (nf != 1 && nf != 3) || seglen != 6 + 3 * nf) return false;
      for (int i = 0; i < nf; ++i) {
        ids[i] = seg[6 + 3 * i];
        h->hs[i] = seg[7 + 3 * i] >> 4;
        h->vs[i] = seg[7 + 3 * i] & 15;
        tq[i] = seg[8 + 3 * i];
        if (h->hs[i] < 1 || h->hs[i] > 4 || h->vs[i] < 1 || h->vs[i] > 4 || tq[i] > 3) return false;
        for (int k = 0; k < i; ++k)
          if (ids[k] == ids[i]) return false;
      }
      if (nf == 3) {
        const int a = h->hs[0], b = h->vs[0];
        if (!((a == 1 && b == 1) || (a == 2 && b == 1) || (a == 2 && b == 2))) return false;
        for (int i = 1; i < 3; ++i)
          if (h->hs[i] != 1 || h->vs[i] != 1) return false;
      } else {
        h->hs[0] = h->vs[0] = 1;   // a single-component scan is non-interleaved: one block per MCU
      }
      h->ncomp = nf;
      sof = true;
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4) {
      return false;
    } else if (m == 0xC4) {
      int i = 0;
      while (i < seglen) {
        const int tcth = seg[i];
        if (tcth & 0xEC) return false;
        if (i + 17 > seglen) return false;
        int total = 0;
        for (int l = 0; l < 16; ++l) total += seg[i + 1 + l];
        if (total > 256 || i + 17 + total > seglen) return false;
        const int tc = tcth >> 4, th = tcth & 3;
        std::memcpy(hcounts[tc][th], seg + i + 1, 16);
        std::memcpy(hvals[tc][th], seg + i + 17, total);
        hn[tc][th] = total;
        have_h[tc][th] = true;
        i += 17 + total;
      }
    } else if (m == 0xDB) {
      int i = 0;
      while (i < seglen) {
        const int pq = seg[i] >> 4, t = seg[i] & 15;
        if (pq != 0 || t > 3 || i + 65 > seglen) return false;
        for (int k = 0; k < 64; ++k) qtab[t][kZigzag[k]] = seg[i + 1 + k];
        have_q[t] = true;
        i += 65;
      }
    } else if (m == 0xDD) {
      if (length != 4) return false;
      h->restart = be16(seg);
    } else if (m == 0xE0) {
      if (seglen >= 14 && std::memcmp(seg, "JFIF\0", 5) == 0) jfif = true;
    } else if (m == 0xEE) {
      if (seglen >= 12 && std::memcmp(seg, "Adobe", 5) == 0) adobe = seg[11];
    } else if ((m >= 0xE1 && m <= 0xEF) || m == 0xFE) {
    } else if (m == 0xDA) {
      break;
    } else {
      return false;
    }
  }
  if (!sof) return false;
  const int ns = seglen > 0 ? seg[0] : 0;
  if (ns != h->ncomp || seglen != 4 + 2 * ns) return false;
  for (int i = 0; i < ns; ++i) {
    const int cid = seg[1 + 2 * i], td = seg[2 + 2 * i] >> 4, ta = seg[2 + 2 * i] & 15;
    if (cid != ids[i] || td > 3 || ta > 3 || !have_h[0][td] || !have_h[1][ta] || !have_q[tq[i]]) return false;
    if (!derive(hcounts[0][td], hvals[0][td], hn[0][td], true, &h->tab.dc[i])) return false;
    if (!derive(hcounts[1][ta], hvals[1][ta], hn[1][ta], false, &h->tab.ac[i])) return false;
    std::memcpy(h->tab.qt[i], qtab[tq[i]], sizeof(qtab[0]));
  }
  if (seg[1 + 2 * ns] != 0 || seg[2 + 2 * ns] != 63 || seg[3 + 2 * ns] != 0) return false;
  if (h->ncomp == 3) {
    if (adobe >= 0 && adobe != 1) return false;
    if (!jfif && adobe < 0 && ids[0] == 82 && ids[1] == 71 && ids[2] == 66) return false;
  }
  // the entropy-coded segment: to the first marker that is neither 0xFF00 nor RSTn, which must be EOI
  h->ecs0 = pos;
  for (int64_t i = pos;; ++i) {
    const uint8_t* f = static_cast<const uint8_t*>(std::memchr(d + i, 0xFF, n - i));
    if (f == nullptr || f + 1 >= d + n) return false;
    i = f - d;
    const int nx = f[1];
    if (nx == 0 || (nx >= 0xD0 && nx <= 0xD7)) {
      ++i;
      continue;
    }
    if (nx != 0xD9) return false;
    h->ecs1 = i;
    break;
  }
  return true;
}

struct Layout {
  int hm, vm, mcux, mcuy, bpm, bw[3], bh[3], blk_comp[6], blk_x[6], blk_y[6];
};

Layout layout(const Header& h) {
  Layout L{};
  if (h.ncomp == 1) {
    L.hm = L.vm = 1;
    L.mcux = (h.W + 7) / 8;
    L.mcuy = (h.H + 7) / 8;
    L.bpm = 1;
    L.bw[0] = L.mcux;
    L.bh[0] = L.mcuy;
    return L;
  }
  L.hm = h.hs[0];
  L.vm = h.vs[0];
  L.mcux = (h.W + 8 * L.hm - 1) / (8 * L.hm);
  L.mcuy = (h.H + 8 * L.vm - 1) / (8 * L.vm);
  for (int c = 0; c < 3; ++c) {
    for (int by = 0; by < h.vs[c]; ++by)
      for (int bx = 0; bx < h.hs[c]; ++bx) {
        L.blk_comp[L.bpm] = c;
        L.blk_x[L.bpm] = bx;
        L.blk_y[L.bpm] = by;
        ++L.bpm;
      }
    L.bw[c] = L.mcux * h.hs[c];
    L.bh[c] = L.mcuy * h.vs[c];
  }
  return L;
}

// The shared body of both entries: coefficients only (coef_out != nullptr: the caller's buffer, photos' planes
// back to back) or the whole decode into the photos' outputs.
int run(const int64_t* photos, int B, int subseq_bits, int16_t* coef_out, int32_t* status, int32_t* passes,
        void* stream) {
  MHMR_REQUIRE(photos != nullptr && status != nullptr, "null argument");
  MHMR_REQUIRE(B >= 1 && B <= 65535, "jpeg: 1 <= B <= 65535 photos");
  MHMR_REQUIRE(subseq_bits >= 1 && subseq_bits <= (1 << 24), "jpeg: 1 <= subsequence bits <= 2^24");
  std::vector<Header> hdr(B);
  std::vector<JPhoto> ph(B);
  std::vector<Chunk> chunks;
  std::vector<JIv> ivs;
  std::vector<PlaneRef> planes;
  int64_t max_sub = 0, coef_elems = 0, plane_bytes = 0, dst_bytes = 0, nblocks = 0;
  int maxW = 0, maxH = 0;
  for (int b = 0; b < B; ++b) {
    const int64_t* d = photos + 7 * b;
    MHMR_REQUIRE(d[0] != 0 && d[2] != 0, "jpeg: null photo bytes");
    MHMR_REQUIRE(d[1] >= 4 && d[1] <= kMaxBytes, "jpeg: file size in [4, 2^28] bytes");
    Header& h = hdr[b];
    MHMR_REQUIRE(parse(reinterpret_cast<const uint8_t*>(d[0]), d[1], &h),
                 "jpeg: a photo is not one the device decodes (mhmr_jpeg_info says which are)");
    MHMR_REQUIRE(d[5] == h.H && d[6] == h.W, "jpeg: output size differs from the header's");
    if (coef_out == nullptr) MHMR_REQUIRE(d[3] != 0 && d[4] >= 3ll * h.W, "jpeg: null output or pitch below 3 W");
    const Layout L = layout(h);
    JPhoto& p = ph[b];
    std::memset(&p, 0, sizeof(p));
    p.ecs = reinterpret_cast<const uint8_t*>(d[2]) + h.ecs0;
    p.ecs_len = static_cast<int>(h.ecs1 - h.ecs0);
    p.chunk0 = static_cast<int>(chunks.size());
    p.nchunk = std::max(1, (p.ecs_len + kChunk - 1) / kChunk);
    for (int c = 0; c < p.nchunk; ++c) chunks.push_back({b, c * kChunk});
    const int mcus = L.mcux * L.mcuy;
    p.per = h.restart > 0 ? h.restart : mcus;
    p.iv0 = static_cast<int>(ivs.size());
    p.niv = (mcus + p.per - 1) / p.per;
    for (int k = 0; k < p.niv; ++k) ivs.push_back({b, k * p.per, std::min(p.per, mcus - k * p.per), 0, 0, 0, 0});
    p.W = h.W;
    p.H = h.H;
    p.ncomp = h.ncomp;
    p.hm = L.hm;
    p.vm = L.vm;
    for (int c = 0; c < 3; ++c) {
      p.hs[c] = h.ncomp == 1 ? 1 : h.hs[c];
      p.vs[c] = h.ncomp == 1 ? 1 : h.vs[c];
      p.bw[c] = c < h.ncomp ? L.bw[c] : 0;
      p.bh[c] = c < h.ncomp ? L.bh[c] : 0;
    }
    p.bpm = L.bpm;
    p.mcux = L.mcux;
    p.mcuy = L.mcuy;
    for (int i = 0; i < 6; ++i) {
      p.blk_comp[i] = L.blk_comp[i];
      p.blk_x[i] = L.blk_x[i];
      p.blk_y[i] = L.blk_y[i];
    }
    p.out = reinterpret_cast<uint8_t*>(d[3]);
    p.pitch = d[4];
    for (int c = 0; c < h.ncomp; ++c) {
      planes.push_back({b, c, static_cast<int>(nblocks)});
      nblocks += static_cast<int64_t>(p.bw[c]) * p.bh[c];
    }
    max_sub += (8ll * p.ecs_len + subseq_bits - 1) / subseq_bits + p.niv;
    dst_bytes += align256(p.ecs_len + kSlack);
    maxW = std::max(maxW, h.W);
    maxH = std::max(maxH, h.H);
  }
  MHMR_REQUIRE(nblocks < (1ll << 31) && max_sub < (1ll << 31) && chunks.size() < (1u << 31) && ivs.size() < (1u << 31),
               "jpeg: batch too large for one call");
  coef_elems = nblocks * 64;
  plane_bytes = nblocks * 64;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int NC = static_cast<int>(chunks.size()), NI = static_cast<int>(ivs.size()), NS = static_cast<int>(max_sub);

  // workspace: [photos | tables | chunks | intervals | planes] (uploaded) then device-only arrays
  CallScratch ws(st);
  const size_t r_ph = ws.region(sizeof(JPhoto) * B, true), r_tab = ws.region(sizeof(JTables) * B, true),
               r_ch = ws.region(sizeof(Chunk) * NC, true), r_iv = ws.region(sizeof(JIv) * NI, true),
               r_pl = ws.region(sizeof(PlaneRef) * planes.size(), true);
  const size_t r_kept = ws.region(4ll * NC), r_marks = ws.region(4ll * NC), r_nsub = ws.region(4),
               r_subiv = ws.region(4ll * NS), r_start = ws.region(8ll * NS), r_end = ws.region(16ll * NS),
               r_cnt = ws.region(4ll * NS), r_dcs = ws.region(12ll * NS), r_cntx = ws.region(4ll * NS),
               r_dcx = ws.region(12ll * NS), r_part = ws.region(16ll * ((NS + 1023) / 1024)), r_done = ws.region(4ll * NI),
               r_flags = ws.region(16), r_dst = ws.region(dst_bytes), r_coef = ws.region(coef_out ? 0 : 2 * coef_elems),
               r_plane = ws.region(coef_out ? 0 : plane_bytes);
  TRY(ws.allocate());
  // device addresses of each photo's destuffed stream, coefficients and planes
  size_t dpos = 0;
  int64_t cpos = 0;
  for (int b = 0; b < B; ++b) {
    JPhoto& p = ph[b];
    p.dst = ws.dev<uint8_t>(r_dst) + dpos;
    dpos += align256(p.ecs_len + kSlack);
    for (int c = 0; c < p.ncomp; ++c) {
      const int64_t n = static_cast<int64_t>(p.bw[c]) * p.bh[c] * 64;
      p.coef[c] = (coef_out ? coef_out : ws.dev<int16_t>(r_coef)) + cpos;
      if (!coef_out) p.plane[c] = ws.dev<uint8_t>(r_plane) + cpos;
      cpos += n;
    }
  }
  std::memcpy(ws.host<JPhoto>(r_ph), ph.data(), sizeof(JPhoto) * B);
  for (int b = 0; b < B; ++b) ws.host<JTables>(r_tab)[b] = hdr[b].tab;
  std::memcpy(ws.host<Chunk>(r_ch), chunks.data(), sizeof(Chunk) * NC);
  std::memcpy(ws.host<JIv>(r_iv), ivs.data(), sizeof(JIv) * NI);
  std::memcpy(ws.host<PlaneRef>(r_pl), planes.data(), sizeof(PlaneRef) * planes.size());

  Ctx ctx{};
  ctx.ph = ws.dev<const JPhoto>(r_ph);
  ctx.tab = ws.dev<const JTables>(r_tab);
  ctx.iv = ws.dev<JIv>(r_iv);
  ctx.niv = NI;
  ctx.subseq_bits = subseq_bits;
  ctx.max_sub = NS;
  ctx.nsub = ws.dev<int>(r_nsub);
  ctx.sub_iv = ws.dev<int>(r_subiv);
  ctx.start = ws.dev<int2>(r_start);
  ctx.endst = ws.dev<int2>(r_end);
  ctx.cnt = ws.dev<int>(r_cnt);
  ctx.dcs = ws.dev<uint32_t>(r_dcs);
  ctx.cntx = ws.dev<int>(r_cntx);
  ctx.dcx = ws.dev<uint32_t>(r_dcx);
  ctx.part = ws.dev<uint32_t>(r_part);
  ctx.nparts = (NS + 1023) / 1024;
  ctx.done = ws.dev<int>(r_done);
  ctx.flags = ws.dev<int>(r_flags);
  ctx.passes = passes;
  ctx.status = status;
  const Chunk* dch = ws.dev<const Chunk>(r_ch);
  int* kept = ws.dev<int>(r_kept);
  int* marks = ws.dev<int>(r_marks);

  static PerDeviceOnce once;
  static int coop_blocks[64];
  int dev = 0;
  MHMR_CUDA_CHECK(cudaGetDevice(&dev));
  if (once.first()) {
    MHMR_CUDA_CHECK(cudaMemcpyToSymbol(c_zigzag, kZigzag, 64));
    int per_sm = 0;
    MHMR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, huff_sync_kernel, 256, 0));
    coop_blocks[dev] = std::max(1, per_sm) * device_sm_count();
  }
  TRY(ws.upload());
  MHMR_CUDA_CHECK(cudaMemsetAsync(status, 0, 4ll * B, st));
  MHMR_CUDA_CHECK(cudaMemsetAsync(ctx.done, 0, ws.dev<uint8_t>(r_dst) - ws.dev<uint8_t>(r_done), st));   // done, flags
  MHMR_CUDA_CHECK(cudaMemsetAsync(ws.dev<uint8_t>(r_dst), 0, dst_bytes, st));   // the zero slack after each stream
  MHMR_CUDA_CHECK(cudaMemsetAsync(coef_out ? coef_out : ws.dev<int16_t>(r_coef), 0, 2 * coef_elems, st));
  seg_count_kernel<<<NC, 256, 0, st>>>(ctx.ph, dch, kept, marks);
  MHMR_CUDA_CHECK(cudaGetLastError());
  seg_scan_kernel<<<B, 1024, 0, st>>>(ctx.ph, ctx.iv, kept, marks, status);
  MHMR_CUDA_CHECK(cudaGetLastError());
  seg_write_kernel<<<NC, 256, 0, st>>>(ctx.ph, dch, kept, marks, ctx.iv, status);
  MHMR_CUDA_CHECK(cudaGetLastError());
  plan_kernel<<<1, 1024, 0, st>>>(ctx);
  MHMR_CUDA_CHECK(cudaGetLastError());
  sub_map_kernel<<<(NS + 255) / 256, 256, 0, st>>>(ctx);
  MHMR_CUDA_CHECK(cudaGetLastError());
  const int grid = static_cast<int>(std::min<int64_t>(coop_blocks[dev], (NS + 255) / 256));
  void* args[] = {&ctx};
  MHMR_CUDA_CHECK(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(huff_sync_kernel), dim3(grid), dim3(256), args,
                                              0, st));
  sub_tile_sum_kernel<<<ctx.nparts, 1024, 0, st>>>(ctx);
  MHMR_CUDA_CHECK(cudaGetLastError());
  sub_tile_scan_kernel<<<1, 1024, 0, st>>>(ctx);
  MHMR_CUDA_CHECK(cudaGetLastError());
  sub_scan_kernel<<<ctx.nparts, 1024, 0, st>>>(ctx);
  MHMR_CUDA_CHECK(cudaGetLastError());
  huff_write_kernel<<<(NS + 255) / 256, 256, 0, st>>>(ctx);
  MHMR_CUDA_CHECK(cudaGetLastError());
  check_done_kernel<<<(NI + 255) / 256, 256, 0, st>>>(ctx);
  MHMR_CUDA_CHECK(cudaGetLastError());
  if (!coef_out) {
    idct_kernel<<<static_cast<int>((nblocks + 31) / 32), 256, 0, st>>>(
        ctx.ph, ctx.tab, ws.dev<const PlaneRef>(r_pl), static_cast<int>(planes.size()), static_cast<int>(nblocks), status);
    MHMR_CUDA_CHECK(cudaGetLastError());
    const dim3 cgrid((maxW + 255) / 256, std::min(maxH, 1024), B);
    color_kernel<<<cgrid, 256, 0, st>>>(ctx.ph);
    MHMR_CUDA_CHECK(cudaGetLastError());
  }
  return ws.release();
}

}  // namespace

extern "C" {

int mhmr_jpeg_info(const uint8_t* data, int64_t nbytes, int* info) {
  MHMR_REQUIRE(data != nullptr && info != nullptr && nbytes >= 0, "null argument");
  Header h;
  const bool ok = parse(data, nbytes, &h);
  info[0] = ok ? h.W : 0;
  info[1] = ok ? h.H : 0;
  info[2] = ok ? h.ncomp : 0;
  info[3] = ok ? (h.ncomp == 3 ? h.hs[0] : 1) : 0;
  info[4] = ok ? (h.ncomp == 3 ? h.vs[0] : 1) : 0;
  info[5] = ok ? 1 : 0;
  return MHMR_OK;
}

int mhmr_op_jpeg_decode(const int64_t* photos, int B, int32_t* status, void* stream) {
  return run(photos, B, kDefaultSubseqBits, nullptr, status, nullptr, stream);
}

int mhmr_op_jpeg_coefficients(const int64_t* photos, int B, int subseq_bits, int16_t* coefs, int32_t* status,
                              int32_t* passes, void* stream) {
  MHMR_REQUIRE(coefs != nullptr, "null coefficient buffer");
  return run(photos, B, subseq_bits, coefs, status, passes, stream);
}

}  // extern "C"
