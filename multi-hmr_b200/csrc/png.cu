// PNG -> RGB on the device, byte for byte equal to Pillow's `Image.open(f).convert("RGB")` (the arithmetic is restated
// in oracle/png_ref.py and pinned against Pillow and zlib there).
//
// The host walks each file's chunks, decides eligibility (8-bit, non-interlaced gray, RGB, palette, gray + alpha or
// RGBA; see `parse`) and the caller uploads every photo's IDAT payloads back to back: one zlib stream per photo.
// The device then runs, for the whole batch (pugz, Kerbiriou & Chikhi 2019; rapidgzip, Knespel & Brunst 2023):
//   search    one thread per bit offset of each stream tests whether a dynamic-Huffman block header starts there,
//             with every check zlib's inflate makes of one (HLIT <= 286, HDIST <= 30, a complete code-length code,
//             repeats that neither start the list nor overrun it, a nonzero end-of-block length, both codes neither
//             over-subscribed nor incomplete unless they hold one code).  A warp's answers go into a bitmap word;
//             one CTA per photo then compacts them into the photo's candidate list, in bit order.
//   measure   one thread per candidate decodes its block to the end-of-block code without any window and records
//             the end bit, the output length, the farthest reference before the block's first byte and any error.
//             Nothing is written.
//   chain     one thread per photo checks the zlib header and follows the real blocks from bit 16: end -> next start
//             until the BFINAL block.  A start that is a candidate takes its measurement; any other start (a stored
//             or fixed-Huffman block, or a header the search did not see) is measured there and then, by the same
//             function.  The chain is the sequential decode by construction: a false candidate is never reached,
//             and a stream of fixed-Huffman blocks degrades to a sequential measurement, never to a wrong byte.
//   emit      one thread per chain block decodes again, into a 32-bit symbol per output byte: a literal, or, for a
//             copy whose source lies before the block's first byte, a placeholder holding the source's position.  A
//             copy of a placeholder copies the placeholder, so every placeholder of block k points before block k.
//   resolve   one CTA per photo takes the blocks in order; once blocks < k are final it replaces block k's
//             placeholders by the bytes they point at, and sums Adler-32 over the bytes (per-thread sums, combined).
//   unfilter  one CTA per photo undoes None / Sub / Up / Average / Paeth in place on a skewed wavefront: lane l of a
//             warp takes row r0 + l and at step s pixel s - l, so the pixel above comes from lane l - 1 by shuffle.
//             The CTA's warps take consecutive 32-row bands; lane 0 of a band reads the row above from memory once
//             the warp of the band before has published, in a shared-memory counter, that it got that far.  The
//             same pass writes HWC RGB at the caller's pitch: gray replicated, alpha dropped, palette looked up.
// Anything the device cannot vouch for sets a bit of the photo's status instead (kBad* below) and the caller decodes
// that photo with Pillow, which then decodes it or raises as it always did.
//
// Memory safety for any content of the streams: each stream is copied into the workspace with 8 zero bytes after
// it, and the bit reader reads a word only inside that copy (zeros past it), so a read never leaves the photo's span.  Every
// decode stops at the first bit past the stream (kBadChain) and at more output than the photo's expected length
// (kBadLength); emits write symbol q of a chain block only for q below that block's measured length, inside the
// photo's expected length.  A placeholder is honoured only when it indexes [0, block start), and resolve writes
// only [0, expected length).  The unfilter reads and writes only the inflated buffer (rows of the expected length,
// filter byte included) and writes the output at rows < H, columns < 3 W, of the caller's pitch.  Candidate and chain
// lists are capped; a capped search only loses speed, a capped chain flags the photo.  The workspace is
// stream-ordered (CallScratch).
#include "common.cuh"

#include <algorithm>
#include <cstring>
#include <vector>

using namespace mhmr;

namespace {

// status bits (oracle/png_ref.py has the same values)
constexpr int kBadCode = 1;     // invalid block type, stored length, code-length code, code lengths, tree or code
constexpr int kBadDist = 2;     // a distance reaching before the stream's first byte
constexpr int kBadChain = 4;    // a block reading past the stream, or more blocks than the chain holds
constexpr int kBadLength = 8;   // inflated length other than H (1 + row bytes)
constexpr int kBadFilter = 16;  // a filter byte above 4
constexpr int kBadAdler = 32;   // Adler-32 missing or different
constexpr int kBadHeader = 64;  // CMF / FLG check, method, window size or a preset dictionary

constexpr int64_t kMaxBytes = 1ll << 28;      // per stream: bit positions stay below 2^31
constexpr int64_t kMaxInflated = 1ll << 30;   // per photo: placeholders hold 31-bit positions
constexpr int kSlack = 8;                     // zero bytes after each stream copy
constexpr int kLitLut = 10, kDistLut = 8;     // first-level lookup bits of the decoders
constexpr int kUnfilterWarps = 16;

__host__ __device__ inline int64_t chain_cap(int64_t expect) { return 1024 + expect / 64; }
__host__ __device__ inline int64_t cand_cap(int64_t nbytes) { return 1024 + nbytes / 64; }

struct PPhoto {
  const uint32_t* words;   // the stream's copy (device), nbytes + kSlack zero bytes, 4-byte aligned
  int64_t nbytes;
  int64_t expect;          // inflated bytes: H (1 + row bytes)
  uint32_t* sym;           // expect emitted symbols
  uint8_t* inf;            // expect inflated bytes (the caller's buffer for mhmr_op_png_inflate)
  uint32_t* bitmap;        // one bit per stream bit offset: a candidate header starts there
  int64_t* cand;           // candidate bit offsets, in order
  int64_t* chain;          // [chain_cap][2]: start bit, first output byte of each chain block
  uint8_t* out;            // RGB output (nullptr: inflate only)
  int64_t pitch;
  int64_t word0;           // first bitmap word of this photo in the batch's bitmap
  int W, H, ctype, bpp;
  int ncand_cap, nchain_cap;
  uint8_t pal[768];        // palette entries, zero past the PLTE's (Pillow's convert gives 0, 0, 0 there)
};

struct PState {
  int ncand;               // candidates found (all of them; the first ncand_cap are kept)
  int nchain;              // blocks of the chain
  int nslow;               // chain blocks that were not candidates
  int final_seen;
  int64_t total;           // inflated bytes the chain produced
  int64_t adler_pos;       // byte offset of the stored Adler-32
};

struct Meas {
  int64_t end;             // bit after the block's end-of-block code
  int64_t len;             // output bytes (up to the error, if any)
  int64_t far;             // farthest reference before the block's first byte (0 if none)
  int err;
  int final;
};

// ---- bit reader ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t peek32(const PPhoto& P, int64_t pos) {
  const int64_t nw = (P.nbytes + kSlack) / 4;
  const int64_t w = pos >> 5;
  if (w < 0 || w > nw - 2) return 0;   // past the zero slack: the stream reads as zeros
  const uint32_t lo = __ldg(P.words + w), hi = __ldg(P.words + w + 1);
  return __funnelshift_r(lo, hi, static_cast<uint32_t>(pos & 31));
}

// ---- Huffman codes ------------------------------------------------------------------------------------------------
__constant__ uint16_t c_len_base[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                        31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                         193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

enum CodeKind { kCodes, kLens, kDists };

// zlib's inflate_table verdict on a set of code lengths: over-subscribed is bad; incomplete is bad unless the code
// holds a single code of length 1 in a literal / length or distance code; no code at all is bad for the code-length
// code (every list it could decode lacks an end-of-block code) and fine for distances (using one is then an error).
__device__ bool lengths_ok(const uint8_t* lens, int n, CodeKind kind) {
  int count[16] = {0};
  for (int i = 0; i < n; ++i) count[lens[i]]++;
  int max = 15;
  while (max >= 1 && count[max] == 0) --max;
  if (max == 0) return kind == kDists;
  int left = 1;
  for (int l = 1; l <= 15; ++l) {
    left = (left << 1) - count[l];
    if (left < 0) return false;
  }
  return !(left > 0 && (kind == kCodes || max != 1));
}

template <int LUT, int N>
struct Huff {
  uint16_t lut[1 << LUT];   // next LUT stream bits -> (length << 9 | symbol), 0 for a longer or invalid code
  uint16_t lim[16];         // left-justified (15-bit) end of the codes of each length
  int16_t off[16];          // index in sym of a length's first code, minus that code
  uint16_t sym[N];          // symbols by (length, value)
};

// Canonical codes from lengths already judged by lengths_ok.
template <int LUT, int N>
__device__ void build(const uint8_t* lens, int n, Huff<LUT, N>& h) {
  int count[16] = {0};
  for (int i = 0; i < n; ++i) count[lens[i]]++;
  count[0] = 0;
  int first[16], idx[16];
  int code = 0, k = 0;
  for (int l = 1; l <= 15; ++l) {
    code = (code + count[l - 1]) << 1;
    first[l] = code;
    idx[l] = k;
    h.off[l] = static_cast<int16_t>(k - code);
    k += count[l];
    h.lim[l] = static_cast<uint16_t>((code + count[l]) << (15 - l));
  }
  for (int i = 0; i < (1 << LUT); ++i) h.lut[i] = 0;
  int next[16];
  for (int l = 1; l <= 15; ++l) next[l] = first[l];
  for (int s = 0; s < n; ++s) {
    const int l = lens[s];
    if (l == 0) continue;
    h.sym[idx[l]++] = static_cast<uint16_t>(s);
    const int c = next[l]++;
    if (l <= LUT) {
      const uint32_t rev = __brev(static_cast<uint32_t>(c)) >> (32 - l);   // stream order: first bit lowest
      for (uint32_t f = rev; f < (1u << LUT); f += (1u << l)) h.lut[f] = static_cast<uint16_t>(l << 9 | s);
    }
  }
}

// One symbol from the bits at `bits` (stream order); returns the symbol and sets `len`, or returns -1 (no code).
template <int LUT, int N>
__device__ __forceinline__ int decode_sym(const Huff<LUT, N>& h, uint32_t bits, int& len) {
  const uint16_t e = h.lut[bits & ((1u << LUT) - 1)];
  if (e) {
    len = e >> 9;
    return e & 511;
  }
  const uint32_t v = __brev(bits) >> 17;   // the next 15 bits in code order
  for (int l = LUT + 1; l <= 15; ++l) {
    if (v < h.lim[l]) {
      len = l;
      return h.sym[h.off[l] + static_cast<int>(v >> (15 - l))];
    }
  }
  return -1;
}

struct Tables {
  Huff<kLitLut, 288> lit;
  Huff<kDistLut, 32> dist;
  int nlit, ndist;
};

// Reads a dynamic block's header after its 3 type bits, from `pos` (advanced past it), into `lens` (nlit + ndist
// lengths).  Returns 0 or kBadCode; with `end` = 8 nbytes, a header running past the stream is kBadChain.
__device__ int read_dynamic(const PPhoto& P, int64_t& pos, int64_t end, uint8_t* lens, int& nlit, int& ndist) {
  uint32_t b = peek32(P, pos);
  nlit = (b & 31) + 257;
  ndist = ((b >> 5) & 31) + 1;
  const int ncl = ((b >> 10) & 15) + 4;
  pos += 14;
  if (nlit > 286 || ndist > 30) return kBadCode;
  uint8_t cl[19];
  for (int i = 0; i < 19; ++i) cl[i] = 0;
  for (int i = 0; i < ncl; ++i) cl[c_cl_order[i]] = (peek32(P, pos + 3 * i) & 7);
  pos += 3 * ncl;
  if (pos > end) return kBadChain;
  if (!lengths_ok(cl, 19, kCodes)) return kBadCode;
  Huff<7, 19> h;
  build(cl, 19, h);
  const int total = nlit + ndist;
  int have = 0;
  while (have < total) {
    b = peek32(P, pos);
    int l = 0;
    const int s = decode_sym(h, b, l);   // the code-length code is complete: always a symbol
    pos += l;
    b >>= l;
    if (s < 16) {
      lens[have++] = static_cast<uint8_t>(s);
    } else {
      int rep;
      uint8_t v = 0;
      if (s == 16) {
        if (have == 0) return kBadCode;
        v = lens[have - 1];
        rep = 3 + (b & 3);
        pos += 2;
      } else if (s == 17) {
        rep = 3 + (b & 7);
        pos += 3;
      } else {
        rep = 11 + (b & 127);
        pos += 7;
      }
      if (have + rep > total) return kBadCode;
      for (int i = 0; i < rep; ++i) lens[have++] = v;
    }
    if (pos > end) return kBadChain;
  }
  if (lens[256] == 0) return kBadCode;
  if (!lengths_ok(lens, nlit, kLens) || !lengths_ok(lens + nlit, ndist, kDists)) return kBadCode;
  return 0;
}

// Decodes the block starting at bit `start` (its 3 header bits included) without any window.  Measuring (EMIT
// false) fills m; emitting writes the block's symbols at sym[obase ..], at most `room` of them.  Output beyond
// `cap` bytes is kBadLength.
template <bool EMIT>
__device__ void decode_block(const PPhoto& P, int64_t start, int64_t cap, int64_t obase, int64_t room, Tables& T,
                             Meas& m) {
  const int64_t end = 8 * P.nbytes;
  int64_t pos = start;
  m.err = 0;
  m.len = 0;
  m.far = 0;
  m.end = start;
  uint32_t b = peek32(P, pos);
  m.final = b & 1;
  const int type = (b >> 1) & 3;
  pos += 3;
  if (type == 3) {
    m.err = kBadCode;
    return;
  }
  if (type == 0) {
    pos = (pos + 7) & ~int64_t(7);
    b = peek32(P, pos);
    const int64_t len = b & 0xffff;
    if ((b >> 16) != (~b & 0xffff)) {
      m.err = pos + 32 > end ? kBadChain : kBadCode;
      return;
    }
    pos += 32;
    if (pos + 8 * len > end) {
      m.err = kBadChain;
      return;
    }
    if (len > cap) {
      m.err = kBadLength;
      return;
    }
    if (EMIT) {
      for (int64_t i = 0; i < len && i < room; ++i) P.sym[obase + i] = (peek32(P, pos + 8 * i) & 255);
    }
    m.len = len;
    m.end = pos + 8 * len;
    return;
  }
  if (type == 1) {
    uint8_t lens[320];
    for (int i = 0; i < 144; ++i) lens[i] = 8;
    for (int i = 144; i < 256; ++i) lens[i] = 9;
    for (int i = 256; i < 280; ++i) lens[i] = 7;
    for (int i = 280; i < 288; ++i) lens[i] = 8;
    for (int i = 0; i < 32; ++i) lens[288 + i] = 5;
    build(lens, 288, T.lit);
    build(lens + 288, 32, T.dist);
    T.nlit = 286;   // 286, 287 and distances 30, 31 have codes but no meaning
    T.ndist = 30;
  } else {
    uint8_t lens[320];
    int nlit, ndist;
    const int e = read_dynamic(P, pos, end, lens, nlit, ndist);
    if (e) {
      m.err = e;
      return;
    }
    build(lens, nlit, T.lit);
    bool any = false;
    for (int i = 0; i < ndist; ++i) any |= lens[nlit + i] != 0;
    if (any) build(lens + nlit, ndist, T.dist);
    T.nlit = nlit;
    T.ndist = any ? ndist : 0;
  }
  int64_t n = 0;
  for (;;) {
    if (pos > end) {
      m.err = kBadChain;
      break;
    }
    b = peek32(P, pos);
    int l = 0;
    const int s = decode_sym(T.lit, b, l);
    if (s < 0 || s >= T.nlit) {
      m.err = kBadCode;
      break;
    }
    pos += l;
    if (s < 256) {
      if (n >= cap) {
        m.err = kBadLength;
        break;
      }
      if (EMIT && n < room) P.sym[obase + n] = static_cast<uint32_t>(s);
      ++n;
      continue;
    }
    if (s == 256) {
      if (pos > end) m.err = kBadChain;
      break;
    }
    const int li = s - 257;
    int64_t len = c_len_base[li] + (c_len_extra[li] ? ((b >> l) & ((1u << c_len_extra[li]) - 1)) : 0);
    pos += c_len_extra[li];
    b = peek32(P, pos);
    const int ds = T.ndist ? decode_sym(T.dist, b, l) : -1;
    if (ds < 0 || ds >= T.ndist) {
      m.err = kBadCode;
      break;
    }
    const int64_t dist = c_dist_base[ds] + (c_dist_extra[ds] ? ((b >> l) & ((1u << c_dist_extra[ds]) - 1)) : 0);
    pos += l + c_dist_extra[ds];
    if (dist - n > m.far) m.far = dist - n;
    if (n + len > cap) {
      m.err = kBadLength;
      break;
    }
    if (EMIT) {
      for (int64_t i = 0; i < len && n + i < room; ++i) {
        const int64_t src = n + i - dist;
        uint32_t v;
        if (src >= 0) v = P.sym[obase + src];                    // a byte or a placeholder of this block
        else v = 0x80000000u | static_cast<uint32_t>(obase + src < 0 ? 0 : obase + src);
        P.sym[obase + n + i] = v;
      }
    }
    n += len;
  }
  m.len = n;
  m.end = pos;
}

// ---- search -------------------------------------------------------------------------------------------------------
// One thread per (photo, bit offset): the photo's bitmap words are contiguous, so a warp's ballot is one word.
__global__ void __launch_bounds__(256) search_kernel(const PPhoto* __restrict__ ph, int B, int64_t total_words) {
  const int64_t g = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t word = g >> 5;
  if (word >= total_words) return;   // whole warps leave together
  int lo = 0, hi = B - 1;   // the last photo whose first word is at or before `word`
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (ph[mid].word0 <= word) lo = mid;
    else hi = mid - 1;
  }
  const PPhoto& P = ph[lo];
  const int64_t pos = 32 * (word - P.word0) + (g & 31);
  bool hit = false;
  const int64_t end = 8 * P.nbytes;
  if (pos >= 16 && pos + 17 <= end) {
    const uint32_t b = peek32(P, pos);
    if (((b >> 1) & 3) == 2 && ((b >> 3) & 31) <= 29 && ((b >> 8) & 31) <= 29) {
      uint8_t lens[320];
      int nlit, ndist;
      int64_t q = pos + 3;
      hit = read_dynamic(P, q, end, lens, nlit, ndist) == 0;
    }
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, hit);
  if ((g & 31) == 0) P.bitmap[word - P.word0] = bal;
}

// One CTA per photo: the set bits of its bitmap, in order, into its candidate list (the first ncand_cap of them).
__global__ void __launch_bounds__(1024) compact_kernel(const PPhoto* __restrict__ ph, PState* st) {
  const PPhoto& P = ph[blockIdx.x];
  const int64_t nw = (8 * P.nbytes + 31) / 32;
  const int64_t per = (nw + 1023) / 1024;
  const int64_t w0 = threadIdx.x * per, w1 = min(nw, w0 + per);
  int cnt = 0;
  for (int64_t w = w0; w < w1; ++w) cnt += __popc(P.bitmap[w]);
  __shared__ int part[1024];
  part[threadIdx.x] = cnt;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int v = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  int k = part[threadIdx.x] - cnt;
  for (int64_t w = w0; w < w1 && k < P.ncand_cap; ++w) {
    uint32_t m = P.bitmap[w];
    while (m && k < P.ncand_cap) {
      P.cand[k++] = 32 * w + __ffs(m) - 1;
      m &= m - 1;
    }
  }
  if (threadIdx.x == 1023) st[blockIdx.x].ncand = part[1023];
}

// ---- measure ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) measure_kernel(const PPhoto* __restrict__ ph, const PState* __restrict__ st,
                                                      const int* __restrict__ cand_start, int B, int total,
                                                      Meas* meas) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  int p = 0, hi = B - 1;   // the last photo whose first candidate slot is at or before g
  while (p < hi) {
    const int mid = (p + hi + 1) >> 1;
    if (cand_start[mid] <= g) p = mid;
    else hi = mid - 1;
  }
  const int k = g - cand_start[p];
  const PPhoto& P = ph[p];
  if (k >= min(st[p].ncand, P.ncand_cap)) return;
  Tables T;
  decode_block<false>(P, P.cand[k], P.expect, 0, 0, T, meas[g]);
}

// ---- chain --------------------------------------------------------------------------------------------------------
__global__ void chain_kernel(const PPhoto* __restrict__ ph, PState* st, const int* __restrict__ cand_start,
                             const Meas* __restrict__ meas, int32_t* status) {
  if (threadIdx.x != 0) return;
  const int p = blockIdx.x;
  const PPhoto& P = ph[p];
  PState& S = st[p];
  S.nchain = 0;
  S.nslow = 0;
  S.final_seen = 0;
  S.total = 0;
  S.adler_pos = 0;
  const uint32_t h = peek32(P, 0);
  const int cmf = h & 255, flg = (h >> 8) & 255;
  if (P.nbytes < 2 || (cmf * 256 + flg) % 31 != 0 || (cmf & 15) != 8 || (cmf >> 4) > 7 || (flg & 32)) {
    status[p] = kBadHeader;
    return;
  }
  const int nc = min(S.ncand, P.ncand_cap);
  const Meas* pm = meas + cand_start[p];
  Tables T;
  int64_t pos = 16, total = 0;
  int err = 0;
  for (;;) {
    if (S.nchain >= P.nchain_cap) {
      err = kBadChain;
      break;
    }
    int lo = 0, hi = nc;   // the first candidate at or after pos
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (P.cand[mid] < pos) lo = mid + 1;
      else hi = mid;
    }
    Meas m;
    if (lo < nc && P.cand[lo] == pos) {
      m = pm[lo];
    } else {
      decode_block<false>(P, pos, P.expect, 0, 0, T, m);
      S.nslow++;
    }
    if (m.far > total) err = kBadDist;
    else if (m.err) err = m.err;
    else if (total + m.len > P.expect) err = kBadLength;
    if (err) break;
    P.chain[2 * S.nchain] = pos;
    P.chain[2 * S.nchain + 1] = total;
    S.nchain++;
    total += m.len;
    pos = m.end;
    if (m.final) {
      S.final_seen = 1;
      break;
    }
  }
  S.total = total;
  if (!err && total != P.expect) err = kBadLength;
  if (!err) {
    S.adler_pos = (pos + 7) >> 3;
    if (S.adler_pos + 4 > P.nbytes) err = kBadAdler;
  }
  status[p] = err;
}

// ---- emit ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64) emit_kernel(const PPhoto* __restrict__ ph, const PState* __restrict__ st,
                                                  const int32_t* __restrict__ status) {
  const int p = blockIdx.y;
  if (status[p] != 0) return;
  const PPhoto& P = ph[p];
  const int nb = st[p].nchain;
  Tables T;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < nb; k += gridDim.x * blockDim.x) {
    const int64_t start = P.chain[2 * k], obase = P.chain[2 * k + 1];
    const int64_t next = k + 1 < nb ? P.chain[2 * k + 3] : st[p].total;
    Meas m;
    decode_block<true>(P, start, P.expect, obase, next - obase, T, m);
  }
}

// ---- resolve and Adler-32 -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) resolve_kernel(const PPhoto* __restrict__ ph, const PState* __restrict__ st,
                                                       int32_t* status) {
  const int p = blockIdx.x;
  if (status[p] != 0) return;
  const PPhoto& P = ph[p];
  const int nb = st[p].nchain;
  const int64_t n = P.expect;
  uint64_t a = 0, bsum = 0;
  for (int k = 0; k < nb; ++k) {
    const int64_t s = P.chain[2 * k + 1], e = k + 1 < nb ? P.chain[2 * k + 3] : n;
    for (int64_t i = s + threadIdx.x; i < e; i += blockDim.x) {
      const uint32_t v = P.sym[i];
      uint32_t byte;
      if (v & 0x80000000u) {
        const int64_t src = v & 0x7fffffffu;
        byte = src < s ? P.inf[src] : 0;
      } else {
        byte = v & 255;
      }
      P.inf[i] = static_cast<uint8_t>(byte);
      a += byte;
      bsum += static_cast<uint64_t>((n - i) % 65521) * byte;
    }
    __syncthreads();
  }
  // Adler-32 = (b << 16) | a with a = 1 + sum s_i, b = n + sum (n - i) s_i, both mod 65521
  a %= 65521;
  bsum %= 65521;
  __shared__ uint32_t ra[32], rb[32];
  for (int o = 16; o; o >>= 1) {
    a += __shfl_down_sync(0xffffffffu, a, o);
    bsum += __shfl_down_sync(0xffffffffu, bsum, o);
  }
  if ((threadIdx.x & 31) == 0) {
    ra[threadIdx.x >> 5] = static_cast<uint32_t>(a);
    rb[threadIdx.x >> 5] = static_cast<uint32_t>(bsum);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t A = 1, Bs = static_cast<uint64_t>(n % 65521);
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) {
      A += ra[w];
      Bs += rb[w];
    }
    A %= 65521;
    Bs %= 65521;
    const int64_t q = st[p].adler_pos;
    const uint32_t lo = peek32(P, 8 * q);
    const uint32_t want = (lo & 255) << 24 | ((lo >> 8) & 255) << 16 | ((lo >> 16) & 255) << 8 | (lo >> 24);
    if (want != static_cast<uint32_t>(Bs << 16 | A)) status[p] = kBadAdler;
  }
}

// ---- unfilter and expand ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t recon_byte(int ft, uint32_t f, uint32_t left, uint32_t up, uint32_t ul) {
  switch (ft) {
    case 1: return (f + left) & 255;
    case 2: return (f + up) & 255;
    case 3: return (f + ((left + up) >> 1)) & 255;
    case 4: {
      const int pp = static_cast<int>(left + up) - static_cast<int>(ul);
      const int pa = abs(pp - static_cast<int>(left)), pb = abs(pp - static_cast<int>(up)),
                pc = abs(pp - static_cast<int>(ul));
      const uint32_t pred = (pa <= pb && pa <= pc) ? left : (pb <= pc ? up : ul);
      return (f + pred) & 255;
    }
    default: return f;
  }
}

__global__ void __launch_bounds__(kUnfilterWarps * 32) unfilter_kernel(const PPhoto* __restrict__ ph, int32_t* status) {
  const int p = blockIdx.x;
  const PPhoto& P = ph[p];
  __shared__ uint8_t pal[768];
  __shared__ volatile long long prog[kUnfilterWarps];
  __shared__ int ok;
  if (threadIdx.x == 0) ok = status[p] == 0;
  for (int i = threadIdx.x; i < 768; i += blockDim.x) pal[i] = P.pal[i];
  if (threadIdx.x < kUnfilterWarps) prog[threadIdx.x] = 0;
  __syncthreads();
  if (!ok || P.out == nullptr) return;
  const int W = P.W, H = P.H, bpp = P.bpp, ct = P.ctype;
  const int64_t stride = 1 + static_cast<int64_t>(W) * bpp;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long S = W + 31;   // steps per band
  const int bands = (H + 31) / 32;
  uint8_t* inf = P.inf;
  bool bad = false;
  for (int band = warp, j = 0; band < bands; band += kUnfilterWarps, ++j) {
    const int r = band * 32 + lane;
    const bool row = r < H;
    uint8_t* line = inf + r * stride;
    const int ft = row ? line[0] : 0;
    bad |= ft > 4;
    const int pw = (band - 1) % kUnfilterWarps;   // the warp of the band above (band >= 1)
    const long long pbase = static_cast<long long>((band - 1) / kUnfilterWarps) * S;
    long long seen = 0;
    const volatile uint8_t* above = band > 0 ? inf + (static_cast<int64_t>(band) * 32 - 1) * stride + 1 : nullptr;
    uint32_t left = 0, ul = 0, res = 0;
    for (long long s = 0; s < S; ++s) {
      if (band > 0) {   // lane 0 reads pixel s of the row above: the band above must have finished step s + 31
        const long long need = pbase + min(s + 32, S);
        while (seen < need) {
          seen = __shfl_sync(0xffffffffu, prog[pw], 0);
        }
        __threadfence_block();
      }
      uint32_t up = __shfl_up_sync(0xffffffffu, res, 1);
      const int x = static_cast<int>(s) - lane;
      if (row && x >= 0 && x < W) {
        if (lane == 0) {
          up = 0;
          if (band > 0)
            for (int c = 0; c < bpp; ++c) up |= static_cast<uint32_t>(above[static_cast<int64_t>(x) * bpp + c]) << (8 * c);
        }
        uint8_t* px = line + 1 + static_cast<int64_t>(x) * bpp;
        uint32_t v = 0;
        for (int c = 0; c < bpp; ++c) {
          const uint32_t sh = 8 * c;
          const uint32_t o = recon_byte(ft, px[c], (left >> sh) & 255, (up >> sh) & 255, (ul >> sh) & 255);
          px[c] = static_cast<uint8_t>(o);
          v |= o << sh;
        }
        left = v;
        ul = up;
        res = v;
        uint8_t* o = P.out + r * P.pitch + 3ll * x;
        if (ct == 3) {
          const int e = 3 * (v & 255);
          o[0] = pal[e];
          o[1] = pal[e + 1];
          o[2] = pal[e + 2];
        } else if (ct == 0 || ct == 4) {
          o[0] = o[1] = o[2] = static_cast<uint8_t>(v);
        } else {
          o[0] = static_cast<uint8_t>(v);
          o[1] = static_cast<uint8_t>(v >> 8);
          o[2] = static_cast<uint8_t>(v >> 16);
        }
      } else if (row && x < 0) {
        res = 0;
      }
      if ((s & 31) == 31 || s == S - 1) {
        __threadfence_block();
        __syncwarp();
        if (lane == 0) prog[warp] = static_cast<long long>(j) * S + s + 1;
      }
    }
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status + p, kBadFilter);
}

// ---- host: chunk walk ---------------------------------------------------------------------------------------------
uint32_t be32(const uint8_t* d) { return uint32_t(d[0]) << 24 | uint32_t(d[1]) << 16 | uint32_t(d[2]) << 8 | d[3]; }

uint32_t crc32(const uint8_t* d, int64_t n, uint32_t c = 0) {
  static uint32_t table[256];
  static bool init = false;
  if (!init) {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t v = i;
      for (int k = 0; k < 8; ++k) v = v & 1 ? 0xEDB88320u ^ (v >> 1) : v >> 1;
      table[i] = v;
    }
    init = true;
  }
  c = ~c;
  for (int64_t i = 0; i < n; ++i) c = table[(c ^ d[i]) & 255] ^ (c >> 8);
  return ~c;
}

struct Header {
  int W = 0, H = 0, ctype = 0, npal = 0;
  int64_t idat_bytes = 0;
  uint8_t pal[768] = {};
};

bool is_letter(uint8_t c) { return (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'); }

// The files the device decodes (oracle/png_ref.py `parse` states the same rules).  Conservative by design: a file
// Pillow would decode but this refuses only goes to Pillow.  Pillow checks the CRC of every chunk before the first
// IDAT (not of IDAT or later chunks), so those are checked here; the chunks it interprets before IDAT are accepted
// only in the forms its handlers take without raising or warning, and the chunks it interprets after the image data
// are avoided by requiring IEND right after the IDAT run.
bool parse(const uint8_t* d, int64_t n, Header* h) {
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  if (n < 8 || n > kMaxBytes + (1 << 20) || std::memcmp(d, sig, 8) != 0) return false;
  int64_t pos = 8;
  bool ihdr = false, plte = false, trns = false, idat_done = false;
  int64_t text = 0;
  int idat_runs = 0;
  bool in_idat = false;
  while (true) {
    if (pos + 12 > n) return false;
    const uint32_t len = be32(d + pos);
    const uint8_t* t = d + pos + 4;
    if (len > 0x7fffffffu || pos + 12 + static_cast<int64_t>(len) > n) return false;
    for (int i = 0; i < 4; ++i)
      if (!is_letter(t[i])) return false;
    const uint8_t* c = d + pos + 8;
    auto is = [&](const char* name) { return std::memcmp(t, name, 4) == 0; };
    const bool idat = is("IDAT");
    if (!ihdr) {
      if (!is("IHDR") || len != 13) return false;
      const uint32_t W = be32(c), H = be32(c + 4);
      if (W < 1 || H < 1 || W > 0x7fffffffu || H > 0x7fffffffu) return false;
      if (c[8] != 8 || !(c[9] == 0 || c[9] == 2 || c[9] == 3 || c[9] == 4 || c[9] == 6)) return false;
      if (c[10] != 0 || c[11] != 0 || c[12] != 0) return false;
      h->W = static_cast<int>(W);
      h->H = static_cast<int>(H);
      h->ctype = c[9];
      ihdr = true;
    } else if (idat) {
      if (idat_done) return false;
      if (h->ctype == 3 && !plte) return false;
      if (!in_idat) ++idat_runs;
      in_idat = true;
      h->idat_bytes += len;
    } else if (in_idat) {
      // the chunk after the IDAT run: only IEND (Pillow's load_end interprets any other)
      return is("IEND") && idat_runs == 1;
    } else {
      if (is("PLTE")) {
        if (plte || len % 3 || len < 3 || len > 768 || h->ctype == 0 || h->ctype == 4) return false;
        plte = true;
        h->npal = static_cast<int>(len / 3);
        std::memcpy(h->pal, c, len);
      } else if (is("tRNS")) {
        if (trns) return false;
        trns = true;
        if (h->ctype == 0) {
          if (len != 2) return false;
        } else if (h->ctype == 2) {
          if (len != 6) return false;
        } else if (h->ctype == 3) {
          // one 0x00 among 0xff (Pillow's "simple" form; any other makes convert("RGB") warn)
          if (!plte || len < 1 || static_cast<int>(len) > h->npal) return false;
          int zeros = 0;
          for (uint32_t i = 0; i < len; ++i) {
            if (c[i] == 0) ++zeros;
            else if (c[i] != 0xff) return false;
          }
          if (zeros != 1) return false;
        } else {
          return false;
        }
      } else if (is("gAMA")) {
        if (len != 4) return false;
      } else if (is("cHRM")) {
        if (len != 32) return false;
      } else if (is("sRGB")) {
        if (len != 1) return false;
      } else if (is("pHYs")) {
        if (len != 9) return false;
      } else if (is("tEXt")) {
        text += len;
        if (text > (1 << 20)) return false;
      } else if (is("IHDR") || is("IEND") || is("iCCP") || is("zTXt") || is("iTXt") || is("eXIf") || is("acTL") ||
                 is("fcTL") || is("fdAT")) {
        return false;
      }
      // any other chunk Pillow reads without interpreting
    }
    if (!idat && crc32(c, len, crc32(t, 4)) != be32(c + len)) return false;
    pos += 12 + len;
  }
}

int channels(int ctype) { return ctype == 0 ? 1 : ctype == 2 ? 3 : ctype == 3 ? 1 : ctype == 4 ? 2 : 4; }

struct Stream {
  const uint8_t* src;   // device
  int64_t nbytes, expect;
  uint8_t* out_inf;     // caller's inflated buffer, or nullptr
  uint8_t* out;         // RGB output, or nullptr
  int64_t pitch;
  int W, H, ctype;
  const uint8_t* pal;
};

// The shared body of both entries: the inflated bytes into the caller's buffers (inflate), or the RGB photos.
int run(const std::vector<Stream>& ss, int32_t* status, int32_t* counts, void* stream) {
  const int B = static_cast<int>(ss.size());
  std::vector<PPhoto> ph(B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallScratch ws(st);
  const size_t r_ph = ws.region(sizeof(PPhoto) * B, true), r_cs = ws.region(4ll * (B + 1), true);
  const size_t r_st = ws.region(sizeof(PState) * B);
  std::vector<size_t> r_words(B), r_bm(B), r_cand(B), r_chain(B), r_sym(B), r_inf(B);
  int* cand_start = ws.host<int>(r_cs);
  int64_t words = 0, ncand = 0;
  for (int b = 0; b < B; ++b) {
    const Stream& s = ss[b];
    PPhoto& P = ph[b];
    std::memset(&P, 0, sizeof(P));
    P.nbytes = s.nbytes;
    P.expect = s.expect;
    P.W = s.W;
    P.H = s.H;
    P.ctype = s.ctype;
    P.bpp = s.out ? channels(s.ctype) : 1;
    P.out = s.out;
    P.pitch = s.pitch;
    P.ncand_cap = static_cast<int>(cand_cap(s.nbytes));
    P.nchain_cap = static_cast<int>(chain_cap(s.expect));
    if (s.pal) std::memcpy(P.pal, s.pal, 768);
    P.word0 = words;
    const int64_t nw = (8 * s.nbytes + 31) / 32;
    words += nw;
    cand_start[b] = static_cast<int>(ncand);
    ncand += P.ncand_cap;
    r_words[b] = ws.region(s.nbytes + kSlack);
    r_bm[b] = ws.region(4 * nw);
    r_cand[b] = ws.region(8ll * P.ncand_cap);
    r_chain[b] = ws.region(16ll * P.nchain_cap);
    r_sym[b] = ws.region(4 * s.expect);
    r_inf[b] = s.out_inf ? 0 : ws.region(s.expect);
  }
  cand_start[B] = static_cast<int>(ncand);
  MHMR_REQUIRE(ncand < (1ll << 31) && words * 32 < (1ll << 62), "png: batch too large for one call");
  const size_t r_meas = ws.region(sizeof(Meas) * ncand);
  TRY(ws.allocate());
  for (int b = 0; b < B; ++b) {
    PPhoto& P = ph[b];
    P.words = ws.dev<const uint32_t>(r_words[b]);
    P.bitmap = ws.dev<uint32_t>(r_bm[b]);
    P.cand = ws.dev<int64_t>(r_cand[b]);
    P.chain = ws.dev<int64_t>(r_chain[b]);
    P.sym = ws.dev<uint32_t>(r_sym[b]);
    P.inf = ss[b].out_inf ? ss[b].out_inf : ws.dev<uint8_t>(r_inf[b]);
  }
  std::memcpy(ws.host<PPhoto>(r_ph), ph.data(), sizeof(PPhoto) * B);
  const PPhoto* dph = ws.dev<const PPhoto>(r_ph);
  PState* dst = ws.dev<PState>(r_st);
  int* dcs = ws.dev<int>(r_cs);
  Meas* dmeas = ws.dev<Meas>(r_meas);
  TRY(ws.upload());
  MHMR_CUDA_CHECK(cudaMemsetAsync(status, 0, 4ll * B, st));
  for (int b = 0; b < B; ++b) {
    uint8_t* copy = ws.dev<uint8_t>(r_words[b]);
    MHMR_CUDA_CHECK(cudaMemsetAsync(copy, 0, align256(ss[b].nbytes + kSlack), st));
    if (ss[b].nbytes) MHMR_CUDA_CHECK(cudaMemcpyAsync(copy, ss[b].src, ss[b].nbytes, cudaMemcpyDeviceToDevice, st));
  }
  if (words > 0) {
    search_kernel<<<static_cast<unsigned>((words * 32 + 255) / 256), 256, 0, st>>>(dph, B, words);
    MHMR_CUDA_CHECK(cudaGetLastError());
  }
  compact_kernel<<<B, 1024, 0, st>>>(dph, dst);
  MHMR_CUDA_CHECK(cudaGetLastError());
  measure_kernel<<<static_cast<unsigned>((ncand + 127) / 128), 128, 0, st>>>(dph, dst, dcs, B,
                                                                               static_cast<int>(ncand), dmeas);
  MHMR_CUDA_CHECK(cudaGetLastError());
  chain_kernel<<<B, 32, 0, st>>>(dph, dst, dcs, dmeas, status);
  MHMR_CUDA_CHECK(cudaGetLastError());
  emit_kernel<<<dim3(8, B), 64, 0, st>>>(dph, dst, status);
  MHMR_CUDA_CHECK(cudaGetLastError());
  resolve_kernel<<<B, 1024, 0, st>>>(dph, dst, status);
  MHMR_CUDA_CHECK(cudaGetLastError());
  unfilter_kernel<<<B, kUnfilterWarps * 32, 0, st>>>(dph, status);
  MHMR_CUDA_CHECK(cudaGetLastError());
  if (counts) {
    for (int b = 0; b < B; ++b) {
      // chain blocks, candidates, slow-path blocks, inflated bytes (low 32 bits)
      const PState* s = dst + b;
      MHMR_CUDA_CHECK(cudaMemcpyAsync(counts + 4 * b, &s->nchain, 4, cudaMemcpyDeviceToDevice, st));
      MHMR_CUDA_CHECK(cudaMemcpyAsync(counts + 4 * b + 1, &s->ncand, 4, cudaMemcpyDeviceToDevice, st));
      MHMR_CUDA_CHECK(cudaMemcpyAsync(counts + 4 * b + 2, &s->nslow, 4, cudaMemcpyDeviceToDevice, st));
      MHMR_CUDA_CHECK(cudaMemcpyAsync(counts + 4 * b + 3, &s->total, 4, cudaMemcpyDeviceToDevice, st));
    }
  }
  return ws.release();
}

}  // namespace

extern "C" {

int mhmr_png_info(const uint8_t* data, int64_t nbytes, int* info) {
  MHMR_REQUIRE(data != nullptr && info != nullptr && nbytes >= 0, "null argument");
  Header h;
  const bool ok = parse(data, nbytes, &h);
  info[0] = ok ? h.W : 0;
  info[1] = ok ? h.H : 0;
  info[2] = ok ? h.ctype : 0;
  info[3] = ok ? 1 : 0;
  return MHMR_OK;
}

int mhmr_op_png_decode(const int64_t* photos, int B, int32_t* status, void* stream) {
  MHMR_REQUIRE(photos != nullptr && status != nullptr, "null argument");
  MHMR_REQUIRE(B >= 1 && B <= 65535, "png: 1 <= B <= 65535 photos");
  std::vector<Header> hdr(B);
  std::vector<Stream> ss(B);
  for (int b = 0; b < B; ++b) {
    const int64_t* d = photos + 8 * b;
    MHMR_REQUIRE(d[0] != 0 && d[1] >= 8, "png: null photo bytes");
    Header& h = hdr[b];
    MHMR_REQUIRE(parse(reinterpret_cast<const uint8_t*>(d[0]), d[1], &h),
                 "png: a photo is not one the device decodes (mhmr_png_info says which are)");
    MHMR_REQUIRE(d[3] == h.idat_bytes, "png: stream length differs from the file's IDAT payloads");
    MHMR_REQUIRE(d[2] != 0 || d[3] == 0, "png: null stream");
    MHMR_REQUIRE(d[6] == h.H && d[7] == h.W, "png: output size differs from the header's");
    MHMR_REQUIRE(d[4] != 0 && d[5] >= 3ll * h.W, "png: null output or pitch below 3 W");
    const int64_t expect = static_cast<int64_t>(h.H) * (1 + static_cast<int64_t>(h.W) * channels(h.ctype));
    MHMR_REQUIRE(expect <= kMaxInflated && d[3] <= kMaxBytes, "png: photo too large for the device decoder");
    ss[b] = {reinterpret_cast<const uint8_t*>(d[2]), d[3], expect, nullptr, reinterpret_cast<uint8_t*>(d[4]), d[5],
             h.W, h.H, h.ctype, h.pal};
  }
  return run(ss, status, nullptr, stream);
}

int mhmr_op_png_inflate(const int64_t* streams, int B, int32_t* status, int32_t* counts, void* stream) {
  MHMR_REQUIRE(streams != nullptr && status != nullptr, "null argument");
  MHMR_REQUIRE(B >= 1 && B <= 65535, "png: 1 <= B <= 65535 streams");
  std::vector<Stream> ss(B);
  for (int b = 0; b < B; ++b) {
    const int64_t* d = streams + 4 * b;
    MHMR_REQUIRE((d[0] != 0 || d[1] == 0) && d[1] >= 0 && d[1] <= kMaxBytes, "png: stream of 0 to 2^28 bytes");
    MHMR_REQUIRE(d[2] != 0 && d[3] >= 1 && d[3] <= kMaxInflated, "png: output of 1 to 2^30 bytes");
    ss[b] = {reinterpret_cast<const uint8_t*>(d[0]), d[1], d[3], reinterpret_cast<uint8_t*>(d[2]), nullptr, 0,
             0, 0, 0, nullptr};
  }
  return run(ss, status, counts, stream);
}

}  // extern "C"
