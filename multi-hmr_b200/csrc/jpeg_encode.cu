// JPEG encoding on the device, byte for byte as Pillow's `Image.fromarray(img).save(f, "JPEG", quality=q,
// subsampling=s)` writes RGB and L images (libjpeg-turbo's baseline path: islow fDCT, the Annex K Huffman tables; the
// arithmetic is restated in oracle/jpeg_encode_ref.py).  The host builds each photo's header (SOI to SOS), its
// quantisation tables and the scan layout; the device runs, for the whole batch:
//   blocks   one thread per MCU block slot of the scan: colour conversion, edge replication, downsampling, the fDCT
//            and quantisation fused, the block's zig-zag coefficients written out with the bit length of its AC codes.
//            A dummy block (an MCU block past its component's blocks) takes the block its DC is copied from, and
//            keeps only that DC.
//   bits     exclusive scan of the block lengths, per photo, in two levels (1024-block tiles, then one CTA over the
//            tile totals).  A block's DC difference depends on the block before it in its component, which another
//            CTA may own, so its bits are added where the scan reads the lengths.
//   pack     each block emits its codes at its bit offset into the photo's zeroed word buffer: MSB-first 32-bit words,
//            atomicOr (exact, OR commutes) since neighbouring blocks share their first and last words.
//   stuff    the entropy-coded bytes, the last one padded with 1-bits, with 0x00 after every 0xFF: a count of the 0xFF
//            bytes per 4 KB tile, a scan of those counts, a scatter; then the header and EOI around them.
// Outputs have the capacity the caller gives.  A file longer than its capacity is not written at all (not even in
// part); its status is 1 and its size is the size it needs, so a caller can allocate that and encode again.  The
// worst case is `mhmr_op_jpeg_encode`'s bound (include/mhmr.h), which never overflows.
#include "common.cuh"

#include <algorithm>
#include <utility>
#include <vector>

using namespace mhmr;

namespace {

constexpr int kBlockThreads = 128;
constexpr int kTile = 1024;          // blocks per bit-scan tile: 256 threads x 4 consecutive blocks
constexpr int kByteTile = 4096;      // bytes per stuffing tile: 256 threads x 16 bytes
constexpr int kMaxBlockBits = 1660;  // DC: 11-bit code + 11 bits; 63 AC: 16-bit code + 10 bits each

struct EncPhoto {
  const uint8_t* src;
  int64_t pitch;
  int H, W, gray;
  int hs, vs;             // luma sampling of the scan (1, 1 for gray: a non-interleaved scan)
  int mcux, bpm;          // MCUs per row (blocks per row for gray), blocks per MCU
  int wib[3], hib[3];     // each component's real blocks wide / high
  int qt;                 // offset of the photo's luma then chroma table (int32 [2][64] natural order)
  int64_t slot0, nslots;  // first global block slot, block slots of the scan
  int64_t tile0;          // first global bit-scan tile; the photo has ceil(nslots / kTile)
  int64_t btile0, nbtiles;  // first global byte tile, byte tiles of the worst case
  uint32_t* words;        // the photo's bit buffer (worst case, zeroed)
  const uint8_t* hdr;
  int hdr_len;
  uint8_t* out;
  int64_t cap;
};

struct Huff {
  uint32_t dc[2][12];   // (length << 16) | code
  uint32_t ac[2][256];
};

// T.81 Annex K.1 (natural order) and K.3.
constexpr int kBasic[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
     14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
     47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
constexpr uint8_t kDcBits[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                    {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
constexpr uint8_t kAcBits[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125},
                                    {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119}};
constexpr uint8_t kAcVals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
     0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
     0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
     0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
     0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
     0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
     0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
     0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
     0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
     0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
     0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
     0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
     0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
     0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
     0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};
// Natural index of zig-zag position k (the walk along the anti-diagonals); folds to a constant for a constant k.
__host__ __device__ constexpr int zigzag(int k) {
  int x = 0, y = 0;
  for (int n = 0; n < k; ++n) {
    if ((x + y) % 2 == 0) {
      if (x == 7) ++y; else if (y == 0) ++x; else { ++x; --y; }
    } else {
      if (y == 7) ++x; else if (x == 0) ++y; else { --x; ++y; }
    }
  }
  return y * 8 + x;
}
template <int K>
struct Zigzag {
  static constexpr int n = zigzag(K);
};

__device__ __forceinline__ int quantise(int v, int q) {  // sign(v) ((|v| + 4 q) / 8 q)
  const int a = ((v < 0 ? -v : v) + 4 * q) / (8 * q);
  return v < 0 ? -a : a;
}

// z[k] = quantised fDCT output at zig-zag position k (natural-order d and q), unrolled at compile time.
template <int... K>
__device__ __forceinline__ void quantise_zigzag(const int* d, const int32_t* __restrict__ q, int* z,
                                                std::integer_sequence<int, K...>) {
  ((z[K] = quantise(d[Zigzag<K>::n], __ldg(q + Zigzag<K>::n))), ...);
}

// libjpeg's 16-bit fixed point, FIX(x) = (int)(x * 65536 + 0.5)
constexpr int fix16(double x) { return static_cast<int>(x * 65536.0 + 0.5); }
constexpr int kYr = fix16(0.299), kYg = fix16(0.587), kYb = fix16(0.114), kCbR = fix16(0.16874),
              kCbG = fix16(0.33126), kHalfC = fix16(0.5), kCrG = fix16(0.41869), kCrB = fix16(0.08131);

__device__ __forceinline__ int ycc(int c, int r, int g, int b) {
  constexpr int kOffset = (128 << 16) + (1 << 15) - 1;
  if (c == 0) return (kYr * r + kYg * g + kYb * b + (1 << 15)) >> 16;
  if (c == 1) return (-kCbR * r - kCbG * g + kHalfC * b + kOffset) >> 16;
  return (kHalfC * r - kCrG * g - kCrB * b + kOffset) >> 16;
}

__device__ __forceinline__ int pixel(const EncPhoto& P, int c, int x, int y) {
  const uint8_t* s = P.src + static_cast<int64_t>(y) * P.pitch;
  if (P.gray) return __ldg(s + x);
  s += 3ll * x;
  return ycc(c, __ldg(s), __ldg(s + 1), __ldg(s + 2));
}

// Sample (sx, sy) of component c's padded plane: edges replicated, chroma downsampled h2v1 / h2v2 from the
// full-resolution plane replicated rightwards (and to an even row count for h2v2); chroma rows past the downsampled
// plane repeat its last row.
__device__ __forceinline__ int sample(const EncPhoto& P, int c, int sx, int sy) {
  if (c == 0 || P.hs == 1) return pixel(P, c, min(sx, P.W - 1), min(sy, P.H - 1));
  const int x0 = min(2 * sx, P.W - 1), x1 = min(2 * sx + 1, P.W - 1);
  if (P.vs == 1) {
    const int y = min(sy, P.H - 1);
    return (pixel(P, c, x0, y) + pixel(P, c, x1, y) + (sx & 1)) >> 1;
  }
  const int cy = min(sy, (P.H + 1) / 2 - 1);
  const int y0 = min(2 * cy, P.H - 1), y1 = min(2 * cy + 1, P.H - 1);
  return (pixel(P, c, x0, y0) + pixel(P, c, x1, y0) + pixel(P, c, x0, y1) + pixel(P, c, x1, y1) + 1 + (sx & 1)) >> 2;
}

template <class T>
__device__ __forceinline__ T descale(T x, int n) {
  return (x + (T(1) << (n - 1))) >> n;
}

// jfdctint.c, one pass over 8 elements `stride` apart: pass 1 (rows) scales up by PASS1_BITS, pass 2 (columns)
// removes it.  T is int for pass 1 and int64 for pass 2, whose products can pass 2^31.
template <class T, bool kFirst>
__device__ __forceinline__ void fdct_1d(int* d, int stride) {
  constexpr int kShift = kFirst ? 13 - 2 : 13 + 2;
  const T t0 = T(d[0]) + d[7 * stride], t7 = T(d[0]) - d[7 * stride];
  const T t1 = T(d[stride]) + d[6 * stride], t6 = T(d[stride]) - d[6 * stride];
  const T t2 = T(d[2 * stride]) + d[5 * stride], t5 = T(d[2 * stride]) - d[5 * stride];
  const T t3 = T(d[3 * stride]) + d[4 * stride], t4 = T(d[3 * stride]) - d[4 * stride];
  const T t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  if (kFirst) {
    d[0] = static_cast<int>((t10 + t11) << 2);
    d[4 * stride] = static_cast<int>((t10 - t11) << 2);
  } else {
    d[0] = static_cast<int>(descale<T>(t10 + t11, 2));
    d[4 * stride] = static_cast<int>(descale<T>(t10 - t11, 2));
  }
  T z1 = (t12 + t13) * 4433;
  d[2 * stride] = static_cast<int>(descale<T>(z1 + t13 * 6270, kShift));
  d[6 * stride] = static_cast<int>(descale<T>(z1 - t12 * 15137, kShift));
  z1 = t4 + t7;
  T z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const T z5 = (z3 + z4) * 9633;
  const T a4 = t4 * 2446, a5 = t5 * 16819, a6 = t6 * 25172, a7 = t7 * 12299;
  z1 = -z1 * 7373;
  z2 = -z2 * 20995;
  z3 = -z3 * 16069 + z5;
  z4 = -z4 * 3196 + z5;
  d[7 * stride] = static_cast<int>(descale<T>(a4 + z1 + z3, kShift));
  d[5 * stride] = static_cast<int>(descale<T>(a5 + z2 + z4, kShift));
  d[3 * stride] = static_cast<int>(descale<T>(a6 + z2 + z3, kShift));
  d[1 * stride] = static_cast<int>(descale<T>(a7 + z1 + z4, kShift));
}

__device__ __forceinline__ int category(int v) { return 32 - __clz(v < 0 ? -v : v); }

// Component, block column and row of a scan slot, and whether it is a dummy.
struct Slot {
  int c, bx, by;
  bool dummy;
};

__device__ __forceinline__ Slot slot_of(const EncPhoto& P, int64_t i) {
  Slot s;
  if (P.gray) {
    s.c = 0;
    s.bx = static_cast<int>(i % P.wib[0]);
    s.by = static_cast<int>(i / P.wib[0]);
    s.dummy = false;
    return s;
  }
  const int64_t m = i / P.bpm;
  const int r = static_cast<int>(i - m * P.bpm), n0 = P.hs * P.vs;
  const int mx = static_cast<int>(m % P.mcux), my = static_cast<int>(m / P.mcux);
  if (r < n0) {
    s.c = 0;
    s.bx = mx * P.hs + r % P.hs;
    s.by = my * P.vs + r / P.hs;
  } else {
    s.c = r - n0 + 1;
    s.bx = mx;
    s.by = my;
  }
  s.dummy = s.bx >= P.wib[s.c] || s.by >= P.hib[s.c];
  if (s.dummy) {  // compress_data: the DC of the last real block before it in the MCU (its row's, or the last row's)
    const int h = s.c == 0 ? P.hs : 1;
    s.bx = min(mx * h + h - 1, P.wib[s.c] - 1);
    s.by = min(s.by, P.hib[s.c] - 1);
  }
  return s;
}

// Scan slot of the block before slot i in its component (-1: none, DC predicted from 0).
__device__ __forceinline__ int64_t pred_of(const EncPhoto& P, int64_t i) {
  if (P.gray) return i - 1;
  const int64_t m = i / P.bpm;
  const int r = static_cast<int>(i - m * P.bpm), n0 = P.hs * P.vs;
  if (r > 0 && r < n0) return i - 1;
  if (m == 0) return -1;
  return i - P.bpm + (r == 0 ? n0 - 1 : 0);
}

__global__ void __launch_bounds__(kBlockThreads) enc_blocks_kernel(const EncPhoto* __restrict__ photos,
                                                                   const int32_t* __restrict__ qtab,
                                                                   const Huff* __restrict__ huff, int16_t* coefs,
                                                                   uint32_t* acbits) {
  const EncPhoto& P = photos[blockIdx.y];
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kBlockThreads + threadIdx.x;
  if (i >= P.nslots) return;
  const Slot s = slot_of(P, i);
  int d[64];
#pragma unroll
  for (int y = 0; y < 8; ++y)
#pragma unroll
    for (int x = 0; x < 8; ++x) d[y * 8 + x] = sample(P, s.c, s.bx * 8 + x, s.by * 8 + y) - 128;
#pragma unroll
  for (int y = 0; y < 8; ++y) fdct_1d<int, true>(d + y * 8, 1);
#pragma unroll
  for (int x = 0; x < 8; ++x) fdct_1d<long long, false>(d + x, 8);
  const int t = s.c == 0 ? 0 : 1;
  const int32_t* q = qtab + P.qt + 64 * t;
  int z[64];
  quantise_zigzag(d, q, z, std::make_integer_sequence<int, 64>());
  if (s.dummy) {
#pragma unroll
    for (int k = 1; k < 64; ++k) z[k] = 0;
  }
  const int64_t g = P.slot0 + i;
  int4* dst = reinterpret_cast<int4*>(coefs + g * 64);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int4 w;
    w.x = (z[8 * k] & 0xFFFF) | (z[8 * k + 1] << 16);
    w.y = (z[8 * k + 2] & 0xFFFF) | (z[8 * k + 3] << 16);
    w.z = (z[8 * k + 4] & 0xFFFF) | (z[8 * k + 5] << 16);
    w.w = (z[8 * k + 6] & 0xFFFF) | (z[8 * k + 7] << 16);
    dst[k] = w;
  }
  const uint32_t* ac = huff->ac[t];
  uint32_t bits = 0;
  int run = 0;
#pragma unroll
  for (int k = 1; k < 64; ++k) {
    if (z[k] == 0) {
      ++run;
    } else {
      for (; run > 15; run -= 16) bits += __ldg(ac + 0xF0) >> 16;
      const int cat = category(z[k]);
      bits += (__ldg(ac + run * 16 + cat) >> 16) + cat;
      run = 0;
    }
  }
  if (run) bits += __ldg(ac) >> 16;
  acbits[g] = bits;
}

__device__ __forceinline__ int dc_diff(const EncPhoto& P, const int16_t* __restrict__ coefs, int64_t i) {
  const int64_t p = pred_of(P, i);
  return coefs[(P.slot0 + i) * 64] - (p < 0 ? 0 : coefs[(P.slot0 + p) * 64]);
}

__device__ __forceinline__ uint32_t block_bits(const EncPhoto& P, const int16_t* __restrict__ coefs,
                                               const uint32_t* __restrict__ acbits, const Huff* __restrict__ huff,
                                               int64_t i) {
  const int64_t g = P.slot0 + i;
  const int t = slot_of(P, i).c == 0 ? 0 : 1;
  const int cat = category(dc_diff(P, coefs, i));
  return acbits[g] + (__ldg(huff->dc[t] + cat) >> 16) + cat;
}

template <class T>
__device__ T block_excl_scan_256(T v, T* total) {
  __shared__ T warp_sums[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  T base = 0, all = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    const T s = warp_sums[w];
    if (w < warp) base += s;
    all += s;
  }
  __syncthreads();
  *total = all;
  return base + x - v;
}

// Bit totals of each photo's 1024-block tiles.
__global__ void __launch_bounds__(256) bits_tile_kernel(const EncPhoto* __restrict__ photos,
                                                        const int16_t* __restrict__ coefs,
                                                        const uint32_t* __restrict__ acbits,
                                                        const Huff* __restrict__ huff, uint64_t* tile_bits) {
  const EncPhoto& P = photos[blockIdx.y];
  const int64_t t = blockIdx.x, i0 = t * kTile + 4 * threadIdx.x;
  if (t * kTile >= P.nslots) return;
  uint32_t v = 0;
  for (int k = 0; k < 4; ++k)
    if (i0 + k < P.nslots) v += block_bits(P, coefs, acbits, huff, i0 + k);
  uint32_t total;
  block_excl_scan_256<uint32_t>(v, &total);
  if (threadIdx.x == 0) tile_bits[P.tile0 + t] = total;
}

// In place exclusive scan of a[0, n); a[n] receives the total.  One CTA.
__global__ void __launch_bounds__(1024) scan_kernel(uint64_t* a, int64_t n) {
  __shared__ uint64_t warp_sums[32];
  __shared__ uint64_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t base = 0; base < n; base += 1024) {
    const int64_t i = base + threadIdx.x;
    const uint64_t v = i < n ? a[i] : 0;
    uint64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    uint64_t before = 0, all = 0;
    for (int w = 0; w < 32; ++w) {
      before += w < warp ? warp_sums[w] : 0;
      all += warp_sums[w];
    }
    const uint64_t c = carry;
    if (i < n) a[i] = c + before + x - v;
    __syncthreads();
    if (threadIdx.x == 0) carry = c + all;
    __syncthreads();
  }
  if (threadIdx.x == 0) a[n] = carry;
}

struct BitWriter {
  uint32_t* w;
  uint64_t acc;
  int n;
  __device__ __forceinline__ void put(uint32_t code, int len) {
    acc = (acc << len) | code;
    n += len;
    if (n >= 32) {
      n -= 32;
      atomicOr(w++, static_cast<uint32_t>(acc >> n));
      acc &= (1ull << n) - 1;
    }
  }
  __device__ __forceinline__ void flush() {
    if (n > 0) atomicOr(w, static_cast<uint32_t>(acc << (32 - n)));
  }
};

__device__ __forceinline__ void put_code(BitWriter& bw, uint32_t e) { bw.put(e & 0xFFFF, static_cast<int>(e >> 16)); }

// Each tile's own scan, then every block's codes at its offset.
__global__ void __launch_bounds__(256) pack_kernel(const EncPhoto* __restrict__ photos,
                                                   const int16_t* __restrict__ coefs,
                                                   const uint32_t* __restrict__ acbits,
                                                   const Huff* __restrict__ huff,
                                                   const uint64_t* __restrict__ tile_bits) {
  const EncPhoto& P = photos[blockIdx.y];
  const int64_t t = blockIdx.x, i0 = t * kTile + 4 * threadIdx.x;
  if (t * kTile >= P.nslots) return;
  uint32_t v = 0;
  for (int k = 0; k < 4; ++k)
    if (i0 + k < P.nslots) v += block_bits(P, coefs, acbits, huff, i0 + k);
  uint32_t total;
  const uint32_t excl = block_excl_scan_256<uint32_t>(v, &total);
  const uint64_t pos = tile_bits[P.tile0 + t] - tile_bits[P.tile0] + excl;
  BitWriter bw{P.words + (pos >> 5), 0, static_cast<int>(pos & 31)};
  for (int k = 0; k < 4 && i0 + k < P.nslots; ++k) {
    const int64_t i = i0 + k;
    const int tb = slot_of(P, i).c == 0 ? 0 : 1;
    const int diff = dc_diff(P, coefs, i);
    int cat = category(diff);
    put_code(bw, __ldg(huff->dc[tb] + cat));
    if (cat) bw.put(static_cast<uint32_t>(diff < 0 ? diff + (1 << cat) - 1 : diff) & ((1u << cat) - 1), cat);
    const uint32_t* ac = huff->ac[tb];
    const int4* src = reinterpret_cast<const int4*>(coefs + (P.slot0 + i) * 64);
    int run = 0;
    for (int q = 0; q < 8; ++q) {
      const int4 w4 = src[q];
      const int w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
      for (int h = 0; h < 8; ++h) {
        if (q == 0 && h == 0) continue;
        const int z = static_cast<int16_t>((w[h >> 1] >> (16 * (h & 1))) & 0xFFFF);
        if (z == 0) {
          ++run;
          continue;
        }
        for (; run > 15; run -= 16) put_code(bw, __ldg(ac + 0xF0));
        cat = category(z);
        put_code(bw, __ldg(ac + run * 16 + cat));
        bw.put(static_cast<uint32_t>(z < 0 ? z + (1 << cat) - 1 : z) & ((1u << cat) - 1), cat);
        run = 0;
      }
    }
    if (run) put_code(bw, __ldg(ac));
  }
  bw.flush();
}

__device__ __forceinline__ uint64_t photo_bits(const EncPhoto& P, const uint64_t* __restrict__ tile_bits) {
  return tile_bits[P.tile0 + (P.nslots + kTile - 1) / kTile] - tile_bits[P.tile0];
}

// Entropy-coded byte j of a photo with `bits` bits: the last one padded with 1-bits.
__device__ __forceinline__ uint32_t ecs_byte(const EncPhoto& P, uint64_t bits, uint64_t j) {
  uint32_t b = (P.words[j >> 2] >> (24 - 8 * (j & 3))) & 0xFF;
  if (j == (bits - 1) / 8 && (bits & 7)) b |= 0xFFu >> (bits & 7);
  return b;
}

__global__ void __launch_bounds__(256) ff_count_kernel(const EncPhoto* __restrict__ photos,
                                                       const uint64_t* __restrict__ tile_bits, uint64_t* tile_ff) {
  const EncPhoto& P = photos[blockIdx.y];
  const int64_t t = blockIdx.x;
  if (t >= P.nbtiles) return;
  const uint64_t bits = photo_bits(P, tile_bits), nb = (bits + 7) / 8;
  const uint64_t j0 = static_cast<uint64_t>(t) * kByteTile + 16 * threadIdx.x;
  uint32_t v = 0;
  if (static_cast<uint64_t>(t) * kByteTile < nb)
    for (int k = 0; k < 16; ++k) v += (j0 + k < nb && ecs_byte(P, bits, j0 + k) == 0xFF) ? 1 : 0;
  uint32_t total;
  block_excl_scan_256<uint32_t>(v, &total);
  if (threadIdx.x == 0) tile_ff[P.btile0 + t] = total;
}

__device__ __forceinline__ uint64_t file_size(const EncPhoto& P, uint64_t bits, const uint64_t* __restrict__ tile_ff) {
  const uint64_t ff = tile_ff[P.btile0 + P.nbtiles] - tile_ff[P.btile0];
  return P.hdr_len + (bits + 7) / 8 + ff + 2;
}

__global__ void __launch_bounds__(256) stuff_kernel(const EncPhoto* __restrict__ photos,
                                                    const uint64_t* __restrict__ tile_bits,
                                                    const uint64_t* __restrict__ tile_ff) {
  const EncPhoto& P = photos[blockIdx.y];
  const int64_t t = blockIdx.x;
  if (t >= P.nbtiles) return;
  const uint64_t bits = photo_bits(P, tile_bits), nb = (bits + 7) / 8;
  if (static_cast<uint64_t>(t) * kByteTile >= nb || file_size(P, bits, tile_ff) > static_cast<uint64_t>(P.cap)) return;
  const uint64_t j0 = static_cast<uint64_t>(t) * kByteTile + 16 * threadIdx.x;
  uint32_t b[16], v = 0;
  for (int k = 0; k < 16; ++k) {
    b[k] = j0 + k < nb ? ecs_byte(P, bits, j0 + k) : 0;
    v += (j0 + k < nb && b[k] == 0xFF) ? 1 : 0;
  }
  uint32_t total;
  const uint32_t excl = block_excl_scan_256<uint32_t>(v, &total);
  uint64_t o = P.hdr_len + j0 + (tile_ff[P.btile0 + t] - tile_ff[P.btile0]) + excl;
  for (int k = 0; k < 16 && j0 + k < nb; ++k) {
    P.out[o++] = static_cast<uint8_t>(b[k]);
    if (b[k] == 0xFF) P.out[o++] = 0;
  }
}

// Header and EOI around the stuffed bytes, sizes and statuses.
__global__ void __launch_bounds__(256) finish_kernel(const EncPhoto* __restrict__ photos,
                                                     const uint64_t* __restrict__ tile_bits,
                                                     const uint64_t* __restrict__ tile_ff, int64_t* sizes,
                                                     int32_t* status) {
  const EncPhoto& P = photos[blockIdx.x];
  const uint64_t size = file_size(P, photo_bits(P, tile_bits), tile_ff);
  const bool fits = size <= static_cast<uint64_t>(P.cap);
  if (threadIdx.x == 0) {
    sizes[blockIdx.x] = static_cast<int64_t>(size);
    status[blockIdx.x] = fits ? 0 : 1;
  }
  if (!fits) return;
  for (int k = threadIdx.x; k < P.hdr_len; k += blockDim.x) P.out[k] = P.hdr[k];
  if (threadIdx.x == 0) {
    P.out[size - 2] = 0xFF;
    P.out[size - 1] = 0xD9;
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------
void quant_tables(int quality, int32_t* out) {  // jpeg_set_quality, force_baseline: [2][64] natural order
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int t = 0; t < 2; ++t)
    for (int k = 0; k < 64; ++k) out[64 * t + k] = std::min(std::max((kBasic[t][k] * scale + 50) / 100, 1), 255);
}

void huff_codes(const uint8_t* bits, const uint8_t* vals, uint32_t* table) {  // T.81 Annex C
  uint32_t code = 0;
  int k = 0;
  for (int len = 1; len <= 16; ++len, code <<= 1)
    for (int n = 0; n < bits[len - 1]; ++n, ++k, ++code) table[vals[k]] = (static_cast<uint32_t>(len) << 16) | code;
}

void put_segment(std::vector<uint8_t>& h, int marker, const std::vector<uint8_t>& body) {
  const size_t n = body.size() + 2;
  h.insert(h.end(), {0xFF, static_cast<uint8_t>(marker), static_cast<uint8_t>(n >> 8), static_cast<uint8_t>(n)});
  h.insert(h.end(), body.begin(), body.end());
}

// SOI, APP0 JFIF 1.01, DQT, SOF0, DHT, SOS as Pillow writes them; `sof_samp` is the luma sampling byte of SOF0.
std::vector<uint8_t> header(int W, int H, int ncomp, int sof_samp, const int32_t* qt) {
  std::vector<uint8_t> h = {0xFF, 0xD8};
  put_segment(h, 0xE0, {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0});
  const int ntab = ncomp == 1 ? 1 : 2;
  for (int t = 0; t < ntab; ++t) {
    std::vector<uint8_t> b = {static_cast<uint8_t>(t)};
    for (int k = 0; k < 64; ++k) b.push_back(static_cast<uint8_t>(qt[64 * t + zigzag(k)]));
    put_segment(h, 0xDB, b);
  }
  std::vector<uint8_t> sof = {8, static_cast<uint8_t>(H >> 8), static_cast<uint8_t>(H), static_cast<uint8_t>(W >> 8),
                              static_cast<uint8_t>(W), static_cast<uint8_t>(ncomp), 1, static_cast<uint8_t>(sof_samp), 0};
  for (int c = 1; c < ncomp; ++c) sof.insert(sof.end(), {static_cast<uint8_t>(c + 1), 0x11, 1});
  put_segment(h, 0xC0, sof);
  for (int t = 0; t < ntab; ++t) {
    std::vector<uint8_t> dc = {static_cast<uint8_t>(t)}, ac = {static_cast<uint8_t>(0x10 + t)};
    dc.insert(dc.end(), kDcBits[t], kDcBits[t] + 16);
    for (int v = 0; v < 12; ++v) dc.push_back(static_cast<uint8_t>(v));
    ac.insert(ac.end(), kAcBits[t], kAcBits[t] + 16);
    ac.insert(ac.end(), kAcVals[t], kAcVals[t] + 162);
    put_segment(h, 0xC4, dc);
    put_segment(h, 0xC4, ac);
  }
  std::vector<uint8_t> sos = {static_cast<uint8_t>(ncomp)};
  for (int c = 0; c < ncomp; ++c) sos.insert(sos.end(), {static_cast<uint8_t>(c + 1), static_cast<uint8_t>(c ? 0x11 : 0)});
  sos.insert(sos.end(), {0, 63, 0});
  put_segment(h, 0xDA, sos);
  return h;
}

}  // namespace

extern "C" {

int mhmr_op_jpeg_encode(const int64_t* photos, int B, int64_t* sizes, int32_t* status, void* stream) {
  MHMR_REQUIRE(B >= 0 && B <= 65535, "jpeg_encode: 0 <= B <= 65535 photos");
  if (B == 0) return MHMR_OK;
  MHMR_REQUIRE(photos != nullptr && sizes != nullptr && status != nullptr, "null argument");
  std::vector<EncPhoto> ph(B);
  std::vector<int32_t> qt(128 * static_cast<size_t>(B));
  std::vector<std::vector<uint8_t>> hdrs(B);
  int64_t slots = 0, tiles = 0, btiles = 0, words = 0, max_slots = 0, max_btiles = 0;
  std::vector<int64_t> word0(B);
  for (int b = 0; b < B; ++b) {
    const int64_t* d = photos + 9 * b;
    const int64_t H = d[1], W = d[2], pitch = d[3], C = d[4], q = d[5], s = d[6];
    MHMR_REQUIRE(d[0] != 0 && d[7] != 0, "jpeg_encode: null photo or output");
    MHMR_REQUIRE(H >= 1 && W >= 1 && H <= 65535 && W <= 65535, "jpeg_encode: photo sides in [1, 65535]");
    MHMR_REQUIRE(C == 1 || C == 3, "jpeg_encode: 1 (gray) or 3 (RGB) channels");
    MHMR_REQUIRE(pitch >= C * W, "jpeg_encode: row pitch below channels x W bytes");
    MHMR_REQUIRE(q >= 1 && q <= 100, "jpeg_encode: quality in [1, 100]");
    MHMR_REQUIRE(s >= 0 && s <= 2, "jpeg_encode: subsampling 0 (4:4:4), 1 (4:2:2) or 2 (4:2:0)");
    MHMR_REQUIRE(d[8] >= 0, "jpeg_encode: negative capacity");
    EncPhoto& P = ph[b];
    P.src = reinterpret_cast<const uint8_t*>(d[0]);
    P.pitch = pitch;
    P.H = static_cast<int>(H);
    P.W = static_cast<int>(W);
    P.gray = C == 1;
    const int hs = s == 0 ? 1 : 2, vs = s == 2 ? 2 : 1;
    P.hs = P.gray ? 1 : hs;
    P.vs = P.gray ? 1 : vs;
    const int ncomp = P.gray ? 1 : 3;
    for (int c = 0; c < 3; ++c) {
      const int h = c == 0 ? P.hs : 1, v = c == 0 ? P.vs : 1;
      const int cw = static_cast<int>((W * h + P.hs - 1) / P.hs), ch = static_cast<int>((H * v + P.vs - 1) / P.vs);
      P.wib[c] = (cw + 7) / 8;
      P.hib[c] = (ch + 7) / 8;
    }
    P.mcux = P.gray ? P.wib[0] : static_cast<int>((W + 8 * P.hs - 1) / (8 * P.hs));
    const int64_t mcuy = P.gray ? P.hib[0] : (H + 8 * P.vs - 1) / (8 * P.vs);
    P.bpm = P.gray ? 1 : P.hs * P.vs + 2;
    P.nslots = static_cast<int64_t>(P.mcux) * mcuy * P.bpm;
    P.slot0 = slots;
    P.tile0 = tiles;
    const int64_t max_words = (P.nslots * kMaxBlockBits + 31) / 32 + 1;
    P.btile0 = btiles;
    P.nbtiles = (4 * max_words + kByteTile - 1) / kByteTile;
    word0[b] = words;
    slots += P.nslots;
    tiles += (P.nslots + kTile - 1) / kTile;
    btiles += P.nbtiles;
    words += max_words;
    max_slots = std::max(max_slots, P.nslots);
    max_btiles = std::max(max_btiles, P.nbtiles);
    P.qt = 128 * b;
    quant_tables(static_cast<int>(q), qt.data() + 128 * b);
    // the SOF0 sampling byte is the one asked for, also for gray, whose scan is non-interleaved all the same
    hdrs[b] = header(P.W, P.H, ncomp, 16 * hs + vs, qt.data() + 128 * b);
    P.hdr_len = static_cast<int>(hdrs[b].size());
    P.out = reinterpret_cast<uint8_t*>(d[7]);
    P.cap = d[8];
  }
  MHMR_REQUIRE((max_slots + kBlockThreads - 1) / kBlockThreads < (1ll << 31), "jpeg_encode: photo too large");

  Huff huff{};
  for (int t = 0; t < 2; ++t) {
    uint8_t dcv[12];
    for (int v = 0; v < 12; ++v) dcv[v] = static_cast<uint8_t>(v);
    huff_codes(kDcBits[t], dcv, huff.dc[t]);
    huff_codes(kAcBits[t], kAcVals[t], huff.ac[t]);
  }
  size_t hdr_bytes = 0;
  for (const auto& h : hdrs) hdr_bytes += h.size();

  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallScratch ws(st);
  const size_t r_ph = ws.region(sizeof(EncPhoto) * B, true), r_qt = ws.region(4 * qt.size(), true),
               r_huff = ws.region(sizeof(Huff), true), r_hdr = ws.region(hdr_bytes, true);
  const size_t r_coefs = ws.region(128 * static_cast<size_t>(slots)), r_ac = ws.region(4 * static_cast<size_t>(slots)),
               r_tb = ws.region(8 * static_cast<size_t>(tiles + 1)), r_ff = ws.region(8 * static_cast<size_t>(btiles + 1)),
               r_words = ws.region(4 * static_cast<size_t>(words));
  TRY(ws.allocate());
  uint8_t* hdr_host = ws.host<uint8_t>(r_hdr);
  const uint8_t* hdr_dev = ws.dev<const uint8_t>(r_hdr);
  uint32_t* d_words = ws.dev<uint32_t>(r_words);
  size_t off = 0;
  for (int b = 0; b < B; ++b) {
    std::copy(hdrs[b].begin(), hdrs[b].end(), hdr_host + off);
    ph[b].hdr = hdr_dev + off;
    ph[b].words = d_words + word0[b];
    off += hdrs[b].size();
  }
  std::copy_n(ph.data(), B, ws.host<EncPhoto>(r_ph));
  std::copy_n(qt.data(), qt.size(), ws.host<int32_t>(r_qt));
  *ws.host<Huff>(r_huff) = huff;
  TRY(ws.upload());
  const EncPhoto* d_ph = ws.dev<const EncPhoto>(r_ph);
  const Huff* d_huff = ws.dev<const Huff>(r_huff);
  int16_t* d_coefs = ws.dev<int16_t>(r_coefs);
  uint32_t* d_ac = ws.dev<uint32_t>(r_ac);
  uint64_t* d_tb = ws.dev<uint64_t>(r_tb);
  uint64_t* d_ff = ws.dev<uint64_t>(r_ff);
  MHMR_CUDA_CHECK(cudaMemsetAsync(d_words, 0, 4 * static_cast<size_t>(words), st));
  const int64_t max_tiles = (max_slots + kTile - 1) / kTile;
  enc_blocks_kernel<<<dim3(static_cast<unsigned>((max_slots + kBlockThreads - 1) / kBlockThreads), B), kBlockThreads,
                      0, st>>>(d_ph, ws.dev<const int32_t>(r_qt), d_huff, d_coefs, d_ac);
  MHMR_CUDA_CHECK(cudaGetLastError());
  bits_tile_kernel<<<dim3(static_cast<unsigned>(max_tiles), B), 256, 0, st>>>(d_ph, d_coefs, d_ac, d_huff, d_tb);
  MHMR_CUDA_CHECK(cudaGetLastError());
  scan_kernel<<<1, 1024, 0, st>>>(d_tb, tiles);
  MHMR_CUDA_CHECK(cudaGetLastError());
  pack_kernel<<<dim3(static_cast<unsigned>(max_tiles), B), 256, 0, st>>>(d_ph, d_coefs, d_ac, d_huff, d_tb);
  MHMR_CUDA_CHECK(cudaGetLastError());
  ff_count_kernel<<<dim3(static_cast<unsigned>(max_btiles), B), 256, 0, st>>>(d_ph, d_tb, d_ff);
  MHMR_CUDA_CHECK(cudaGetLastError());
  scan_kernel<<<1, 1024, 0, st>>>(d_ff, btiles);
  MHMR_CUDA_CHECK(cudaGetLastError());
  stuff_kernel<<<dim3(static_cast<unsigned>(max_btiles), B), 256, 0, st>>>(d_ph, d_tb, d_ff);
  MHMR_CUDA_CHECK(cudaGetLastError());
  finish_kernel<<<B, 256, 0, st>>>(d_ph, d_tb, d_ff, sizes, status);
  MHMR_CUDA_CHECK(cudaGetLastError());
  TRY(ws.release());
  return MHMR_OK;
}

}  // extern "C"
