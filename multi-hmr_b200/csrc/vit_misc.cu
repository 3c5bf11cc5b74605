// Memory-bound helpers of the ViT backbone: patch gathering (im2col for the 14x14/14 conv), LayerNorm
// with fp16 / fp32 outputs, cls-token row initialisation, fp32->fp16 weight repacking.
#include <algorithm>

#include "kernels.cuh"

namespace mhmr {

namespace {

// x [B,3,S,S] fp32 -> A [B*N, ldA] fp16, column k = c*196 + py*14 + px (Conv2d weight flattening order,
// dinov2 PatchEmbed.proj reached from reference blocks/dinov2.py:25).  Columns >= 588 are never written
// (they are out of the tensor-map bounds and read as zero by TMA).
__global__ void im2col_patch14_kernel(const float* __restrict__ x, __half* __restrict__ A, int B, int S,
                                      int ldA) {
  const int hw = S / 14;
  const int m = blockIdx.x;  // patch row index b*N + py_*hw + px_
  const int N = hw * hw;
  const int b = m / N, n = m - b * N;
  const int gy = n / hw, gx = n - gy * hw;
  const float* src = x + static_cast<int64_t>(b) * 3 * S * S;
  __half* dst = A + static_cast<int64_t>(m) * ldA;
  for (int k = threadIdx.x; k < 588; k += blockDim.x) {
    const int c = k / 196, r = k - c * 196;
    const int py = r / 14, px = r - py * 14;
    dst[k] = __float2half_rn(src[(static_cast<int64_t>(c) * S + gy * 14 + py) * S + gx * 14 + px]);
  }
}

// Fused image loader (SURVEY.md §8f row 1): uint8 HWC image -> normalised fp16 patch rows of the patch-embed GEMM in
// one pass.  Same values as normalize_u8_kernel followed by im2col_patch14_kernel (the [3][256] table reproduces the
// reference's normalize_rgb bit for bit, the fp16 rounding is the same __float2half_rn), without the fp32 CHW image
// in between: per image 2.4 MB of bytes in and 4.8 MB of fp16 out instead of 9.6 MB written + 9.6 MB re-read.
// One CTA per patch; thread k = c*196 + py*14 + px reads one byte, 588 consecutive fp16 out.
__global__ void __launch_bounds__(192)
im2col_u8_patch14_kernel(const uint8_t* __restrict__ img, const float* __restrict__ lut, __half* __restrict__ A,
                         int S, int ldA) {
  const int hw = S / 14;
  const int m = blockIdx.x;
  const int N = hw * hw;
  const int b = m / N, n = m - b * N;
  const int gy = n / hw, gx = n - gy * hw;
  const uint8_t* src = img + (static_cast<int64_t>(b) * S + gy * 14) * S * 3 + gx * 14 * 3;
  __half* dst = A + static_cast<int64_t>(m) * ldA;
  for (int k = threadIdx.x; k < 588; k += blockDim.x) {
    const int c = k / 196, r = k - c * 196;
    const int py = r / 14, px = r - py * 14;
    const uint8_t v = src[(static_cast<int64_t>(py) * S + px) * 3 + c];
    dst[k] = __float2half_rn(__ldg(lut + c * 256 + v));
  }
}

// uint8 HWC image -> normalised fp32 CHW through a [3][256] table (reference utils/image.py:12-24 `normalize_rgb`:
// ((v / 255) - mean_c) / std_c evaluated in float64 and rounded to fp32 -- the host builds the table with exactly
// those numpy operations, so the device output is bit-identical to the reference's host preprocessing).
// One thread per 4 pixels of a row: 12 contiguous bytes in, three coalesced float4 out.
__global__ void normalize_u8_kernel(const uint8_t* __restrict__ img, const float* __restrict__ lut,
                                    float* __restrict__ out, int H, int W, int64_t n_quads) {
  __shared__ float s_lut[3 * 256];
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) s_lut[i] = lut[i];
  __syncthreads();
  const int wq = W / 4;
  for (int64_t q = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; q < n_quads;
       q += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int xq = static_cast<int>(q % wq);
    const int64_t row = q / wq;              // b * H + y
    const int64_t b = row / H;
    const int y = static_cast<int>(row - b * H);
    const uint32_t* src = reinterpret_cast<const uint32_t*>(img + (row * W + xq * 4) * 3);
    const uint32_t w0 = src[0], w1 = src[1], w2 = src[2];  // r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
    float4 r, g, bl;
    r.x = s_lut[w0 & 255u];               g.x = s_lut[256 + ((w0 >> 8) & 255u)];   bl.x = s_lut[512 + ((w0 >> 16) & 255u)];
    r.y = s_lut[w0 >> 24];                g.y = s_lut[256 + (w1 & 255u)];          bl.y = s_lut[512 + ((w1 >> 8) & 255u)];
    r.z = s_lut[(w1 >> 16) & 255u];       g.z = s_lut[256 + (w1 >> 24)];           bl.z = s_lut[512 + (w2 & 255u)];
    r.w = s_lut[(w2 >> 8) & 255u];        g.w = s_lut[256 + ((w2 >> 16) & 255u)];  bl.w = s_lut[512 + (w2 >> 24)];
    float* o = out + ((b * 3) * H + y) * static_cast<int64_t>(W) + xq * 4;
    const int64_t plane = static_cast<int64_t>(H) * W;
    *reinterpret_cast<float4*>(o) = r;
    *reinterpret_cast<float4*>(o + plane) = g;
    *reinterpret_cast<float4*>(o + 2 * plane) = bl;
  }
}

// X[b*T + 0, :] = cls_pos (cls_token + pos_embed[0]) for every image.
__global__ void cls_row_kernel(float* __restrict__ X, const float* __restrict__ cls_pos, int T, int D) {
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < D; i += blockDim.x) X[static_cast<int64_t>(b) * T * D + i] = cls_pos[i];
}

// One warp per row.  Two-pass statistics in registers (mean, then centred sum of squares) in fp32.
// Row remap (for the final norm, which drops the cls token): input row r = g*rows_in + t is skipped when
// t < skip, else written to output row g*(rows_in - skip) + (t - skip).
// With `Xlo` set, `X` is the hi plane of a two-term fp16 stream (gemm_tc.cuh) and the row is hi + lo.
template <int VEC>  // D == 128 * VEC  (VEC float4 per lane)
__global__ void layernorm_kernel(const float* __restrict__ X, const __half* __restrict__ Xlo,
                                 const float* __restrict__ gamma,
                                 const float* __restrict__ beta, __half* __restrict__ out16, int64_t ld16,
                                 float* __restrict__ out32, int64_t ld32, int M, int D, float eps,
                                 int rows_in, int skip) {
  const int warps_per_block = blockDim.x >> 5;
  const int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  int64_t orow = row;
  if (rows_in > 0) {
    const int g = row / rows_in, t = row - g * rows_in;
    if (t < skip) return;
    orow = static_cast<int64_t>(g) * (rows_in - skip) + (t - skip);
  }
  float4 v[VEC];
  float s = 0.f;
  if (Xlo == nullptr) {
    const float4* xr = reinterpret_cast<const float4*>(X + static_cast<int64_t>(row) * D);
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = xr[lane + 32 * i];
  } else {
    const uint2* hr = reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(X) + static_cast<int64_t>(row) * D);
    const uint2* lr = reinterpret_cast<const uint2*>(Xlo + static_cast<int64_t>(row) * D);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const uint2 h = hr[lane + 32 * i], l = lr[lane + 32 * i];
      const float2 h0 = __half22float2(*reinterpret_cast<const __half2*>(&h.x));
      const float2 h1 = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
      const float2 l0 = __half22float2(*reinterpret_cast<const __half2*>(&l.x));
      const float2 l1 = __half22float2(*reinterpret_cast<const __half2*>(&l.y));
      v[i] = make_float4(h0.x + l0.x, h0.y + l0.y, h1.x + l1.x, h1.y + l1.y);
    }
  }
#pragma unroll
  for (int i = 0; i < VEC; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) / D + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const float4 g = __ldg(g4 + lane + 32 * i), bb = __ldg(b4 + lane + 32 * i);
    float4 y;
    y.x = (v[i].x - mean) * rstd * g.x + bb.x;
    y.y = (v[i].y - mean) * rstd * g.y + bb.y;
    y.z = (v[i].z - mean) * rstd * g.z + bb.z;
    y.w = (v[i].w - mean) * rstd * g.w + bb.w;
    if (out32 != nullptr)
      reinterpret_cast<float4*>(out32 + orow * ld32)[lane + 32 * i] = y;
    if (out16 != nullptr) {
      const __half2 h0 = __floats2half2_rn(y.x, y.y), h1 = __floats2half2_rn(y.z, y.w);
      uint2 pk;
      pk.x = *reinterpret_cast<const uint32_t*>(&h0);
      pk.y = *reinterpret_cast<const uint32_t*>(&h1);
      reinterpret_cast<uint2*>(out16 + orow * ld16)[lane + 32 * i] = pk;
    }
  }
}

// Entry of the folded-LayerNorm chain (gemm_tc.cuh): the fp32 tokens (patch embedding + position) become the two-term
// fp16 residual stream x = hi + lo, with (sum, sum of squares) of every row in slot 0 of its statistics and the other
// slots cleared.  Layer 0 only: later layers get all three from the epilogue of attn.proj / mlp.fc2.  One warp per row.
template <int VEC>
__global__ void split_rowstats_kernel(const float* __restrict__ X, __half* __restrict__ xhi, __half* __restrict__ xlo,
                                      int64_t ld16, float2* __restrict__ stats, int slots, int M, int D) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const float4* xr = reinterpret_cast<const float4*>(X + static_cast<int64_t>(row) * D);
  float s = 0.f, q = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const float4 v = xr[lane + 32 * i];
    s += (v.x + v.y) + (v.z + v.w);
    q += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
    const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
    const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
    const __half2 l0 = __floats2half2_rn(v.x - f0.x, v.y - f0.y), l1 = __floats2half2_rn(v.z - f1.x, v.w - f1.y);
    uint2 ph, pl;
    ph.x = *reinterpret_cast<const uint32_t*>(&h0);
    ph.y = *reinterpret_cast<const uint32_t*>(&h1);
    pl.x = *reinterpret_cast<const uint32_t*>(&l0);
    pl.y = *reinterpret_cast<const uint32_t*>(&l1);
    reinterpret_cast<uint2*>(xhi + static_cast<int64_t>(row) * ld16)[lane + 32 * i] = ph;
    reinterpret_cast<uint2*>(xlo + static_cast<int64_t>(row) * ld16)[lane + 32 * i] = pl;
  }
  s = warp_sum(s);
  q = warp_sum(q);
  if (lane < slots)
    stats[static_cast<int64_t>(row) * slots + lane] = (lane == 0) ? make_float2(s, q) : make_float2(0.f, 0.f);
}

// fp32 view of a two-term fp16 stream (unit-test entry mhmr_op_resid_ln_linear_f16).
__global__ void merge_split_kernel(const __half* __restrict__ xhi, const __half* __restrict__ xlo,
                                   float* __restrict__ X, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    X[i] = __half2float(xhi[i]) + __half2float(xlo[i]);
}

// Load-time folding of a LayerNorm into the Linear that follows it (gemm_tc.cuh): one warp per output feature.
//   W16[n,k] = fp16(W[n,k] ln_gamma[k] - mean_k(W[n,:] ln_gamma));   bias2[n] = bias[n] + sum_k ln_beta[k] W[n,k]
// Rows of the folded weight are centred: sum_k x[k] W16[n,k] then already equals sum_k (x[k] - mean(x)) W'[n,k].
__global__ void fold_ln_linear_kernel(const float* __restrict__ W, const float* __restrict__ bias,
                                      const float* __restrict__ ln_g, const float* __restrict__ ln_b,
                                      __half* __restrict__ W16, float* __restrict__ bias2, int N, int K) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  const int lane = threadIdx.x & 31;
  const float* wr = W + static_cast<int64_t>(n) * K;
  float c = 0.f, bb = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float w = wr[k];
    c += w * ln_g[k];
    bb += ln_b[k] * w;
  }
  const float mean = warp_sum(c) / static_cast<float>(K);
  bb = warp_sum(bb);
  for (int k = lane; k < K; k += 32)
    W16[static_cast<int64_t>(n) * K + k] = __float2half_rn(wr[k] * ln_g[k] - mean);
  if (lane == 0) bias2[n] = bias[n] + bb;
}

__global__ void f32_to_f16_2d_kernel(const float* __restrict__ src, int64_t lds, __half* __restrict__ dst,
                                     int64_t ldd, int rows, int cols) {
  const int64_t total = static_cast<int64_t>(rows) * cols;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols, c = i - r * cols;
    dst[r * ldd + c] = __float2half_rn(src[r * lds + c]);
  }
}

}  // namespace

int im2col_patch14(const float* x, __half* A, int B, int S, int ldA, cudaStream_t stream) {
  MHMR_REQUIRE(S % 14 == 0 && ldA >= 588, "im2col: bad geometry");
  const int N = (S / 14) * (S / 14);
  im2col_patch14_kernel<<<B * N, 128, 0, stream>>>(x, A, B, S, ldA);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int im2col_u8_patch14(const uint8_t* img, const float* lut, __half* A, int B, int S, int ldA, cudaStream_t stream) {
  MHMR_REQUIRE(S % 14 == 0, "Invalid img size");
  const int N = (S / 14) * (S / 14);
  im2col_u8_patch14_kernel<<<B * N, 192, 0, stream>>>(img, lut, A, S, ldA);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int normalize_u8(const uint8_t* img, const float* lut, float* out, int B, int H, int W, cudaStream_t stream) {
  MHMR_REQUIRE(B > 0 && H > 0 && W > 0 && W % 4 == 0, "normalize_u8: width must be a multiple of 4");
  MHMR_REQUIRE((reinterpret_cast<uintptr_t>(img) & 3u) == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0,
               "normalize_u8: image must be 4-byte aligned, output 16-byte aligned");
  const int64_t n_quads = static_cast<int64_t>(B) * H * (W / 4);
  const int blocks = static_cast<int>(std::min<int64_t>((n_quads + 255) / 256, device_sm_count() * 8));
  normalize_u8_kernel<<<blocks, 256, 0, stream>>>(img, lut, out, H, W, n_quads);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int cls_rows(float* X, const float* cls_pos, int B, int T, int D, cudaStream_t stream) {
  cls_row_kernel<<<B, 256, 0, stream>>>(X, cls_pos, T, D);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int layernorm(const float* X, const float* gamma, const float* beta, __half* out16, int64_t ld16,
              float* out32, int64_t ld32, int M, int D, float eps, int rows_in, int skip,
              cudaStream_t stream) {
  return layernorm_split(X, nullptr, gamma, beta, out16, ld16, out32, ld32, M, D, eps, rows_in, skip, stream);
}

int layernorm_split(const void* X, const __half* Xlo, const float* gamma, const float* beta, __half* out16,
                    int64_t ld16, float* out32, int64_t ld32, int M, int D, float eps, int rows_in, int skip,
                    cudaStream_t stream) {
  MHMR_REQUIRE(D % 128 == 0 && D <= 1024, "layernorm: D must be a multiple of 128, <= 1024");
  MHMR_REQUIRE(out16 != nullptr || out32 != nullptr, "layernorm: no output");
  const int wpb = 8;
  dim3 grid((M + wpb - 1) / wpb), block(wpb * 32);
#define MHMR_LN_CASE(V)                                                                              \
  case V:                                                                                            \
    layernorm_kernel<V><<<grid, block, 0, stream>>>(static_cast<const float*>(X), Xlo, gamma, beta, out16, ld16, \
                                                    out32, ld32, M, D, eps, rows_in, skip);          \
    break;
  switch (D / 128) {
    MHMR_LN_CASE(1) MHMR_LN_CASE(2) MHMR_LN_CASE(3) MHMR_LN_CASE(4) MHMR_LN_CASE(5) MHMR_LN_CASE(6)
    MHMR_LN_CASE(7) MHMR_LN_CASE(8)
    default: break;
  }
#undef MHMR_LN_CASE
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int split_rowstats(const float* X, __half* xhi, __half* xlo, int64_t ld16, float2* stats, int slots, int M, int D,
                   cudaStream_t stream) {
  MHMR_REQUIRE(D % 128 == 0 && D <= 1024 && slots >= 1 && slots <= 32, "split_rowstats: bad geometry");
  const int wpb = 8;
  dim3 grid((M + wpb - 1) / wpb), block(wpb * 32);
#define MHMR_CS_CASE(V) \
  case V: split_rowstats_kernel<V><<<grid, block, 0, stream>>>(X, xhi, xlo, ld16, stats, slots, M, D); break;
  switch (D / 128) {
    MHMR_CS_CASE(1) MHMR_CS_CASE(2) MHMR_CS_CASE(3) MHMR_CS_CASE(4) MHMR_CS_CASE(5) MHMR_CS_CASE(6)
    MHMR_CS_CASE(7) MHMR_CS_CASE(8)
    default: break;
  }
#undef MHMR_CS_CASE
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int merge_split(const __half* xhi, const __half* xlo, float* X, int64_t n, cudaStream_t stream) {
  merge_split_kernel<<<static_cast<int>(std::min<int64_t>((n + 255) / 256, device_sm_count() * 16)), 256, 0, stream>>>(xhi, xlo, X, n);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int fold_ln_linear(const float* W, const float* bias, const float* ln_g, const float* ln_b, __half* W16,
                   float* bias2, int N, int K, cudaStream_t stream) {
  fold_ln_linear_kernel<<<(N + 7) / 8, 256, 0, stream>>>(W, bias, ln_g, ln_b, W16, bias2, N, K);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int f32_to_f16_2d(const float* src, int64_t lds, __half* dst, int64_t ldd, int rows, int cols,
                  cudaStream_t stream) {
  const int64_t total = static_cast<int64_t>(rows) * cols;
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
  if (blocks < 1) blocks = 1;
  f32_to_f16_2d_kernel<<<blocks, 256, 0, stream>>>(src, lds, dst, ldd, rows, cols);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

}  // namespace mhmr

namespace mhmr {
namespace {
// dst[r, dcol + c] = src[r, scol + c] for c < cols; when `zero_fill`, the rest of the dst row is zeroed.
__global__ void repack_f32_kernel(const float* __restrict__ src, int64_t lds, int scol, float* __restrict__ dst,
                                  int64_t ldd, int dcol, int rows, int cols, int zero_fill) {
  const int r = blockIdx.x;
  if (r >= rows) return;
  if (zero_fill) {
    for (int c = threadIdx.x; c < ldd; c += blockDim.x) {
      const int sc = c - dcol;
      dst[r * ldd + c] = (sc >= 0 && sc < cols) ? src[r * lds + scol + sc] : 0.f;
    }
  } else {
    for (int c = threadIdx.x; c < cols; c += blockDim.x) dst[r * ldd + dcol + c] = src[r * lds + scol + c];
  }
}
__global__ void add_vec_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out,
                               int64_t n, int64_t b_period) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    out[i] = a[i] + b[i % b_period];
}
}  // namespace

int repack_f32(const float* src, int64_t lds, int scol, float* dst, int64_t ldd, int dcol, int rows,
               int cols, bool zero_fill, cudaStream_t stream) {
  repack_f32_kernel<<<rows, 256, 0, stream>>>(src, lds, scol, dst, ldd, dcol, rows, cols, zero_fill ? 1 : 0);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

// out[i] = a[i] + b[i % b_period]
int add_vec(const float* a, const float* b, float* out, int64_t n, int64_t b_period, cudaStream_t stream) {
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > 2048) blocks = 2048;
  add_vec_kernel<<<blocks, 256, 0, stream>>>(a, b, out, n, b_period);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}
}  // namespace mhmr
