// Fused GEMM epilogue of the wgmma kernels (gemm_tc.cu).
#pragma once
#include "gemm_tc.cuh"

namespace mhmr {

constexpr int kScratchStride = 36;               // floats per scratch row (32 + 4: conflict-free float4)
constexpr int kScratchBytes = 32 * kScratchStride * 4;


// The accumulator chunk (32 rows x 32 columns) is staged by the caller in a per-warp smem scratch (row r at
// r * kScratchStride) and read back so that global memory is accessed with lanes along the contiguous dimension:
//   fp32 outputs: 8 lanes x float4 cover one 128-byte row segment, 4 rows per warp instruction;
//   fp16 outputs: 4 lanes x (8 halves) cover one 64-byte row segment, 8 rows per warp instruction.
// Per-warp, per-tile state of the folded-LayerNorm epilogues (gemm_tc.cuh); empty work for the other kinds.
struct EpiRowState {
  float sum[4], sq[4];  // EPI_LS_RESID_SPLIT: partial sum / sum of squares of rows k*8 + (lane >> 2) over this
                        // lane's columns of every chunk of the tile
  float rstd;           // EPI_LN_*: 1/sigma of row m_base + lane
};

template <int EPI>
constexpr bool epi_is_ln_consumer() { return EPI == EPI_LN_BIAS_F16 || EPI == EPI_LN_GELU_F16; }

// Row statistics of a consumer tile, loaded one tile ahead (the epilogue of mlp.fc1 has no slack for an exposed L2
// round trip per tile): lane i holds the <= 8 partial (sum, sumsq) pairs of row m_base + i.
struct EpiStatsPrefetch {
  float4 v[4];
};
constexpr int kMaxStatSlots = 8;

template <int EPI>
__device__ __forceinline__ void epilogue_load_row_stats(EpiStatsPrefetch& pf, const GemmEpi& ep, int M, int m_base,
                                                        int lane) {
  if constexpr (epi_is_ln_consumer<EPI>()) {
    const int m = m_base + lane;
    const float4* p = reinterpret_cast<const float4*>(ep.stats + static_cast<int64_t>(m) * ep.stat_slots);
    const int n4 = (m < M) ? (ep.stat_slots >> 1) : 0;  // stat_slots is even (two epilogue warps per column tile)
#pragma unroll
    for (int i = 0; i < 4; ++i) pf.v[i] = (i < n4) ? __ldcg(p + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// Start of a tile: consumers reduce the prefetched partial statistics (one row per lane), producers clear their
// partial sums.  `K` is the LayerNorm width (= the consumer GEMM's K).
template <int EPI>
__device__ __forceinline__ void epilogue_tile_begin(EpiRowState& st, const EpiStatsPrefetch& pf, const GemmEpi& ep,
                                                    int K) {
  if constexpr (EPI == EPI_LS_RESID_SPLIT) {
#pragma unroll
    for (int k = 0; k < 4; ++k) st.sum[k] = st.sq[k] = 0.f;
  }
  if constexpr (epi_is_ln_consumer<EPI>()) {
    const float s = (pf.v[0].x + pf.v[0].z) + (pf.v[1].x + pf.v[1].z) + (pf.v[2].x + pf.v[2].z) + (pf.v[3].x + pf.v[3].z);
    const float q = (pf.v[0].y + pf.v[0].w) + (pf.v[1].y + pf.v[1].w) + (pf.v[2].y + pf.v[2].w) + (pf.v[3].y + pf.v[3].w);
    const float inv = 1.0f / static_cast<float>(K);
    const float mean = s * inv;
    const float var = fmaxf(q * inv - mean * mean, 0.f);
    st.rstd = rsqrtf(var + ep.ln_eps);
  }
}

// End of a tile (EPI_LS_RESID_SPLIT): the 4 lanes that share a row group hold 4 rows x their 8 columns of every chunk;
// a halving exchange (2 + 1 shuffles per quantity) leaves lane `cg` with the totals of row cg*8 + rs.
template <int EPI>
__device__ __forceinline__ void epilogue_tile_end(EpiRowState& st, const GemmEpi& ep, int M, int m_base, int slot,
                                                  int lane) {
  if constexpr (EPI == EPI_LS_RESID_SPLIT) {
    const int cg = lane & 3, rs = lane >> 2;
    const bool h2 = cg & 2, h1 = cg & 1;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float ss = h2 ? st.sum[i] : st.sum[i + 2], ks = h2 ? st.sum[i + 2] : st.sum[i];
      const float sq = h2 ? st.sq[i] : st.sq[i + 2], kq = h2 ? st.sq[i + 2] : st.sq[i];
      st.sum[i] = ks + __shfl_xor_sync(0xffffffffu, ss, 2);
      st.sq[i] = kq + __shfl_xor_sync(0xffffffffu, sq, 2);
    }
    {
      const float ss = h1 ? st.sum[0] : st.sum[1], ks = h1 ? st.sum[1] : st.sum[0];
      const float sq = h1 ? st.sq[0] : st.sq[1], kq = h1 ? st.sq[1] : st.sq[0];
      st.sum[0] = ks + __shfl_xor_sync(0xffffffffu, ss, 1);
      st.sq[0] = kq + __shfl_xor_sync(0xffffffffu, sq, 1);
    }
    const int m = m_base + cg * 8 + rs;
    if (m < M) ep.stats[static_cast<int64_t>(m) * ep.stat_slots + slot] = make_float2(st.sum[0], st.sq[0]);
  }
}

__device__ __forceinline__ void unpack_half8(const uint4& u, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

template <int EPI>
__device__ __forceinline__ void epilogue_chunk(const float* scratch, const GemmEpi& ep, int M, int N, int m_base,
                                               int n0, int lane, EpiRowState& st) {
  constexpr bool kLn = epi_is_ln_consumer<EPI>();
  constexpr bool kRowAdd16 = (EPI == EPI_ROWADD_F16);
  constexpr bool kF16 = (EPI == EPI_BIAS_F16 || EPI == EPI_BIAS_GELU_F16 || EPI == EPI_BIAS_RELU_F16 || kLn || kRowAdd16);
  constexpr bool kResid = (EPI == EPI_LS_RESID_F32);
  if constexpr (EPI == EPI_LS_RESID_SPLIT) {
    // residual stream as two fp16 planes: same lane mapping as the fp16 outputs (8 columns x 2 planes = 2 x 16 B)
    const int cg = lane & 3, rs = lane >> 2;
    const int n = n0 + cg * 8;
    float bb[8], gg[8];
    *reinterpret_cast<float4*>(bb) = __ldg(reinterpret_cast<const float4*>(ep.bias + n));
    *reinterpret_cast<float4*>(bb + 4) = __ldg(reinterpret_cast<const float4*>(ep.bias + n + 4));
    *reinterpret_cast<float4*>(gg) = __ldg(reinterpret_cast<const float4*>(ep.gamma + n));
    *reinterpret_cast<float4*>(gg + 4) = __ldg(reinterpret_cast<const float4*>(ep.gamma + n + 4));
    uint4 hi[4], lo[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int m = m_base + k * 8 + rs;
      const int64_t off = static_cast<int64_t>(m) * ep.ldx16 + n;
      hi[k] = lo[k] = make_uint4(0u, 0u, 0u, 0u);
      if (m < M) {
        hi[k] = *reinterpret_cast<const uint4*>(ep.x16 + off);
        lo[k] = *reinterpret_cast<const uint4*>(ep.xlo + off);
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int rl = k * 8 + rs;
      float v[8], xh[8], xl[8], a[8];
      *reinterpret_cast<float4*>(v) = *reinterpret_cast<const float4*>(scratch + rl * kScratchStride + cg * 8);
      *reinterpret_cast<float4*>(v + 4) = *reinterpret_cast<const float4*>(scratch + rl * kScratchStride + cg * 8 + 4);
      unpack_half8(hi[k], xh);
      unpack_half8(lo[k], xl);
      float s = 0.f, q = 0.f;
      uint32_t ph[4], pl[4];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        a[i] = fmaf(gg[i], v[i] + bb[i], xh[i] + xl[i]);
        s += a[i];
        q = fmaf(a[i], a[i], q);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const __half2 h = __floats2half2_rn(a[2 * i], a[2 * i + 1]);
        const float2 hf = __half22float2(h);
        const __half2 l = __floats2half2_rn(a[2 * i] - hf.x, a[2 * i + 1] - hf.y);
        ph[i] = *reinterpret_cast<const uint32_t*>(&h);
        pl[i] = *reinterpret_cast<const uint32_t*>(&l);
      }
      st.sum[k] += s;
      st.sq[k] += q;
      if (m_base + rl < M) {
        const int64_t off = static_cast<int64_t>(m_base + rl) * ep.ldx16 + n;
        *reinterpret_cast<uint4*>(ep.x16 + off) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
        *reinterpret_cast<uint4*>(ep.xlo + off) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
      }
    }
  } else if constexpr (kF16) {
    const int cg = lane & 3, rs = lane >> 2;  // 8 columns per lane, 8 rows per instruction
    const int n = n0 + cg * 8;
    float4 b0 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = b0;
    if constexpr (!kRowAdd16) {
      b0 = __ldg(reinterpret_cast<const float4*>(ep.bias + n));
      b1 = __ldg(reinterpret_cast<const float4*>(ep.bias + n + 4));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int rl = k * 8 + rs;
      const int m = m_base + rl;
      if constexpr (kRowAdd16) {  // per-row addend: row m % rows_in of the table
        if (m < M) {
          const float* ra = ep.rowadd + static_cast<int64_t>(m % ep.rows_in) * N + n;
          b0 = __ldg(reinterpret_cast<const float4*>(ra));
          b1 = __ldg(reinterpret_cast<const float4*>(ra + 4));
        }
      }
      const float4 v0 = *reinterpret_cast<const float4*>(scratch + rl * kScratchStride + cg * 8);
      const float4 v1 = *reinterpret_cast<const float4*>(scratch + rl * kScratchStride + cg * 8 + 4);
      float2 y[4];
      if constexpr (kLn) {
        // rstd * acc + b'  (the folded weight rows are centred: the mean term is already inside acc)
        const float rstd = __shfl_sync(0xffffffffu, st.rstd, rl);
        const float2 r2 = make_float2(rstd, rstd);
        y[0] = fma2(make_float2(v0.x, v0.y), r2, make_float2(b0.x, b0.y));
        y[1] = fma2(make_float2(v0.z, v0.w), r2, make_float2(b0.z, b0.w));
        y[2] = fma2(make_float2(v1.x, v1.y), r2, make_float2(b1.x, b1.y));
        y[3] = fma2(make_float2(v1.z, v1.w), r2, make_float2(b1.z, b1.w));
      } else {
        y[0] = add2(make_float2(v0.x, v0.y), make_float2(b0.x, b0.y));
        y[1] = add2(make_float2(v0.z, v0.w), make_float2(b0.z, b0.w));
        y[2] = add2(make_float2(v1.x, v1.y), make_float2(b1.x, b1.y));
        y[3] = add2(make_float2(v1.z, v1.w), make_float2(b1.z, b1.w));
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if constexpr (EPI == EPI_BIAS_GELU_F16 || EPI == EPI_LN_GELU_F16) y[i] = gelu_erf_fast2(y[i]);
        if constexpr (EPI == EPI_BIAS_RELU_F16) y[i] = make_float2(fmaxf(y[i].x, 0.0f), fmaxf(y[i].y, 0.0f));
      }
      const float x[8] = {y[0].x, y[0].y, y[1].x, y[1].y, y[2].x, y[2].y, y[3].x, y[3].y};
      const __half2 h0 = __floats2half2_rn(x[0], x[1]), h1 = __floats2half2_rn(x[2], x[3]);
      const __half2 h2 = __floats2half2_rn(x[4], x[5]), h3 = __floats2half2_rn(x[6], x[7]);
      uint4 pk;
      pk.x = *reinterpret_cast<const uint32_t*>(&h0);
      pk.y = *reinterpret_cast<const uint32_t*>(&h1);
      pk.z = *reinterpret_cast<const uint32_t*>(&h2);
      pk.w = *reinterpret_cast<const uint32_t*>(&h3);
      if (m < M)
        *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(ep.out) + static_cast<int64_t>(m) * ep.ldo + n) = pk;
    }
  } else {
    const int cg = lane & 7, rs = lane >> 3;  // 4 columns per lane, 4 rows per instruction
    const int n = n0 + cg * 4;
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f), g = make_float4(1.f, 1.f, 1.f, 1.f);
    if constexpr (kResid) {
      b = __ldg(reinterpret_cast<const float4*>(ep.bias + n));
      g = __ldg(reinterpret_cast<const float4*>(ep.gamma + n));
    } else if constexpr (EPI == EPI_BIAS_F32) {
      if (ep.bias != nullptr) b = __ldg(reinterpret_cast<const float4*>(ep.bias + n));
    }
    float* outp[8];
    float4 xres[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int m = m_base + k * 4 + rs;
      int64_t orow = m;
      if constexpr (EPI == EPI_ROWADD_F32) {
        const int grp = m / ep.rows_in, rin = m - grp * ep.rows_in;
        orow = static_cast<int64_t>(grp) * ep.rows_out + ep.row_off + rin;
        xres[k] = (m < M) ? __ldg(reinterpret_cast<const float4*>(ep.rowadd + static_cast<int64_t>(rin) * N + n))
                          : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      outp[k] = reinterpret_cast<float*>(ep.out) + orow * ep.ldo + n;
      if constexpr (kResid)
        xres[k] = (m < M) ? *reinterpret_cast<const float4*>(outp[k]) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int rl = k * 4 + rs;
      const float4 v = *reinterpret_cast<const float4*>(scratch + rl * kScratchStride + cg * 4);
      float4 a;
      if constexpr (kResid) {
        a.x = xres[k].x + g.x * (v.x + b.x);
        a.y = xres[k].y + g.y * (v.y + b.y);
        a.z = xres[k].z + g.z * (v.z + b.z);
        a.w = xres[k].w + g.w * (v.w + b.w);
      } else if constexpr (EPI == EPI_ROWADD_F32) {
        a.x = v.x + xres[k].x; a.y = v.y + xres[k].y; a.z = v.z + xres[k].z; a.w = v.w + xres[k].w;
      } else {
        a.x = v.x + b.x; a.y = v.y + b.y; a.z = v.z + b.z; a.w = v.w + b.w;
      }
      if (m_base + rl < M) *reinterpret_cast<float4*>(outp[k]) = a;
    }
  }
  __syncwarp();
}

}  // namespace mhmr
