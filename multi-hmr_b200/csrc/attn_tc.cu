// Multi-head self-attention of the DINOv2 backbone (head dim 64) on wgmma tensor cores.
//
// Replaces `softmax(q k^T / 8) v` of dinov2 `Attention.forward` (reached from the reference at
// blocks/dinov2.py:25; SURVEY.md §2.4 k4).  Flash-style: the T x T score matrix never leaves the SM.
//
//   grid  = one CTA per (image, head, 128-row query tile); query tile fastest, so that the CTAs running at the
//           same time share the K / V of few (image, head) pairs in L2.
//   CTA   = 384 threads = 3 warpgroups: warpgroup 0 loads Q once and streams K / V tiles of 128 keys through a
//           ring of 4 smem stages (TMA, one elected lane of warp 0); warpgroups 1 and 2 each own 64 query rows.
//   smem  = Q (16 KB) | kStages x (K 16 KB | V 16 KB), 128B swizzle, one TMA box per tile.
//   S = Q K^T : wgmma m64n128k16, A = Q (smem, K-major), B = K tile (smem, K-major); S in registers.
//   O += P V  : wgmma m64n64k16, A = P (registers: the fp16 S fragments ARE the A fragments of the next MMA),
//               B = V tile (smem, MN-major).
// Online softmax in fp32 in the exp2 domain; each thread holds 2 rows x 32 columns of S, the row max and sum
// are reduced over the 4 lanes that share a row.
//
// The consumer warpgroups overlap tensor-core work with the softmax twice over: each issues S_{j} = Q K_j^T
// together with O += P_{j-1} V_{j-1} and runs the softmax of S_j while that PV is in flight, and the two take
// turns issuing their wgmmas (named barriers), so one's softmax runs under the other's MMAs.
//
// Ragged sequence (T = N + 1 is 1 mod 128 at 224, 448, 672 and 896 px, 17 mod 128 at 280 and 1288 px): the QKV
// tensor map is 3-D (column, token, image), so TMA zero-fills the rows of a tile beyond the image's T rather than
// reading the next image's (P = 0 times a non-finite value there would be NaN); the keys beyond T in the last
// tile are masked to -inf. A last tile of at most 32 keys runs 32 keys wide (S by m64n32, PV by 2 k-steps). Query
// rows beyond T are computed and not stored.
//
// Grid at ViT-L (16 heads) on 132 SMs: 896 px batch 8 (T = 4097) 4224 CTAs = 32.0 waves; 672 px batch 4
// (T = 2305) 1216 CTAs = 9.2 waves; 1288 px batch 2 (T = 8465) 2144 CTAs = 16.2 waves.
#include "kernels.cuh"

namespace mhmr {

namespace {

constexpr int kHeadDim = 64;
constexpr int kBlockQ = 128;
constexpr int kBlockKV = 128;
constexpr int kTileBytes = 128 * kHeadDim * 2;  // 16 KB: Q, K or V tile
constexpr int kStages = 4;
constexpr int kAttnThreads = 384;
constexpr int kRegsProducer = 40, kRegsConsumer = 232;
// Q + K/V ring + 1 KB alignment pad + barriers
constexpr int kAttnSmemBytes = kTileBytes * (1 + 2 * kStages) + 1024 + 256;

__device__ __forceinline__ float ex2(float x) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x));
  return e;
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// S = Q K^T over the first kN keys (128 or 32) of a K tile; the caller fences and commits.
template <int kN>
__device__ __forceinline__ void issue_qk(float (&sc)[64], uint64_t q_desc, uint64_t k_desc) {
#pragma unroll
  for (int k = 0; k < kHeadDim / 16; ++k) {
    if constexpr (kN == 128)
      wgmma_m64n128_ss(sc, q_desc + 2u * k, k_desc + 2u * k, k > 0 ? 1u : 0u);
    else
      wgmma_m64n32_ss(*reinterpret_cast<float(*)[16]>(sc), q_desc + 2u * k, k_desc + 2u * k, k > 0 ? 1u : 0u);
  }
}

// O += P V over the first 16 kK keys of a V tile (128 keys x 64 dims, N contiguous: MN-major, 8-key groups 1024 B
// apart, 16 keys per step); the caller fences and commits.
template <int kK>
__device__ __forceinline__ void issue_pv(float (&o)[32], const uint32_t (&p)[8][4], uint64_t v_desc) {
#pragma unroll
  for (int kk = 0; kk < kK; ++kk) wgmma_m64n64_rs_bt(o, p[kk], v_desc + 128u * kk);
}

// One online-softmax step over the first kN columns of S, of which the first `valid` are keys of this image:
// S <- exp2(S scale_log2 - m_new) in place, m_run / l_run updated, alpha = the factor the old O is scaled by.
template <int kN>
__device__ __forceinline__ void softmax_step(float (&sc)[64], int valid, float scale_log2, int lane,
                                             float (&m_run)[2], float (&l_run)[2], float (&alpha)[2]) {
  if (valid < kN) {
#pragma unroll
    for (int i = 0; i < kN / 2; ++i)
      if (8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= valid) sc[i] = -INFINITY;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float mx = -INFINITY;
#pragma unroll
    for (int g = 0; g < kN / 8; ++g) mx = fmaxf(mx, fmaxf(sc[4 * g + 2 * h], sc[4 * g + 2 * h + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_new = fmaxf(m_run[h], mx * scale_log2);
    alpha[h] = ex2(m_run[h] - m_new);  // 0 on the first tile
    m_run[h] = m_new;
    float sum = 0.f;
#pragma unroll
    for (int g = 0; g < kN / 8; ++g) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 4 * g + 2 * h + e;
        sc[i] = ex2(fmaf(sc[i], scale_log2, -m_new));
        sum += sc[i];
      }
    }
    l_run[h] = l_run[h] * alpha[h] + sum;  // partial over this lane's columns; reduced over the quad at the end
  }
}

// P as fp16 A fragments, one set of 4 registers per 16 keys
template <int kK>
__device__ __forceinline__ void pack_p(const float (&sc)[64], uint32_t (&p)[8][4]) {
#pragma unroll
  for (int kk = 0; kk < kK; ++kk) {
    p[kk][0] = pack_half2(sc[8 * kk + 0], sc[8 * kk + 1]);
    p[kk][1] = pack_half2(sc[8 * kk + 2], sc[8 * kk + 3]);
    p[kk][2] = pack_half2(sc[8 * kk + 4], sc[8 * kk + 5]);
    p[kk][3] = pack_half2(sc[8 * kk + 6], sc[8 * kk + 7]);
  }
}

// kLastN = 32 runs the last key tile (at most 32 keys of this image, n_kv >= 2) 32 keys wide: S by m64n32 and
// PV by 2 k-steps instead of 8; kLastN = 128 runs every tile full width.
template <int kLastN>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQKV, __half* __restrict__ out, int64_t ldo, int T, int D,
                int heads, int n_qt, float scale_log2) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + kTileBytes;  // stage s: K at sKV + 2 s kTileBytes, V right behind it
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kTileBytes * (1 + 2 * kStages));
  uint64_t* q_full = bars;                 // TMA -> consumers
  uint64_t* kv_full = bars + 1;            // [kStages]  TMA -> consumers
  uint64_t* kv_empty = kv_full + kStages;  // [kStages]  consumers -> TMA

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int qt = blockIdx.x % n_qt;
  const int bh = blockIdx.x / n_qt;
  const int head = bh % heads, img = bh / heads;
  const int q0 = qt * kBlockQ;
  const int row0 = img * T;  // first token row of this image in the [B*T, 3D] matrix
  const int n_kv = (T + kBlockKV - 1) / kBlockKV;

  griddep_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    mbar_init(q_full, 1);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();  // qkv of the preceding GEMM is complete and visible

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegsProducer));
    if (warp == 0) {
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(q_full, kTileBytes);
        // Q is read by one CTA, K / V by every query tile of the (image, head): keep K / V in L2
        tma_load_3d_hint(sQ, &tmQKV, q_full, head * kHeadDim, q0, img, kCacheEvictFirst);
      }
      __syncwarp();
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % kStages;
        mbar_wait(&kv_empty[s], ((j / kStages) & 1) ^ 1);
        if (elect_one_sync()) {
          uint8_t* dk = sKV + 2 * s * kTileBytes;
          mbar_arrive_expect_tx(&kv_full[s], 2 * kTileBytes);
          tma_load_3d_hint(dk, &tmQKV, &kv_full[s], D + head * kHeadDim, j * kBlockKV, img, kCacheEvictLast);
          tma_load_3d_hint(dk + kTileBytes, &tmQKV, &kv_full[s], 2 * D + head * kHeadDim, j * kBlockKV, img,
                           kCacheEvictLast);
        }
        __syncwarp();
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegsConsumer));
  const int cw = wg - 1;  // query rows 64 cw .. 64 cw + 63 of the tile
  const int w = warp & 3;
  const bool release_lane = (threadIdx.x & 127) == 0;
  // accumulator fragments: register i holds row 16 w + lane / 4 + 8 ((i >> 1) & 1) of the warpgroup's 64 rows,
  // column 8 (i >> 2) + 2 (lane & 3) + (i & 1)
  const uint64_t q_desc = make_sw128_desc(smem_u32(sQ + cw * 64 * 128), 16, 1024);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float sc[64], alpha[2];
  uint32_t p[8][4];
  const int valid_last = T - (n_kv - 1) * kBlockKV;
  auto k_desc = [&](int j) { return make_sw128_desc(smem_u32(sKV + 2 * (j % kStages) * kTileBytes), 16, 1024); };
  auto v_desc = [&](int j) {
    return make_sw128_desc(smem_u32(sKV + (2 * (j % kStages) + 1) * kTileBytes), 1024, 1024);
  };
  // Ping-pong: the two consumer warpgroups take turns issuing their wgmmas. Named barrier 1 + cw opens the turn
  // of warpgroup cw; the other warpgroup arrives on it once it has issued its own, so the softmax of one warpgroup
  // runs while the tensor cores work on the other's MMAs. Each warpgroup issues n_kv + 1 times; warpgroup 1 opens
  // the first turn of warpgroup 0 and skips its own last hand-over, which leaves both barriers balanced.
  const uint32_t my_turn = 1 + cw, other_turn = 2 - cw;
  if (cw == 1) named_bar_arrive(other_turn, 256);
  mbar_wait(q_full, 0);

  // Within a warpgroup, S_j = Q K_j^T is issued together with O += P_{j-1} V_{j-1}; the softmax of S_j runs while
  // that PV is in flight, and O is rescaled by alpha_j once it lands, before P_j V_j is issued: the same
  // per-row arithmetic as a sequential S, softmax, PV loop.
  mbar_wait(&kv_full[0], 0);
  named_bar_sync(my_turn, 256);
  wgmma_fence();
  issue_qk<128>(sc, q_desc, k_desc(0));
  wgmma_commit();
  named_bar_arrive(other_turn, 256);
  wgmma_wait<0>();
  wgmma_fence_regs(sc);
  softmax_step<128>(sc, n_kv == 1 ? valid_last : kBlockKV, scale_log2, lane, m_run, l_run, alpha);
  pack_p<8>(sc, p);  // O is still 0: no rescale

  // key tile j >= 1, the first kN keys of it (the wgmma shapes are fixed at compile time: a runtime choice
  // between them would make ptxas serialize every wgmma of the kernel)
  auto step = [&](int j, auto width) {
    constexpr int kN = decltype(width)::value;
    mbar_wait(&kv_full[j % kStages], (j / kStages) & 1);
    named_bar_sync(my_turn, 256);
    wgmma_fence();
    issue_qk<kN>(sc, q_desc, k_desc(j));
    wgmma_commit();
    issue_pv<8>(o, p, v_desc(j - 1));
    wgmma_commit();
    named_bar_arrive(other_turn, 256);
    wgmma_wait<1>();  // S_j
    wgmma_fence_regs(sc);
    softmax_step<kN>(sc, j == n_kv - 1 ? valid_last : kBlockKV, scale_log2, lane, m_run, l_run, alpha);
    wgmma_wait<0>();  // P_{j-1} V_{j-1}: stage j - 1 is no longer read
    wgmma_fence_regs(o);
    if (release_lane) mbar_arrive(&kv_empty[(j - 1) % kStages]);
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      o[4 * g + 0] *= alpha[0];
      o[4 * g + 1] *= alpha[0];
      o[4 * g + 2] *= alpha[1];
      o[4 * g + 3] *= alpha[1];
    }
    pack_p<kN / 16>(sc, p);
  };
  constexpr bool kNarrow = kLastN < kBlockKV;  // then n_kv >= 2 (attention_forward)
  for (int j = 1; j < n_kv - (kNarrow ? 1 : 0); ++j) step(j, std::integral_constant<int, kBlockKV>{});
  if constexpr (kNarrow) step(n_kv - 1, std::integral_constant<int, kLastN>{});

  named_bar_sync(my_turn, 256);
  wgmma_fence();
  issue_pv<kLastN / 16>(o, p, v_desc(n_kv - 1));
  wgmma_commit();
  if (cw == 0) named_bar_arrive(other_turn, 256);
  wgmma_wait<0>();
  wgmma_fence_regs(o);
  if (release_lane) mbar_arrive(&kv_empty[(n_kv - 1) % kStages]);

  // epilogue: O / l -> fp16 -> out[img*T + q, head*64 + :]
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = 1.0f / l;
    const int q = q0 + cw * 64 + w * 16 + (lane >> 2) + 8 * h;
    if (q < T) {
      __half* dst = out + static_cast<int64_t>(row0 + q) * ldo + head * kHeadDim + 2 * (lane & 3);
#pragma unroll
      for (int g = 0; g < 8; ++g)
        *reinterpret_cast<uint32_t*>(dst + 8 * g) = pack_half2(o[4 * g + 2 * h] * inv_l, o[4 * g + 2 * h + 1] * inv_l);
    }
  }
}

}  // namespace

// qkv: [B*T, 3*D] fp16 (row pitch ld_qkv), q|k|v column blocks, head h = columns h*64..h*64+63 of each.
// out: [B*T, D] fp16 (row pitch ldo).
int attention_forward(const __half* qkv, int64_t ld_qkv, __half* out, int64_t ldo, int B, int T, int D,
                      cudaStream_t stream) {
  MHMR_REQUIRE(D % kHeadDim == 0, "attention: embed dim must be a multiple of 64");
  MHMR_REQUIRE(ld_qkv % 8 == 0 && ldo % 8 == 0, "attention: row pitches must be multiples of 8");
  MHMR_REQUIRE(B > 0 && T > 0, "attention: empty problem");
  CUtensorMap tm;  // (column, token, image): boxes of 64 columns x 128 tokens of one image
  int rc = make_tmap_3d(&tm, qkv, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, B, T, 3ull * D,
                        static_cast<uint64_t>(T) * ld_qkv * 2, ld_qkv * 2, 128, 64, true);
  if (rc != MHMR_OK) return rc;
  const int heads = D / kHeadDim;
  const int n_qt = (T + kBlockQ - 1) / kBlockQ;
  const int n_kv = (T + kBlockKV - 1) / kBlockKV;
  static PerDeviceOnce once;
  if (once.first()) {
    MHMR_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kAttnSmemBytes));
    MHMR_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kAttnSmemBytes));
  }
  const bool narrow_tail = n_kv >= 2 && T - (n_kv - 1) * kBlockKV <= 32;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(B * heads * n_qt);
  cfg.blockDim = dim3(kAttnThreads);
  cfg.dynamicSmemBytes = kAttnSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  const float scale_log2 = 0.125f * 1.4426950408889634f;  // head_dim^-0.5 * log2(e)
  MHMR_CUDA_CHECK(cudaLaunchKernelEx(&cfg, narrow_tail ? attn_fwd_kernel<32> : attn_fwd_kernel<128>, tm, out, ldo,
                                     T, D, heads, n_qt, scale_log2));
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

}  // namespace mhmr
