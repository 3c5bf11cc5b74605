// wgmma + TMA persistent GEMM (see gemm_tc.cuh for the contract).
//
// CTA = 384 threads = 3 warpgroups, one CTA per SM, persistent over output tiles (128 x BN):
//   warpgroup 0   : TMA producer (warp 0, one elected lane)   global -> 128B-swizzled smem ring of 3 stages of
//                   48 KB at BN = 256 (5 of 32 KB at BN = 128)
//   warpgroups 1-2: consumers; warpgroup 1 + c computes columns [c BN/2, (c+1) BN/2) of the tile with
//                   wgmma m64 x (BN/2) x k16 (fp32 accumulators in registers), then runs the fused epilogue
//                   (gemm_epilogue.cuh) on them.
// Each consumer issues its 128 rows as two m64 wgmmas whose A descriptors interleave the 8-row swizzle atoms
// (start +0 / +1024 B, stride 2048 B): warp w of the warpgroup then holds the 32 CONSECUTIVE rows 32w..32w+31,
// the row block the epilogue works on.
//
// block_n 512: a cluster of two CTAs computes a 256 x 256 tile.  Each CTA stages its own 128 rows of A and
// loads half of the 256-row weight tile, multicast into both CTAs, so the weight traffic from L2 per CTA
// halves.  A smem stage is refilled only once the consumers of BOTH CTAs have released it.
//
// A consumer warpgroup releases a stage once the wgmma_wait after the next k block's issue shows the stage's
// wgmmas complete.  The release is a plain mbarrier arrive on its own CTA's barrier and a remote arrive on the
// peer's, with no memory fence: a .release.cluster arrive compiles to a CTA- and a GPU-scope MEMBAR, which also
// waits for the releasing lane's outstanding epilogue stores, and the whole warpgroup waits for that lane.
#include "gemm_tc.cuh"
#include "gemm_epilogue.cuh"

namespace mhmr {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 fp16 = 128 B = one swizzle row
constexpr int kConsumers = 2;
constexpr int kThreads = 128 * (1 + kConsumers);
constexpr int kEpiWarps = 4 * kConsumers;
constexpr int kRegsProducer = 40, kRegsConsumer = 232;

template <int BN>
struct GemmCfg {
  static constexpr int kStages = (BN == 256) ? 3 : 5;
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarBytes = 256;
  static constexpr int kSmemBytes =
      kStages * kStageBytes + kEpiWarps * kScratchBytes + kBarBytes + 1024;  // +1024: manual align
  static constexpr int kAcc = BN / 4;  // fp32 accumulators per thread and m64 wgmma (n = BN / 2)
};

template <int NACC>
__device__ __forceinline__ void wgmma_ss(float (&d)[NACC], uint64_t da, uint64_t db, uint32_t acc) {
  if constexpr (NACC == 64) wgmma_m64n128_ss(d, da, db, acc);
  else wgmma_m64n64_ss(d, da, db, acc);
}

template <int BN, int CL, int EPI>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               int M, int N, int K, GemmEpi ep) {
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kAcc = Cfg::kAcc;

  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (128B swizzle atoms) by POINTER arithmetic, so that the compiler keeps the
  // shared address space (a round trip through uintptr_t degrades every access to generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* scratch_base = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes + kEpiWarps * kScratchBytes);
  uint64_t* full_bar = bars;             // [kStages]  TMA -> consumers
  uint64_t* empty_bar = bars + kStages;  // [kStages]  consumers (of every CTA of the cluster) -> TMA

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const uint32_t rank = (CL > 1) ? cluster_ctarank() : 0u;

  const int num_m = (M + BM * CL - 1) / (BM * CL);
  const int num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (K + BK - 1) / BK;
  const int first_tile = blockIdx.x / CL, tile_stride = gridDim.x / CL;

  griddep_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumers * CL);  // one arrive per consumer warpgroup of every CTA
    }
    fence_barrier_init();
  }
  if constexpr (CL > 1) cluster_sync_all();  // the peer's barriers exist before any multicast or remote arrive
  else __syncthreads();
  griddep_wait();  // the previous kernel's outputs (A rows, residual, statistics) are complete and visible

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegsProducer));
    if (warp == 0) {
      // ------------------------------ TMA producer ------------------------------
      uint32_t stage = 0, phase = 0;
      for (int tile = first_tile; tile < num_tiles; tile += tile_stride) {
        const int m_blk = tile / num_n, n_blk = tile % num_n;
        const int row0 = m_blk * BM * CL + static_cast<int>(rank) * BM;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          if (elect_one_sync()) {
            mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
            tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, row0);
            if constexpr (CL > 1) {
              constexpr int kHalf = BN / CL;
              tma_load_2d_multicast(sb + rank * (kHalf * BK * 2), &tmB, &full_bar[stage], kb * BK,
                                    n_blk * BN + static_cast<int>(rank) * kHalf, static_cast<uint16_t>((1u << CL) - 1u));
            } else {
              tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n_blk * BN);
            }
          }
          __syncwarp();
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegsConsumer));
    // ------------------------------ consumers -----------------------------------
    const int cw = wg - 1;          // column half of the tile
    const int w = warp & 3;         // rows 32w..32w+31 of the tile
    const bool release_lane = (threadIdx.x & 127) == 0;
    float* scratch = scratch_base + (warp - 4) * (kScratchBytes / 4);
    // Frees stage s in every CTA of the cluster.  No fence: this warpgroup's wgmma reads of the stage are
    // complete at the wgmma_wait that precedes every release, and the refill is a TMA (async-proxy) write that
    // the producer issues only after its empty_bar wait has observed the arrives.
    auto release = [&](uint32_t s) {
      if (release_lane) {
        mbar_arrive(&empty_bar[s]);
        if constexpr (CL > 1) {
#pragma unroll
          for (int c = 0; c < CL; ++c)
            if (c != static_cast<int>(rank)) mbar_arrive_remote(&empty_bar[s], static_cast<uint32_t>(c));
        }
      }
    };
    uint32_t stage = 0, phase = 0;
    EpiStatsPrefetch pf;
    auto tile_m_base = [&](int tile) { return (tile / num_n) * BM * CL + static_cast<int>(rank) * BM + 32 * w; };
    if (first_tile < num_tiles) epilogue_load_row_stats<EPI>(pf, ep, M, tile_m_base(first_tile), lane);
    for (int tile = first_tile; tile < num_tiles; tile += tile_stride) {
      const int n_blk = tile % num_n;
      const int m_base = tile_m_base(tile);
      EpiRowState rowst;
      epilogue_tile_begin<EPI>(rowst, pf, ep, K);
      if (tile + tile_stride < num_tiles)  // next tile's row statistics: under this tile's main loop
        epilogue_load_row_stats<EPI>(pf, ep, M, tile_m_base(tile + tile_stride), lane);

      float acc[2][kAcc];
      uint32_t prev_stage = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
        const uint32_t sb = sa + Cfg::kABytes + cw * (BN / 2) * (BK * 2);
        const uint64_t a_desc0 = make_sw128_desc(sa, 16, 2048);
        const uint64_t a_desc1 = make_sw128_desc(sa + 1024, 16, 2048);
        const uint64_t b_desc = make_sw128_desc(sb, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // advance K by 16 fp16 = 32 B inside the 128-B swizzle row: +2 in (addr >> 4) units
          const uint32_t accumulate = (kb > 0 || k > 0) ? 1u : 0u;
          wgmma_ss<kAcc>(acc[0], a_desc0 + 2u * k, b_desc + 2u * k, accumulate);
          wgmma_ss<kAcc>(acc[1], a_desc1 + 2u * k, b_desc + 2u * k, accumulate);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k block's wgmmas are complete: its stage can be refilled
        if (kb > 0) release(prev_stage);
        prev_stage = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
      release(prev_stage);

      // ------------------------------ epilogue ----------------------------------
      // accumulator fragment of wgmma h: register i holds row 8h + 16((i >> 1) & 1) + lane / 4 of this warp's
      // block, column 8 (i >> 2) + 2 (lane & 3) + (i & 1) of the warpgroup's half
#pragma unroll
      for (int c = 0; c < BN / 64; ++c) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
              const int i = 4 * (4 * c + g) + 2 * rr;
              const int r = (lane >> 2) + 8 * h + 16 * rr;
              *reinterpret_cast<float2*>(scratch + r * kScratchStride + g * 8 + 2 * (lane & 3)) =
                  make_float2(acc[h][i], acc[h][i + 1]);
            }
        __syncwarp();
        const int n0 = n_blk * BN + cw * (BN / 2) + c * 32;
        if (n0 < N) epilogue_chunk<EPI>(scratch, ep, M, N, m_base, n0, lane, rowst);
        __syncwarp();
      }
      epilogue_tile_end<EPI>(rowst, ep, M, m_base, n_blk * kConsumers + cw, lane);
    }
  }
  // no CTA of a cluster leaves while its peer may still arrive on its barriers
  if constexpr (CL > 1) cluster_sync_all();
}

template <int BN, int CL, int EPI>
int launch_one(const GemmPlan* p, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_tc_kernel<BN, CL, EPI>;
  static PerDeviceOnce once;
  if (once.first()) {
    MHMR_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes));
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(p->grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (CL > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = CL;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  MHMR_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, p->tmA, p->tmB, p->M, p->N, p->K, p->ep));
  return MHMR_OK;
}

template <int BN, int CL>
int launch_bn(const GemmPlan* p, cudaStream_t stream) {
  switch (p->epi) {
    case EPI_BIAS_F16: return launch_one<BN, CL, EPI_BIAS_F16>(p, stream);
    case EPI_BIAS_GELU_F16: return launch_one<BN, CL, EPI_BIAS_GELU_F16>(p, stream);
    case EPI_BIAS_RELU_F16: return launch_one<BN, CL, EPI_BIAS_RELU_F16>(p, stream);
    case EPI_LS_RESID_F32: return launch_one<BN, CL, EPI_LS_RESID_F32>(p, stream);
    case EPI_ROWADD_F32: return launch_one<BN, CL, EPI_ROWADD_F32>(p, stream);
    case EPI_BIAS_F32: return launch_one<BN, CL, EPI_BIAS_F32>(p, stream);
    case EPI_LS_RESID_SPLIT: return launch_one<BN, CL, EPI_LS_RESID_SPLIT>(p, stream);
    case EPI_LN_BIAS_F16: return launch_one<BN, CL, EPI_LN_BIAS_F16>(p, stream);
    case EPI_LN_GELU_F16: return launch_one<BN, CL, EPI_LN_GELU_F16>(p, stream);
    case EPI_ROWADD_F16: return launch_one<BN, CL, EPI_ROWADD_F16>(p, stream);
    default: break;
  }
  set_last_error("gemm: unknown epilogue kind");
  return MHMR_ERR_ARG;
}

}  // namespace

int gemm_plan_init(GemmPlan* plan, const __half* A, int64_t lda, const __half* W, int64_t ldw, int M,
                   int N, int K, int epi_kind, const GemmEpi& ep, int bn) {
  MHMR_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem");
  MHMR_REQUIRE(N % 32 == 0, "gemm: N must be a multiple of 32");
  MHMR_REQUIRE(lda % 8 == 0 && ldw % 8 == 0, "gemm: row pitches must be multiples of 8 fp16 (16 B, TMA)");
  MHMR_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
               "gemm: operands must be 16-byte aligned");
  MHMR_REQUIRE(bn == 128 || bn == 256 || bn == 512, "gemm: block_n must be 128, 256 or 512 (CTA pair)");
  MHMR_REQUIRE(epi_kind >= 0 && epi_kind < EPI_NUM_KINDS, "gemm: bad epilogue kind");
  if (epi_kind != EPI_LS_RESID_SPLIT)
    MHMR_REQUIRE(ep.out != nullptr && ep.ldo % 8 == 0, "gemm: output missing or pitch not multiple of 8");
  if (epi_kind != EPI_BIAS_F32 && epi_kind != EPI_ROWADD_F32 && epi_kind != EPI_ROWADD_F16)
    MHMR_REQUIRE(ep.bias != nullptr, "gemm: bias required for this epilogue");
  if (epi_kind == EPI_LS_RESID_F32 || epi_kind == EPI_LS_RESID_SPLIT)
    MHMR_REQUIRE(ep.gamma != nullptr, "gemm: gamma required");
  if (epi_kind == EPI_LS_RESID_SPLIT)
    MHMR_REQUIRE(ep.x16 != nullptr && ep.xlo != nullptr && ep.ldx16 % 8 == 0 && ep.stats != nullptr &&
                     ep.stat_slots == gemm_stat_slots(N, bn) && N % (bn == 128 ? 128 : 256) == 0,
                 "gemm: split-stream epilogue needs both planes, stats, whole column tiles and matching slot count");
  if (epi_kind == EPI_LN_BIAS_F16 || epi_kind == EPI_LN_GELU_F16)
    MHMR_REQUIRE(ep.stats != nullptr && ep.stat_slots > 0 && ep.stat_slots % 2 == 0 && ep.stat_slots <= 8,
                 "gemm: folded-LN consumer needs row statistics (even slot count, at most 8)");
  if (epi_kind == EPI_ROWADD_F32 || epi_kind == EPI_ROWADD_F16)
    MHMR_REQUIRE(ep.rowadd != nullptr && ep.rows_in > 0, "gemm: rowadd/rows_in required");
  plan->M = M; plan->N = N; plan->K = K; plan->bn = bn; plan->epi = epi_kind; plan->ep = ep;
  int rc = make_tmap_2d(&plan->tmA, A, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, M, K, lda * 2, BM, BK, true);
  if (rc != MHMR_OK) return rc;
  // CTA pair: every CTA loads half (128 rows) of the 256-row weight tile
  rc = make_tmap_2d(&plan->tmB, W, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, N, K, ldw * 2, bn == 512 ? 128 : bn, BK,
                    true);
  if (rc != MHMR_OK) return rc;
  plan->grid = gemm_plan_grid(plan, M);
  return MHMR_OK;
}

int gemm_plan_grid(const GemmPlan* plan, int M) {
  const int sms = device_sm_count();
  if (plan->bn == 512) {
    const int tiles = ((M + 255) / 256) * ((plan->N + 255) / 256);
    const int pairs = sms / 2;
    return 2 * (tiles < pairs ? tiles : pairs);
  }
  const int tiles = ((M + BM - 1) / BM) * ((plan->N + plan->bn - 1) / plan->bn);
  return tiles < sms ? tiles : sms;
}

int gemm_stat_slots(int N, int bn) {
  const int tile_n = (bn == 128) ? 128 : 256;  // bn 512 = CTA pair with 256-column tiles
  return ((N + tile_n - 1) / tile_n) * kConsumers;
}

int gemm_plan_run(const GemmPlan* plan, cudaStream_t stream) {
  if (plan->bn == 512) return launch_bn<256, 2>(plan, stream);
  return plan->bn == 256 ? launch_bn<256, 1>(plan, stream) : launch_bn<128, 1>(plan, stream);
}

int gemm_plan_run_rows(const GemmPlan* plan, int M, cudaStream_t stream) {
  MHMR_REQUIRE(M > 0 && M <= plan->M, "gemm: a plan runs at most the rows it was built for");
  GemmPlan p = *plan;  // the tensor map of A still spans plan->M rows; the kernel stores only rows below p.M
  p.M = M;
  p.grid = gemm_plan_grid(&p, M);
  return gemm_plan_run(&p, stream);
}

}  // namespace mhmr
