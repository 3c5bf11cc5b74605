// Central-stream refinement (DESIGN.md §3): the residual streams of the detected tokens recomputed in fp32.
//
//   x = W_patch . pixels + (pos + bias)                                   (refine_prepare + one skinny linear, head.cu)
//   per block l:  x += ls1_l * (W_proj_l . O16_l[row] + b_proj_l)         (A)  depends on the bulk pass only
//                 x += ls2_l * (W_fc2_l . gelu(W_fc1_l . LN2_l(x) + b_fc1_l) + b_fc2_l)        (B)
// Same arithmetic as dinov2 Block.forward (reached from reference blocks/dinov2.py:25) for the few rows that the
// per-person outputs are sensitive to.
//
// x and h are written and re-read across grid barriers by different SMs: the rows are staged into shared memory by bulk
// copies (async proxy, L2) and single elements are read with ld.global.cg, never through the (incoherent) L1.
//
// The first version launched three skinny linears per block: 74 dependent launches of ~20 us (latency chains, not
// bandwidth: 2.1 ms of a 39.5 ms step).  Here
//   * every term (A) is computed up front by ONE batched launch (blockIdx.z = block): they only need the attention
//     outputs O16_l of the bulk pass, not x;
//   * the chain (B) of all blocks runs in ONE persistent cooperative kernel: each CTA owns a fixed slice of the fc1 /
//     fc2 output columns, stages the (few) person rows in shared memory, and a grid barrier separates the two phases
//     of a block; the next phase's weight slice is pulled into L2 before the barrier.  Column ownership is fixed, so
//     the result does not depend on scheduling (bit-reproducible).
#include "kernels.cuh"

namespace mhmr {

namespace {

constexpr int kPT = 8;       // persons per pass
constexpr int kKT = 1024;    // K tile staged per person (floats)

__device__ __forceinline__ void prefetch_l2_rows(const float* W, int64_t ldw, int n0, int ncols, int Nout, int Kp, int warp,
                                                 int lane) {
  for (int c = warp; c < ncols; c += 8) {
    const int n = n0 + c;
    if (n >= Nout) break;
    const char* wr = reinterpret_cast<const char*>(W + static_cast<int64_t>(n) * ldw);
    for (int b = lane * 128; b < Kp * 4; b += 32 * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(wr + b));
  }
}

// Butterfly reduction of NV = CPW * 8 values per lane: lane L ends with the total of value (L mod NV) in a[0].
template <int NV>
__device__ __forceinline__ void butterfly(float (&a)[NV], int lane) {
  if constexpr (NV < 32) {
#pragma unroll
    for (int o = 16; o >= NV; o >>= 1)
#pragma unroll
      for (int i = 0; i < NV; ++i) a[i] += __shfl_xor_sync(0xffffffffu, a[i], o);
  }
#pragma unroll
  for (int o = (NV < 32 ? NV / 2 : 16); o >= 1; o >>= 1) {
    const bool up = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < o; ++i) {
      const float send = up ? a[i] : a[i + o];
      const float keep = up ? a[i + o] : a[i];
      a[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
}

// acc[c][j] += W[n_base + c, k0 : k0 + kt] . xs[j][0 : kt]   for this warp's CPW columns and the 8 staged rows
template <int CPW>
__device__ __forceinline__ void tile_dot(const float* __restrict__ W, int64_t ldw, int n_base, int Nout, int k0, int kt,
                                         const float (*xs)[kKT], int lane, float (&acc)[CPW][kPT]) {
  for (int k = lane * 4; k < kt; k += 128) {
    float4 w4[CPW];
#pragma unroll
    for (int c = 0; c < CPW; ++c) {
      const int n = min(n_base + c, Nout - 1);
      w4[c] = __ldg(reinterpret_cast<const float4*>(W + static_cast<int64_t>(n) * ldw + k0 + k));
    }
#pragma unroll
    for (int j = 0; j < kPT; ++j) {
      const float4 x4 = *reinterpret_cast<const float4*>(&xs[j][k]);
#pragma unroll
      for (int c = 0; c < CPW; ++c) acc[c][j] += w4[c].x * x4.x + w4[c].y * x4.y + w4[c].z * x4.z + w4[c].w * x4.w;
    }
  }
}

// ---- (A) all projection terms at once: term[l][p][n] = ls1_l[n] * (W_proj_l[n, :] . O16_l[row_p, :] + b_proj_l[n])
__global__ void __launch_bounds__(256)
refine_proj_terms_kernel(const RefineLayer* __restrict__ layers, const int* __restrict__ rowidx,
                         const int* __restrict__ count, int D, int max_persons, float* __restrict__ term) {
  __shared__ __align__(16) float xs[kPT][kKT];
  constexpr int CPW = 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const RefineLayer L = layers[blockIdx.z];
  const int n_base = blockIdx.x * (8 * CPW) + warp * CPW;
  griddep_launch_dependents();
  if (blockIdx.y == 0) prefetch_l2_rows(L.Wproj, D, blockIdx.x * 8 * CPW, 8 * CPW, D, D, warp, lane);
  griddep_wait();
  const int P = *count;
  const int p0 = blockIdx.y * kPT;
  if (p0 >= P) return;
  const int np = min(kPT, P - p0);
  float acc[CPW][kPT];
#pragma unroll
  for (int c = 0; c < CPW; ++c)
#pragma unroll
    for (int j = 0; j < kPT; ++j) acc[c][j] = 0.f;
  for (int k0 = 0; k0 < D; k0 += kKT) {
    const int kt = min(kKT, D - k0), q4 = kt >> 2;
    for (int idx = threadIdx.x; idx < kPT * q4; idx += 256) {
      const int j = idx / q4, q = idx - j * q4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j < np) {
        const uint2 pk = *reinterpret_cast<const uint2*>(L.O16 + static_cast<int64_t>(rowidx[p0 + j]) * D + k0 + 4 * q);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&pk.x));
        const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&pk.y));
        v = make_float4(a.x, a.y, b.x, b.y);
      }
      *reinterpret_cast<float4*>(&xs[j][4 * q]) = v;
    }
    __syncthreads();
    tile_dot<CPW>(L.Wproj, D, n_base, D, k0, kt, xs, lane, acc);
    __syncthreads();
  }
  float a[CPW * kPT];
#pragma unroll
  for (int c = 0; c < CPW; ++c)
#pragma unroll
    for (int j = 0; j < kPT; ++j) a[c * kPT + j] = acc[c][j];
  butterfly<CPW * kPT>(a, lane);
  const int vi = lane & (CPW * kPT - 1), c = vi / kPT, j = vi - c * kPT, n = n_base + c;
  if (lane < CPW * kPT && j < np && n < D)
    term[(static_cast<int64_t>(blockIdx.z) * max_persons + p0 + j) * D + n] = L.ls1[n] * (a[0] + L.bproj[n]);
}

// ---- (B) the MLP chain of every block in one persistent cooperative kernel
__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned int spins = 0;
    while (*reinterpret_cast<volatile unsigned int*>(counter) < target) {
      if (++spins > (1u << 30)) __trap();  // a protocol bug must surface as an error, never as a hung GPU
    }
    __threadfence();
  }
  __syncthreads();
}

// One linear layer phase for the 8 staged rows xs[8][K]: this CTA's columns [n0, n0 + 4 * ngroups), K split across the
// 8 warps (each warp a contiguous K slice, every lane 4 consecutive k per 128-wide step), 4 columns at a time; the
// per-warp partial sums go through shared memory (red[warp][group * 32 + lane]) and are added up by one thread per
// (column, person).  Many independent weight loads in flight per lane, one pass over the staged rows per group.
// 16 warps = 2 teams x 8 K-slices; team u takes the column groups u, u + 2, ...
constexpr int kChainThreads = 512;

template <typename Epi>
__device__ __forceinline__ void cta_linear(const float* __restrict__ W, int64_t ldw, int Nout, int K, int n0, int ngroups,
                                           const float* xs, int ldxs, float* red, int warp, int lane, Epi epi) {
  const int slice = ((K + 31) / 32) * 4;          // K slice of a warp: a multiple of 4, 8 slices cover K
  const int kw = warp & 7, team = warp >> 3;
  const int kbeg = kw * slice, kend = min(K, kbeg + slice);
  for (int g = team; g < ngroups; g += kChainThreads / 256) {
    const int n_base = n0 + 4 * g;
    float acc[4][kPT];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int j = 0; j < kPT; ++j) acc[c][j] = 0.f;
    for (int k = kbeg + lane * 4; k < kend; k += 128) {
      float4 w4[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int n = min(n_base + c, Nout - 1);
        w4[c] = __ldg(reinterpret_cast<const float4*>(W + static_cast<int64_t>(n) * ldw + k));
      }
#pragma unroll
      for (int j = 0; j < kPT; ++j) {
        const float4 x4 = *reinterpret_cast<const float4*>(xs + j * ldxs + k);
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[c][j] += w4[c].x * x4.x + w4[c].y * x4.y + w4[c].z * x4.z + w4[c].w * x4.w;
      }
    }
    float a[4 * kPT];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int j = 0; j < kPT; ++j) a[c * kPT + j] = acc[c][j];
    butterfly<4 * kPT>(a, lane);
    red[kw * 256 + g * 32 + lane] = a[0];     // value index lane = (column c = lane / 8, person j = lane % 8)
  }
  __syncthreads();
  const int t = threadIdx.x;
  if (t < ngroups * 32) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += red[w * 256 + t];
    const int g = t >> 5, c = (t & 31) / kPT, j = t & (kPT - 1);
    const int n = n0 + 4 * g + c;
    if (n < Nout) epi(n, j, v);
  }
  fence_proxy_async_smem();   // this CTA's generic-proxy writes of the staged rows precede the next bulk copy into them
  __syncthreads();
}

// Row staging of the chain: every CTA needs ALL staged rows (8 x D for fc1, 8 x 4D for fc2).  One thread fetches them
// with bulk copies (one round trip, no load instructions; per-thread ld.global.cg loops cost 6 k of the 42 k clk of a
// block at 8 persons, `tools/gpu_trace_chain.sh`).  Caller: after a __syncthreads that follows the last read of `dst`
// and, when `src` was written by other CTAs of this launch, after the grid barrier.
__device__ __forceinline__ void bulk_rows(float* dst, const float* src, uint32_t bytes, uint64_t* bar) {
  for (uint32_t off = 0; off < bytes; off += 32768u) {
    const uint32_t n = min(32768u, bytes - off);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(reinterpret_cast<char*>(dst) + off)),
                 "l"(reinterpret_cast<const char*>(src) + off), "r"(n), "r"(smem_u32(bar))
                 : "memory");
  }
}

// ---- (B) the MLP chain of every block in one persistent cooperative kernel
__global__ void __launch_bounds__(kChainThreads)
refine_mlp_chain_kernel(const RefineLayer* __restrict__ layers, int depth, const int* __restrict__ count, int D,
                        int max_persons, const float* __restrict__ term, float* x, float* h, unsigned int* barrier) {
  extern __shared__ __align__(16) float dyn[];
  const int H = 4 * D;
  float* xs = dyn;                 // [8][H] (phase 2) / [8][D] (phase 1)
  float* red = dyn + kPT * H;      // [8 warps][256]
  __shared__ float stats[kPT][2];
  __shared__ __align__(8) uint64_t rbar;   // staged rows have landed
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = gridDim.x;
  uint32_t rpar = 0;
  if (threadIdx.x == 0) {
    mbar_init(&rbar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  // fixed column ownership: fc1 (4D outputs) in slices of 32 per CTA, fc2 (D outputs) in slices of 8 per CTA,
  // both strided over the grid
  const int P = *count;
  unsigned int phase = 0;
  for (int l = 0; l < depth; ++l) {
    const RefineLayer L = layers[l];
    const float* tl = term + static_cast<int64_t>(l) * max_persons * D;
    // ---------------- phase 1: h = gelu(W_fc1 . LN2(x + term_l) + b_fc1)
    for (int p0 = 0; p0 < P; p0 += kPT) {
      const int np = min(kPT, P - p0);
      // raw rows x and term_l: two bulk fetches into xs[0 : 8D) and xs[8D : 16D), summed in place
      if (threadIdx.x == 0) {
        // x was written through the generic proxy by other CTAs; xs by this CTA's threads (fenced below)
        asm volatile("fence.proxy.async;" ::: "memory");
        const uint32_t rb = static_cast<uint32_t>(np) * D * 4u;
        mbar_arrive_expect_tx(&rbar, 2u * rb);
        bulk_rows(xs, x + static_cast<int64_t>(p0) * D, rb, &rbar);
        bulk_rows(xs + kPT * D, tl + static_cast<int64_t>(p0) * D, rb, &rbar);
      }
      mbar_wait(&rbar, rpar);
      rpar ^= 1u;
      for (int idx = threadIdx.x; idx < kPT * (D >> 2); idx += kChainThreads) {
        const int j = idx / (D >> 2), k = 4 * (idx - j * (D >> 2));
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (j < np) {
          const float4 a = *reinterpret_cast<const float4*>(xs + j * D + k);
          const float4 t = *reinterpret_cast<const float4*>(xs + (kPT + j) * D + k);
          v = make_float4(a.x + t.x, a.y + t.y, a.z + t.z, a.w + t.w);
        }
        *reinterpret_cast<float4*>(xs + j * D + k) = v;
      }
      __syncthreads();
      if (warp < np) {  // LayerNorm statistics (eps 1e-6) of row `warp`, two passes over shared memory
        const float* r = xs + warp * D;
        float s = 0.f;
        for (int k = lane; k < D; k += 32) s += r[k];
        const float mean = warp_sum(s) / D;
        float q = 0.f;
        for (int k = lane; k < D; k += 32) { const float d = r[k] - mean; q += d * d; }
        const float rstd = rsqrtf(warp_sum(q) / D + 1e-6f);
        if (lane == 0) { stats[warp][0] = mean; stats[warp][1] = rstd; }
      }
      __syncthreads();
      for (int idx = threadIdx.x; idx < np * (D >> 2); idx += kChainThreads) {    // normalise in place
        const int j = idx / (D >> 2), k = 4 * (idx - j * (D >> 2));
        float4 v = *reinterpret_cast<float4*>(xs + j * D + k);
        const float4 g = __ldg(reinterpret_cast<const float4*>(L.ln2_g + k));
        const float4 b = __ldg(reinterpret_cast<const float4*>(L.ln2_b + k));
        const float mean = stats[j][0], rstd = stats[j][1];
        v.x = (v.x - mean) * rstd * g.x + b.x;
        v.y = (v.y - mean) * rstd * g.y + b.y;
        v.z = (v.z - mean) * rstd * g.z + b.z;
        v.w = (v.w - mean) * rstd * g.w + b.w;
        *reinterpret_cast<float4*>(xs + j * D + k) = v;
      }
      __syncthreads();
      for (int cb = blockIdx.x; cb * 32 < H; cb += G) {
        const int ngroups = min(8, (H - cb * 32 + 3) / 4);
        cta_linear(L.Wfc1, D, H, D, cb * 32, ngroups, xs, D, red, warp, lane, [&](int n, int j, float v) {
          if (j < np) h[static_cast<int64_t>(p0 + j) * H + n] = gelu_erf(v + L.bfc1[n]);
        });
      }
    }
    for (int cb = blockIdx.x; cb * 8 < D; cb += G) prefetch_l2_rows(L.Wfc2, H, cb * 8, 8, D, H, warp, lane);
    grid_barrier(barrier, ++phase * G);
    // ---------------- phase 2: x = (x + term_l) + ls2 * (W_fc2 . h + b_fc2)
    for (int p0 = 0; p0 < P; p0 += kPT) {
      const int np = min(kPT, P - p0);
      if (threadIdx.x == 0) {
        asm volatile("fence.proxy.async;" ::: "memory");   // h was written through the generic proxy by other CTAs
        const uint32_t rb = static_cast<uint32_t>(np) * H * 4u;
        mbar_arrive_expect_tx(&rbar, rb);
        bulk_rows(xs, h + static_cast<int64_t>(p0) * H, rb, &rbar);
      }
      if (np < kPT)   // rows beyond the last person: zeros (generic proxy, disjoint from the copy)
        for (int idx = threadIdx.x + np * (H >> 2); idx < kPT * (H >> 2); idx += kChainThreads)
          *reinterpret_cast<float4*>(xs + 4 * idx) = make_float4(0.f, 0.f, 0.f, 0.f);
      mbar_wait(&rbar, rpar);
      rpar ^= 1u;
      if (np < kPT) __syncthreads();
      for (int cb = blockIdx.x; cb * 8 < D; cb += G) {
        const int ngroups = min(2, (D - cb * 8 + 3) / 4);
        cta_linear(L.Wfc2, H, D, H, cb * 8, ngroups, xs, H, red, warp, lane, [&](int n, int j, float v) {
          if (j < np) {
            const int64_t o = static_cast<int64_t>(p0 + j) * D + n;
            x[o] = (__ldcg(x + o) + tl[o]) + L.ls2[n] * (v + L.bfc2[n]);
          }
        });
      }
    }
    if (l + 1 < depth) {
      const RefineLayer Ln = layers[l + 1];
      for (int cb = blockIdx.x; cb * 32 < H; cb += G) prefetch_l2_rows(Ln.Wfc1, D, cb * 32, 32, H, D, warp, lane);
    }
    grid_barrier(barrier, ++phase * G);
  }
}

}  // namespace

int refine_proj_terms(const RefineLayer* layers, int depth, const int* rowidx, const int* count, int D,
                      int max_persons, float* term, cudaStream_t st) {
  MHMR_REQUIRE(D % 4 == 0, "refine: D must be a multiple of 4");
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((D + 15) / 16, (max_persons + kPT - 1) / kPT, depth);
  cfg.blockDim = dim3(256);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  MHMR_CUDA_CHECK(cudaLaunchKernelEx(&cfg, refine_proj_terms_kernel, layers, rowidx, count, D, max_persons, term));
  return MHMR_OK;
}

int refine_mlp_chain(const RefineLayer* layers, int depth, const int* count, int D, int max_persons, const float* term,
                     float* x, float* h, unsigned int* barrier, cudaStream_t st) {
  MHMR_REQUIRE(D % 4 == 0, "refine: D must be a multiple of 4");
  MHMR_CUDA_CHECK(cudaMemsetAsync(barrier, 0, sizeof(unsigned int), st));
  // one CTA per 32 fc1 columns, at most one per SM: every CTA is resident (cooperative launch), so the grid barrier
  // cannot deadlock
  int grid = (4 * D + 31) / 32;
  if (grid > device_sm_count()) grid = device_sm_count();
  const int smem = (kPT * 4 * D + 8 * 256) * static_cast<int>(sizeof(float));
  MHMR_REQUIRE(smem <= 200 * 1024, "refine: embed dim too large for the staged hidden rows");
  static PerDeviceOnce once;
  if (once.first()) {
    MHMR_CUDA_CHECK(cudaFuncSetAttribute(refine_mlp_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }
  void* args[] = {(void*)&layers, (void*)&depth, (void*)&count, (void*)&D, (void*)&max_persons,
                  (void*)&term,   (void*)&x,     (void*)&h,     (void*)&barrier};
  MHMR_CUDA_CHECK(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(refine_mlp_chain_kernel), dim3(grid),
                                              dim3(kChainThreads), args, smem, st));
  return MHMR_OK;
}

}  // namespace mhmr
