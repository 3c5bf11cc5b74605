// Shared device/host helpers for the sm_90a kernels of the Multi-HMR hot path.
//
// Everything here is a thin inline-PTX wrapper (mbarrier, TMA, clusters, wgmma) or a
// host-side utility (error reporting, tensor-map encoding through the driver entry
// point so the library has no link-time dependency on libcuda).
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>

#include "../../include/mhmr.h"

namespace mhmr {

// Programmatic dependent launch (PDL).  Every kernel of the chain lets the next grid start its prologue
// (barrier init, descriptor prefetch) while this grid drains, and waits for the full
// completion (and memory visibility) of the previous grid before it touches global memory.  Both are no-ops
// when the kernel was launched without the programmatic-serialization attribute.
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }


// ----------------------------------------------------------------------------------
// Host-side error plumbing: every C-ABI entry returns an int (0 ok, <0 error) and
// leaves a message retrievable through mhmr_last_error().
// ----------------------------------------------------------------------------------
void set_last_error(const std::string& msg);
const char* get_last_error();

#define MHMR_CUDA_CHECK(expr)                                                          \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      ::mhmr::set_last_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + \
                             " at " + __FILE__ + ":" + std::to_string(__LINE__));      \
      return MHMR_ERR_CUDA;                                                    \
    }                                                                                  \
  } while (0)

#define MHMR_REQUIRE(cond, msg)                                                        \
  do {                                                                                 \
    if (!(cond)) {                                                                     \
      ::mhmr::set_last_error(std::string("requirement failed: ") + #cond + " — " + msg); \
      return MHMR_ERR_ARG;                                                     \
    }                                                                                  \
  } while (0)

// Propagates a failed status (variadic: the expression may hold template commas).
#define TRY(...)                    \
  do {                              \
    int rc_ = (__VA_ARGS__);        \
    if (rc_ != MHMR_OK) return rc_; \
  } while (0)

// Encode a 2-D row-major tensor map: `rows` x `cols` elements of `elem_bytes`, row pitch
// `pitch_bytes`; the box is box_rows x box_cols. `swizzle128` selects the 128-byte
// swizzle (box_cols*elem_bytes must then be 128).
int make_tmap_2d(CUtensorMap* out, const void* gptr, CUtensorMapDataType dtype, int elem_bytes,
                 uint64_t rows, uint64_t cols, uint64_t pitch_bytes, uint32_t box_rows,
                 uint32_t box_cols, bool swizzle128);
// The same over a stack of `depth` such matrices, `depth_pitch_bytes` apart; the box is box_rows x box_cols of one
// matrix, so a box that crosses the last row is zero-filled instead of reading the next matrix.
int make_tmap_3d(CUtensorMap* out, const void* gptr, CUtensorMapDataType dtype, int elem_bytes,
                 uint64_t depth, uint64_t rows, uint64_t cols, uint64_t depth_pitch_bytes, uint64_t pitch_bytes,
                 uint32_t box_rows, uint32_t box_cols, bool swizzle128);

int device_sm_count();
// Function attributes (cudaFuncSetAttribute) and the SM count are per DEVICE: `first()` is true the first time
// it is asked on the current device, so that a process with engines on several GPUs configures each of them.
struct PerDeviceOnce {
  bool done[64] = {};
  bool first();
};
// Programmatic dependent launch for the back-to-back kernels of the ViT loop (MHMR_PDL=0 disables).
bool pdl_enabled();

inline size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

// Device memory of one C-ABI call: regions laid out on the host at 256-byte alignment, the staged ones before every
// device-only one, in one stream-ordered allocation on the call's stream.  The staged regions' host bytes, filled by
// the caller (after allocate() when they hold device addresses inside the scratch), go up in one cudaMemcpyAsync from
// pageable memory, which returns once the driver has read them.  The scratch is freed stream-ordered on the same
// stream on every return path: by release() on success, by the destructor on an error return.
class CallScratch {
 public:
  explicit CallScratch(cudaStream_t st) : st_(st) {}
  ~CallScratch();
  CallScratch(const CallScratch&) = delete;
  CallScratch& operator=(const CallScratch&) = delete;
  // Handle of a new region of `bytes` (0 allowed); a staged region is uploaded by upload().
  size_t region(size_t bytes, bool staged = false);
  int allocate();  // the whole layout (at least 256 bytes)
  // Device address of a region, valid after allocate().
  template <class T>
  T* dev(size_t r) const {
    return reinterpret_cast<T*>(base_ + regions_[r].off + (regions_[r].staged ? 0 : staged_bytes_));
  }
  // Host bytes of a staged region (zero-filled); a later staged region() call may move them.
  template <class T>
  T* host(size_t r) {
    return reinterpret_cast<T*>(blob_.data() + regions_[r].off);
  }
  int upload();
  int release();  // frees now, returning the status of the free

 private:
  struct Region {
    size_t off;
    bool staged;
  };
  cudaStream_t st_;
  uint8_t* base_ = nullptr;
  std::vector<Region> regions_;
  std::vector<uint8_t> blob_;  // the staged regions' host bytes
  size_t staged_bytes_ = 0, device_bytes_ = 0;
};

#ifdef __CUDACC__
// ----------------------------------------------------------------------------------
// Device helpers
// ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }
// One leader lane of a fully active warp (the same lane every time).  Issue loops (TMA) run
// with the WHOLE warp on warp-uniform control flow and guard only the issuing instructions with this
// predicate: their descriptors then live in uniform registers.
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, %1;\n\t"
      "selp.u32 %0, 1, 0, px;\n\t}"
      : "=r"(pred)
      : "r"(0xffffffffu));
  return pred != 0;
}

// ---- mbarrier -------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug must surface as a CUDA error (trap), never as a hung GPU.
#ifndef MHMR_SPIN_LIMIT
#define MHMR_SPIN_LIMIT (1u << 28)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > MHMR_SPIN_LIMIT) __trap();
  }
}

// ---- TMA -------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tile load global -> shared, completion signalled on `bar` (complete_tx bytes).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                            int32_t c_inner, int32_t c_outer) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c_inner), "r"(c_outer)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* tmap,
                                                 uint64_t* bar, int32_t c_inner, int32_t c_outer,
                                                 uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c_inner), "r"(c_outer), "l"(cache_hint)
      : "memory");
}
// 3-D tile load (make_tmap_3d): column, row within matrix `c_depth`.
__device__ __forceinline__ void tma_load_3d_hint(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                                 int32_t c_inner, int32_t c_row, int32_t c_depth,
                                                 uint64_t cache_hint) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c_inner), "r"(c_row), "r"(c_depth), "l"(cache_hint)
      : "memory");
}
// 2-D tile store shared -> global (bulk async group).
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tmap, const void* smem_src,
                                             int32_t c_inner, int32_t c_outer) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               :
               : "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(smem_src)), "r"(c_inner),
                 "r"(c_outer)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
constexpr uint64_t kCacheEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kCacheEvictLast = 0x14F0000000000000ull;
constexpr uint64_t kCacheEvictNormal = 0x1000000000000000ull;

// ---- clusters ----------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// Arrive on the barrier at the same shared-memory offset in CTA `cta` of the cluster.  No cluster-scope release
// (that form compiles to a CTA- and a GPU-scope MEMBAR): a waiter in the other CTA must not rely on it to see
// this thread's earlier memory writes.
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// 2-D tile load global -> shared of every CTA in `cta_mask`, at the same offsets; each destination CTA's
// barrier at `bar`'s offset receives the bytes.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                                      int32_t c_inner, int32_t c_outer, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c_inner), "r"(c_outer), "h"(cta_mask)
      : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA) ----------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle.
//   K-major operand:  rows of 64 fp16 (128 B); 8-row swizzle atoms of 1024 B; SBO = byte distance between
//                     consecutive 8-row groups along M/N; LBO unused.
//   MN-major operand: rows of 64 fp16 along MN (128 B) indexed by k; 8 k-rows per atom (1024 B).
// The swizzle is a function of the address bits, so atoms must be 1024-byte aligned.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr, uint32_t lbo_bytes,
                                                    uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= 1ull << 62;  // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Named CTA barriers (ids 1..15; 0 is __syncthreads) over `count` threads, a multiple of 32: sync blocks until
// `count` threads have arrived, arrive counts this warp in and goes on.
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}
// Keeps the compiler from moving accumulator accesses across an in-flight wgmma.
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define MHMR_WG_D8(o) "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), \
                      "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
// D[64 x 64] (+)= A[smem] * B[smem]^T, fp16 operands, both K-major, fp32 accumulate.
__device__ __forceinline__ void wgmma_m64n64_ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : MHMR_WG_D8(0), MHMR_WG_D8(8), MHMR_WG_D8(16), MHMR_WG_D8(24)
      : "l"(da), "l"(db), "r"(acc));
}
// D[64 x 32] (+)= A[smem] * B[smem]^T, fp16 operands, both K-major, fp32 accumulate.
__device__ __forceinline__ void wgmma_m64n32_ss(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, 0, 0;\n\t}"
      : MHMR_WG_D8(0), MHMR_WG_D8(8)
      : "l"(da), "l"(db), "r"(acc));
}
// D[64 x 128] (+)= A[smem] * B[smem]^T, fp16 operands, both K-major, fp32 accumulate.
__device__ __forceinline__ void wgmma_m64n128_ss(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : MHMR_WG_D8(0), MHMR_WG_D8(8), MHMR_WG_D8(16), MHMR_WG_D8(24), MHMR_WG_D8(32), MHMR_WG_D8(40),
        MHMR_WG_D8(48), MHMR_WG_D8(56)
      : "l"(da), "l"(db), "r"(acc));
}
// D[64 x 64] += A[registers, fp16 fragments] * B[smem], B MN-major (transposed); fp32 accumulate.
__device__ __forceinline__ void wgmma_m64n64_rs_bt(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
      : MHMR_WG_D8(0), MHMR_WG_D8(8), MHMR_WG_D8(16), MHMR_WG_D8(24)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
#undef MHMR_WG_D8

// Elementwise float2 arithmetic (two independent fp32 operations, round to nearest).
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

// erf-GELU through the Abramowitz-Stegun 7.1.26 rational form (|abs err| < 5e-7 in fp32, two MUFU ops): used
// where the result is stored in fp16 (tensor-core operand of fc2), far above its precision needs.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-(z * z) * 1.4426950408889634f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float erf_abs = fmaf(-p * t, e, 1.0f);
  return 0.5f * x * (1.0f + copysignf(erf_abs, x));
}

// Two erf-GELUs at once (same Abramowitz-Stegun form as gelu_erf_fast).
__device__ __forceinline__ float2 gelu_erf_fast2(float2 x) {
  const float2 ax = make_float2(fabsf(x.x), fabsf(x.y));
  const float2 z = mul2(ax, make_float2(0.70710678118654752440f, 0.70710678118654752440f));
  const float2 d = fma2(z, make_float2(0.3275911f, 0.3275911f), make_float2(1.0f, 1.0f));
  float2 t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t.x) : "f"(d.x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t.y) : "f"(d.y));
  const float2 a = mul2(mul2(z, z), make_float2(-1.4426950408889634f, -1.4426950408889634f));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(a.x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(a.y));
  float2 p = fma2(make_float2(1.061405429f, 1.061405429f), t, make_float2(-1.453152027f, -1.453152027f));
  p = fma2(p, t, make_float2(1.421413741f, 1.421413741f));
  p = fma2(p, t, make_float2(-0.284496736f, -0.284496736f));
  p = fma2(p, t, make_float2(0.254829592f, 0.254829592f));
  const float2 pte = mul2(mul2(p, t), e);
  const float2 erf_abs = fma2(pte, make_float2(-1.0f, -1.0f), make_float2(1.0f, 1.0f));
  const float2 s = make_float2(copysignf(erf_abs.x, x.x), copysignf(erf_abs.y, x.y));
  const float2 hx = mul2(x, make_float2(0.5f, 0.5f));
  return fma2(hx, s, hx);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
#endif  // __CUDACC__

}  // namespace mhmr
