// SMPL-X layer: blend shapes + linear-blend skinning + camera placement (reference
// blocks/smpl_layer.py:47-155, which calls smplx.SMPLX.forward / lbs at :104; SURVEY.md §2.4 k18,k19).
//
// The stage is HBM-bound: the pose-corrective blend-shape matrix `posedirs` [486, 3V] (61 MB fp32) has to
// be streamed once per forward, everything else is small.  Layout decisions:
//   * PDX [486 + L, ldp]: posedirs with the L = num_betas + 10 shape/expression directions appended as
//     extra rows (shapedirs transposed), so shape and pose blending are ONE streaming pass with the
//     coefficient vector cf[p] = [pose_feature(486) | betas | expression].
//   * J_regressor is folded at load time: J(beta) = Jt + Jdirs . beta  (J is linear in beta), which removes
//     a 2.3 MB read and a cross-CTA reduction.
//   * one CTA per SM (80 vertices = 240 columns per CTA for V = 10475 on the 132 SMs of an H100); the CTA's column slab
//     is streamed through a TMA-fed shared-memory ring and 16 persons are accumulated per streamed row
//     (the matrix is read from HBM once; further blocks of 16 persons re-stream it from L2).
#include <utility>
#include <vector>

#include "kernels.cuh"

namespace mhmr {

namespace {

constexpr int kNJ = 55;
constexpr int kPoseFeat = 486;

// SMPL-X full_pose order (global, body 1..21, jaw, leye, reye, lhand 15, rhand 15) from the reference's
// 53-rotation order [root, body 21, lhand 15, rhand 15, jaw] (blocks/smpl_layer.py:88-101).
__device__ __forceinline__ int full_pose_source(int j) {
  if (j == 0) return -1;            // global_orient = 0 inside the body model (:88)
  if (j <= 21) return j;            // body
  if (j == 22) return 52;           // jaw
  if (j <= 24) return -1;           // eyes = 0 (:100-101)
  if (j <= 39) return 22 + (j - 25);  // left hand
  return 37 + (j - 40);             // right hand
}

// ------------------------------------------------------------------------------------------------
// Per person: Rodrigues xNJ, pose features, joints, kinematic chain, skinning transforms, placement.
// kRaw = false: the engine's SMPL-X layer -- rotvec [P, 53, 3] in the reference's order, global orient and eyes zero
//   inside the body model, root placed by R (x - pelvis) - center (blocks/smpl_layer.py:88-140).
// kRaw = true: the raw `smplx` body model as Trainer.prepare_gt calls it (train.py:76-109) -- rotvec is the full
//   pose [P, NJ, 3] in smplx order with the global rotation inside the chain, as `lbs` does; placement is the
//   identity (R = I, pelvis = 0, centre = 0), so the vertex / joints kernels add `transl` and nothing else.
// ------------------------------------------------------------------------------------------------
template <int NJ, int PF, bool kRaw>
__global__ void __launch_bounds__(64)
body_prep_kernel(const float* __restrict__ rotvec, const float* __restrict__ shape,
                 const float* __restrict__ expr, int n_expr, const float* __restrict__ Jt,
                 const float* __restrict__ Jdirs, const int* __restrict__ parents, const int* __restrict__ count,
                 int num_betas, int center_idx, int KT, float* __restrict__ cf, float* __restrict__ Amat,
                 float* __restrict__ xf, float* __restrict__ jposed) {
  static_assert(NJ <= 64 && PF == (NJ - 1) * 9, "one thread per joint; pose features = 9 (NJ - 1)");
  const int p = blockIdx.x;
  if (p >= *count) return;
  __shared__ float Rs[NJ][9];
  __shared__ float Js[NJ][3];
  __shared__ float Gs[NJ][12];
  __shared__ float beta[32];
  const int j = threadIdx.x;
  const int L = num_betas + n_expr;
  if (j < num_betas) beta[j] = shape[p * num_betas + j];
  if (j >= 32 && j < 32 + n_expr) beta[num_betas + (j - 32)] = expr[p * n_expr + (j - 32)];
  __syncthreads();
  if (j < NJ) {
    float rx = 0.f, ry = 0.f, rz = 0.f;
    const int src = kRaw ? j : full_pose_source(j);
    if (src >= 0) {
      const float* rv = rotvec + (static_cast<int64_t>(p) * (kRaw ? NJ : 53) + src) * 3;
      rx = rv[0]; ry = rv[1]; rz = rv[2];
    }
    // smplx.lbs.batch_rodrigues: angle = || r + 1e-8 ||, axis = r / angle
    const float ex = rx + 1e-8f, ey = ry + 1e-8f, ez = rz + 1e-8f;
    const float ang = sqrtf(ex * ex + ey * ey + ez * ez);
    const float ax = rx / ang, ay = ry / ang, az = rz / ang;
    const float s = sinf(ang), c1 = 1.f - cosf(ang);
    // K = [[0,-az,ay],[az,0,-ax],[-ay,ax,0]];  R = I + s K + (1-c) K K
    const float Kx[9] = {0.f, -az, ay, az, 0.f, -ax, -ay, ax, 0.f};
    float KK[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c)
        KK[r * 3 + c] = Kx[r * 3] * Kx[c] + Kx[r * 3 + 1] * Kx[3 + c] + Kx[r * 3 + 2] * Kx[6 + c];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const float id = (i == 0 || i == 4 || i == 8) ? 1.f : 0.f;
      const float R = id + s * Kx[i] + c1 * KK[i];
      Rs[j][i] = R;
      if (j >= 1) cf[static_cast<int64_t>(p) * KT + (j - 1) * 9 + i] = R - id;
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float v = Jt[j * 3 + r];
      for (int l = 0; l < L; ++l) v += Jdirs[(j * 3 + r) * L + l] * beta[l];
      Js[j][r] = v;
    }
  }
  if (j < L) cf[static_cast<int64_t>(p) * KT + PF + j] = beta[j];
  __syncthreads();
  if (j < NJ) {
    // kinematic chain (smplx.lbs.batch_rigid_transform): G_j = prod over the ancestors (root first) of
    // [R_i | J_i - J_parent(i)].  Every joint walks its own ancestor list (depth <= 16) independently
    // instead of one thread serialising the 55 joints; the product order equals the reference's.
    int anc[16];
    int depth = 0;
    for (int a = j; a >= 0 && depth < 16; a = parents[a]) anc[depth++] = a;
    float G[12];
    {
      const int r0 = anc[depth - 1];  // root
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        G[r * 4 + 0] = Rs[r0][r * 3 + 0];
        G[r * 4 + 1] = Rs[r0][r * 3 + 1];
        G[r * 4 + 2] = Rs[r0][r * 3 + 2];
        G[r * 4 + 3] = Js[r0][r];
      }
    }
    for (int d = depth - 2; d >= 0; --d) {
      const int i = anc[d], par = anc[d + 1];
      const float t0 = Js[i][0] - Js[par][0], t1 = Js[i][1] - Js[par][1], t2 = Js[i][2] - Js[par][2];
      float H[12];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const float g0 = G[r * 4], g1 = G[r * 4 + 1], g2 = G[r * 4 + 2];
#pragma unroll
        for (int c = 0; c < 3; ++c) H[r * 4 + c] = g0 * Rs[i][c] + g1 * Rs[i][3 + c] + g2 * Rs[i][6 + c];
        H[r * 4 + 3] = g0 * t0 + g1 * t1 + g2 * t2 + G[r * 4 + 3];
      }
#pragma unroll
      for (int q = 0; q < 12; ++q) G[q] = H[q];
    }
#pragma unroll
    for (int q = 0; q < 12; ++q) Gs[j][q] = G[q];
  }
  __syncthreads();
  if (j < NJ) {
    // A_j = G_j with translation G_t - G_R J_j; posed joint = G_t
    float* A = Amat + (static_cast<int64_t>(p) * NJ + j) * 12;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float g0 = Gs[j][r * 4], g1 = Gs[j][r * 4 + 1], g2 = Gs[j][r * 4 + 2];
      A[r * 4 + 0] = g0; A[r * 4 + 1] = g1; A[r * 4 + 2] = g2;
      A[r * 4 + 3] = Gs[j][r * 4 + 3] - (g0 * Js[j][0] + g1 * Js[j][1] + g2 * Js[j][2]);
      jposed[(static_cast<int64_t>(p) * NJ + j) * 3 + r] = Gs[j][r * 4 + 3];
    }
  }
  if (kRaw) {
    if (j < 16) xf[static_cast<int64_t>(p) * 16 + j] = (j == 0 || j == 4 || j == 8) ? 1.f : 0.f;
  } else if (j == 63) {
    // root placement (blocks/smpl_layer.py:107-140): R = roma.rotvec_to_rotmat(pose[:,0]),
    // x -> R (x - pelvis) - center + transl, center = R (J[center_idx] - pelvis)
    const float* rv = rotvec + static_cast<int64_t>(p) * 53 * 3;
    const float x = rv[0], y = rv[1], z = rv[2];
    const float th = sqrtf(x * x + y * y + z * z);
    float R[9];
    if (th < 1e-6f) {
      R[0] = 1.f; R[1] = -z; R[2] = y; R[3] = z; R[4] = 1.f; R[5] = -x; R[6] = -y; R[7] = x; R[8] = 1.f;
    } else {
      const float inv = 1.f / fmaxf(th, 1e-6f);
      const float kx = x * inv, ky = y * inv, kz = z * inv;
      const float s = sinf(th), c1 = 1.f - cosf(th);
      const float xs = kx * s, ys = ky * s, zs = kz * s;
      const float xyc = kx * ky * c1, xzc = kx * kz * c1, yzc = ky * kz * c1;
      const float xxc = kx * kx * c1, yyc = ky * ky * c1, zzc = kz * kz * c1;
      R[0] = 1.f - yyc - zzc; R[1] = xyc - zs; R[2] = xzc + ys;
      R[3] = xyc + zs; R[4] = 1.f - xxc - zzc; R[5] = -xs + yzc;
      R[6] = xzc - ys; R[7] = xs + yzc; R[8] = 1.f - xxc - yyc;
    }
    const float pel[3] = {Gs[0][3], Gs[0][7], Gs[0][11]};
    const float d[3] = {Gs[center_idx][3] - pel[0], Gs[center_idx][7] - pel[1], Gs[center_idx][11] - pel[2]};
    float* o = xf + static_cast<int64_t>(p) * 16;
#pragma unroll
    for (int i = 0; i < 9; ++i) o[i] = R[i];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      o[9 + r] = pel[r];
      const float cen = R[r * 3] * d[0] + R[r * 3 + 1] * d[1] + R[r * 3 + 2] * d[2];
      o[12 + r] = cen;  // subtracted after the rotation, then transl added (kept separate for rounding order)
    }
    o[15] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------------
// Vertex kernel: v_posed = v_template + cf . PDX ; skinning ; root placement ; optional projection.
// One CTA per SM (72 vertices = 216 coordinate columns).  A producer warp streams this CTA's column slab
// of PDX through a 6-stage shared-memory ring with TMA (16 rows x 220 columns per box; the 220-float pitch
// makes the consumers' 128-bit reads conflict-free) and bulk-copies the skinning-weight tile; 432 consumer
// threads = 54 column groups x 8 row lanes accumulate PB = 16 persons per streamed row, so the 64 MB matrix
// is read from HBM exactly once per forward with ~80 KB in flight per SM, decoupled from the FMA work.
// ------------------------------------------------------------------------------------------------
constexpr int kTV = 72;            // vertices per CTA
constexpr int kTC = kTV * 3;       // 216 columns
constexpr int kCG = kTC / 4;       // 54 float4 column groups
constexpr int kRL = 8;             // row lanes (adjacent lanes of a warp)
constexpr int kChunkRows = 16;     // PDX rows per TMA box
constexpr int kPitch = 220;        // floats per staged row (box inner size; 880 B)
constexpr int kStagesV = 6;
constexpr int kConsumers = kCG * kRL;              // 432
constexpr int kConsumerWarps = (kConsumers + 31) / 32;  // 14
constexpr int kVertThreads = kConsumerWarps * 32 + 32;  // + producer warp = 480
constexpr int kKTMax = 512;        // >= 486 + 21, multiple of kChunkRows
constexpr int kCfPitch = 20;       // floats per coefficient row (16 persons + pad: conflict-free)
constexpr int kStageFloats = kChunkRows * kPitch;

// PB persons per pass (a multiple of kRL): 16 for SMPL-X; the SMPL instance takes 8, whose 32 accumulators per
// consumer thread fit the 128-register budget without spilling.
template <int NJ, int PB>
struct VertSmem {
  float stage[kStagesV][kStageFloats];   // 6 x 14080 B (TMA destinations: 128-byte aligned)
  float Ws[kTV][NJ];                    // skinning-weight tile (bulk copy destination, 16-byte aligned)
  float pfs[kKTMax][kCfPitch];
  float As[PB][NJ * 12];
  float xf[PB][16];
  float tr[PB][4];
  float Kd[PB][12];
  float vps[PB][kTC];
  float outs[PB][kTC];
  float outs2[PB][kTV * 2];
  uint64_t full_bar[kStagesV];
  uint64_t empty_bar[kStagesV];
  uint64_t w_bar;
};

template <int NJ, int PB>
__global__ void __launch_bounds__(kVertThreads, 1)
smplx_vertex_kernel(const __grid_constant__ CUtensorMap tmPDX, int KT, const float* __restrict__ vt,
                    const float* __restrict__ Wl_padded, const float* __restrict__ cf,
                    const float* __restrict__ Amat, const float* __restrict__ xf,
                    const float* __restrict__ transl, const float* __restrict__ K_det,
                    const int* __restrict__ count, int V, float* __restrict__ v3d,
                    float* __restrict__ v2d) {
  extern __shared__ uint8_t vsmem_raw[];
  // 128-byte alignment by pointer arithmetic (keeps the shared address space: LDS/STS, not generic LD/ST)
  static_assert(PB % kRL == 0 && PB <= 16, "whole persons per row lane; pfs rows hold 16");
  VertSmem<NJ, PB>& sm = *reinterpret_cast<VertSmem<NJ, PB>*>(vsmem_raw + ((128u - (smem_u32(vsmem_raw) & 127u)) & 127u));
  const int P = *count;
  if (P <= 0) return;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int v0 = blockIdx.x * kTV;
  const int col0 = v0 * 3;
  const int nv = min(kTV, V - v0);
  const int ncol = nv * 3;
  const int n_chunks = (KT + kChunkRows - 1) / kChunkRows;
  const int n_pass = (P + PB - 1) / PB;
  const bool is_producer = (warp == kConsumerWarps);

  if (tid == 0) {
    for (int s = 0; s < kStagesV; ++s) {
      mbar_init(&sm.full_bar[s], 1);
      mbar_init(&sm.empty_bar[s], kConsumerWarps);
    }
    mbar_init(&sm.w_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (is_producer) {
    if (lane == 0) {
      tma_prefetch_desc(&tmPDX);
      // skinning-weight tile: rows v0..v0+71 of the padded [ceil(V/72)*72, 55] matrix are contiguous
      mbar_arrive_expect_tx(&sm.w_bar, kTV * NJ * 4);
      asm volatile(
          "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
              smem_u32(&sm.Ws[0][0])),
          "l"(Wl_padded + static_cast<int64_t>(v0) * NJ), "r"(kTV * NJ * 4), "r"(smem_u32(&sm.w_bar))
          : "memory");
      // fill the ring right away: the first kStagesV boxes need no hand-shake, so the HBM stream starts
      // while the other warps are still staging the per-person coefficients
      for (int c = 0; c < min(kStagesV, n_chunks); ++c) {
        mbar_arrive_expect_tx(&sm.full_bar[c], kStageFloats * 4);
        tma_load_2d_hint(&sm.stage[c][0], &tmPDX, &sm.full_bar[c], col0, c * kChunkRows,
                         n_pass > 1 ? kCacheEvictLast : kCacheEvictFirst);
      }
    }
  }

  const int ctid = min(tid, kConsumers - 1);  // idle lanes of the last consumer warp shadow a real thread
  const bool active = !is_producer && tid < kConsumers;
  const int cg = ctid >> 3, r = ctid & 7;
  uint32_t it = 0;

  for (int pass = 0; pass < n_pass; ++pass) {
    const int pb0 = pass * PB;
    const int np = min(PB, P - pb0);
    __syncthreads();  // previous pass finished with the per-person buffers
    for (int i = tid; i < kKTMax * PB; i += kVertThreads) {
      const int k = i / PB, j = i - k * PB;
      sm.pfs[k][j] = (j < np && k < KT) ? cf[static_cast<int64_t>(pb0 + j) * KT + k] : 0.f;
    }
    for (int i = tid; i < PB * NJ * 12; i += kVertThreads) {
      const int j = i / (NJ * 12), q = i - j * (NJ * 12);
      sm.As[j][q] = (j < np) ? Amat[static_cast<int64_t>(pb0 + j) * NJ * 12 + q] : 0.f;
    }
    for (int i = tid; i < PB * 16; i += kVertThreads) {
      const int j = i >> 4, q = i & 15;
      sm.xf[j][q] = (j < np) ? xf[static_cast<int64_t>(pb0 + j) * 16 + q] : 0.f;
      if (q < 4) sm.tr[j][q] = (j < np && q < 3) ? transl[(pb0 + j) * 3 + q] : 0.f;
      if (q < 9) sm.Kd[j][q] = (j < np) ? K_det[(pb0 + j) * 9 + q] : 0.f;
    }
    __syncthreads();

    if (!is_producer) {
      // ---- consume the streamed rows: acc[i][j] += cf[j][k] * PDX[k][col + i]
      float acc[4][PB];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < PB; ++j) acc[i][j] = 0.f;
      for (int c = 0; c < n_chunks; ++c, ++it) {
        const uint32_t s = it % kStagesV, ph = (it / kStagesV) & 1u;
        mbar_wait(&sm.full_bar[s], ph);
#pragma unroll
        for (int h = 0; h < kChunkRows / kRL; ++h) {
          const int row = h * kRL + r;
          const int k = c * kChunkRows + row;  // rows >= KT are zero-filled by TMA, pfs rows are zero
          const float4 w = *reinterpret_cast<const float4*>(&sm.stage[s][row * kPitch + cg * 4]);
#pragma unroll
          for (int q = 0; q < PB / 4; ++q) {
            const float4 cc = *reinterpret_cast<const float4*>(&sm.pfs[k][q * 4]);
            const float cj[4] = {cc.x, cc.y, cc.z, cc.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              acc[0][q * 4 + j] = fmaf(cj[j], w.x, acc[0][q * 4 + j]);
              acc[1][q * 4 + j] = fmaf(cj[j], w.y, acc[1][q * 4 + j]);
              acc[2][q * 4 + j] = fmaf(cj[j], w.z, acc[2][q * 4 + j]);
              acc[3][q * 4 + j] = fmaf(cj[j], w.w, acc[3][q * 4 + j]);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty_bar[s]);
      }
      // ---- fold the 8 row lanes (adjacent lanes), add the template; lane r keeps persons 2r, 2r+1
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < PB; ++j) {
          float v = acc[i][j];
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          acc[i][j] = v;
        }
      if (active) {
#pragma unroll
        for (int j = 0; j < PB; ++j) {
          if (j / (PB / kRL) == r) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int cc = cg * 4 + i;
              sm.vps[j][cc] = (cc < ncol) ? (vt[col0 + cc] + acc[i][j]) : 0.f;
            }
          }
        }
      }
    } else if (lane == 0) {
      // ---- producer: stream this CTA's column slab, 16 rows per box, through the ring
      for (int c = 0; c < n_chunks; ++c, ++it) {
        if (pass == 0 && c < kStagesV) continue;  // already in flight (prologue)
        const uint32_t s = it % kStagesV, ph = (it / kStagesV) & 1u;
        mbar_wait(&sm.empty_bar[s], ph ^ 1u);
        mbar_arrive_expect_tx(&sm.full_bar[s], kStageFloats * 4);
        tma_load_2d_hint(&sm.stage[s][0], &tmPDX, &sm.full_bar[s], col0, c * kChunkRows,
                         n_pass > 1 ? kCacheEvictLast : kCacheEvictFirst);
      }
    }
    if (pass == 0) mbar_wait(&sm.w_bar, 0);  // skinning weights have landed
    __syncthreads();

    // ---- skinning + root placement + projection, one (vertex, person) pair per thread-iteration
    for (int i = tid; i < kTV * PB; i += kVertThreads) {
      const int j = i / kTV, v = i - j * kTV;
      if (v >= nv || j >= np) continue;
      float4 T0 = make_float4(0.f, 0.f, 0.f, 0.f), T1 = T0, T2 = T0;
      for (int jj = 0; jj < NJ; ++jj) {
        const float w = sm.Ws[v][jj];
        const float4* A = reinterpret_cast<const float4*>(&sm.As[j][jj * 12]);
        const float4 a0 = A[0], a1 = A[1], a2 = A[2];
        T0.x = fmaf(w, a0.x, T0.x); T0.y = fmaf(w, a0.y, T0.y); T0.z = fmaf(w, a0.z, T0.z); T0.w = fmaf(w, a0.w, T0.w);
        T1.x = fmaf(w, a1.x, T1.x); T1.y = fmaf(w, a1.y, T1.y); T1.z = fmaf(w, a1.z, T1.z); T1.w = fmaf(w, a1.w, T1.w);
        T2.x = fmaf(w, a2.x, T2.x); T2.y = fmaf(w, a2.y, T2.y); T2.z = fmaf(w, a2.z, T2.z); T2.w = fmaf(w, a2.w, T2.w);
      }
      const float x = sm.vps[j][v * 3], y = sm.vps[j][v * 3 + 1], z = sm.vps[j][v * 3 + 2];
      const float q0 = T0.x * x + T0.y * y + T0.z * z + T0.w;
      const float q1 = T1.x * x + T1.y * y + T1.z * z + T1.w;
      const float q2 = T2.x * x + T2.y * y + T2.z * z + T2.w;
      const float* X = sm.xf[j];
      const float dx = q0 - X[9], dy = q1 - X[10], dz = q2 - X[11];
      float o[3];
#pragma unroll
      for (int q = 0; q < 3; ++q)
        o[q] = ((X[q * 3] * dx + X[q * 3 + 1] * dy + X[q * 3 + 2] * dz) - X[12 + q]) + sm.tr[j][q];
      sm.outs[j][v * 3] = o[0];
      sm.outs[j][v * 3 + 1] = o[1];
      sm.outs[j][v * 3 + 2] = o[2];
      // perspective_projection (utils/camera.py:14-27): K . (p / p_z)
      const float* Kd = sm.Kd[j];
      const float u = o[0] / o[2], w_ = o[1] / o[2], one = o[2] / o[2];
      sm.outs2[j][v * 2] = Kd[0] * u + Kd[1] * w_ + Kd[2] * one;
      sm.outs2[j][v * 2 + 1] = Kd[3] * u + Kd[4] * w_ + Kd[5] * one;
    }
    __syncthreads();
    for (int i = tid; i < PB * kTC; i += kVertThreads) {
      const int j = i / kTC, c = i - j * kTC;
      if (j < np && c < ncol) v3d[(static_cast<int64_t>(pb0 + j) * V) * 3 + col0 + c] = sm.outs[j][c];
    }
    if (v2d != nullptr) {
      for (int i = tid; i < PB * kTV * 2; i += kVertThreads) {
        const int j = i / (kTV * 2), c = i - j * (kTV * 2);
        if (j < np && c < nv * 2) v2d[(static_cast<int64_t>(pb0 + j) * V) * 2 + v0 * 2 + c] = sm.outs2[j][c];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Joints: NJ posed LBS joints + 21 vertex-picked joints + NL barycentric face landmarks (smplx.SMPLX.forward:
// 55 + 21 + 51 = 127; smplx.SMPL.forward: 24 + 21 + 0 = 45), placed like the vertices; 2-D projection; transl_pelvis.
// ------------------------------------------------------------------------------------------------
template <int NJ, int NL>
__global__ void __launch_bounds__(128)
smplx_joints_kernel(const float* __restrict__ jposed, const float* __restrict__ xf,
                    const float* __restrict__ transl, const float* __restrict__ K_det,
                    const float* __restrict__ v3d, const int* __restrict__ extra_idx,
                    const int* __restrict__ lmk_tri, const float* __restrict__ lmk_bary,
                    const int* __restrict__ count, int V, float* __restrict__ j3d, float* __restrict__ j2d,
                    float* __restrict__ transl_pelvis) {
  const int p = blockIdx.x;
  if (p >= *count) return;
  const int j = threadIdx.x;
  constexpr int kJ = NJ + 21 + NL;
  static_assert(kJ <= 128, "one thread per joint");
  if (j >= kJ) return;
  float o[3];
  const float* vp = v3d + static_cast<int64_t>(p) * V * 3;
  if (j < NJ) {
    const float* X = xf + static_cast<int64_t>(p) * 16;
    const float* q = jposed + (static_cast<int64_t>(p) * NJ + j) * 3;
    const float dx = q[0] - X[9], dy = q[1] - X[10], dz = q[2] - X[11];
#pragma unroll
    for (int r = 0; r < 3; ++r)
      o[r] = ((X[r * 3] * dx + X[r * 3 + 1] * dy + X[r * 3 + 2] * dz) - X[12 + r]) + transl[p * 3 + r];
  } else if (j < NJ + 21) {
    const int v = extra_idx[j - NJ];
    o[0] = vp[v * 3]; o[1] = vp[v * 3 + 1]; o[2] = vp[v * 3 + 2];
  } else {
    const int l = j - NJ - 21;
    o[0] = o[1] = o[2] = 0.f;
#pragma unroll
    for (int f = 0; f < 3; ++f) {
      const int v = lmk_tri[l * 3 + f];
      const float b = lmk_bary[l * 3 + f];
      o[0] = fmaf(b, vp[v * 3], o[0]);
      o[1] = fmaf(b, vp[v * 3 + 1], o[1]);
      o[2] = fmaf(b, vp[v * 3 + 2], o[2]);
    }
  }
  float* jo = j3d + (static_cast<int64_t>(p) * kJ + j) * 3;
  jo[0] = o[0]; jo[1] = o[1]; jo[2] = o[2];
  if (j == 0) {
    transl_pelvis[p * 3] = o[0]; transl_pelvis[p * 3 + 1] = o[1]; transl_pelvis[p * 3 + 2] = o[2];
  }
  const float* Kd = K_det + p * 9;
  const float u = o[0] / o[2], w = o[1] / o[2], one = o[2] / o[2];
  j2d[(static_cast<int64_t>(p) * kJ + j) * 2] = Kd[0] * u + Kd[1] * w + Kd[2] * one;
  j2d[(static_cast<int64_t>(p) * kJ + j) * 2 + 1] = Kd[3] * u + Kd[4] * w + Kd[5] * one;
}

// ------------------------------------------------------------------------------------------------
// Load-time folding / repacking kernels
// ------------------------------------------------------------------------------------------------
// PDX[k, c]: k < PF -> posedirs[k, c]; k >= PF -> shapedirs_full[c, k - PF]  (shapedirs_full [3V, L])
__global__ void build_pdx_kernel(const float* __restrict__ posedirs, const float* __restrict__ sdirs, int PF, int L,
                                 int V3, int ldp, float* __restrict__ PDX) {
  const int k = blockIdx.y;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < ldp; c += gridDim.x * blockDim.x) {
    float v = 0.f;
    if (c < V3) v = (k < PF) ? posedirs[static_cast<int64_t>(k) * V3 + c] : sdirs[static_cast<int64_t>(c) * L + (k - PF)];
    PDX[static_cast<int64_t>(k) * ldp + c] = v;
  }
}

// out[j, q] = sum_v Jr[j, v] * M[v, q]   (q < Q) — folds J_regressor into the template / shape directions
__global__ void fold_jreg_kernel(const float* __restrict__ Jr, const float* __restrict__ M, int V, int Q,
                                 float* __restrict__ out) {
  const int j = blockIdx.x, q = blockIdx.y;
  __shared__ float red[8];
  float s = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) s += Jr[static_cast<int64_t>(j) * V + v] * M[static_cast<int64_t>(v) * Q + q];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += red[w];
    out[j * Q + q] = t;
  }
}

// prep -> vertices -> joints for one body-model shape (NJ kinematic joints, PF pose features, NL landmarks)
template <int NJ, int PF, int NL, int PB, bool kRaw>
int body_forward_impl(const SmplxDeviceModel& bm, const float* rotvec, const float* shape, const float* expr,
                      const float* transl, const float* K_det, const int* count, int max_persons, SmplxScratch& ws,
                      float* v3d, float* v2d, float* j3d, float* j2d, float* transl_pelvis, cudaStream_t st) {
  const int KT = PF + bm.L;
  MHMR_REQUIRE(KT <= kKTMax, "smplx: too many blend-shape coefficients");
  MHMR_REQUIRE(bm.num_joints == NJ && bm.pose_feat == PF && bm.n_lmk == NL, "body model / kernel shape mismatch");
  body_prep_kernel<NJ, PF, kRaw><<<max_persons, 64, 0, st>>>(rotvec, shape, expr, bm.L - bm.num_betas, bm.Jt,
                                                             bm.Jdirs, bm.parents, count, bm.num_betas, bm.center_idx,
                                                             KT, ws.cf, ws.Amat, ws.xf, ws.jposed);
  MHMR_CUDA_CHECK(cudaGetLastError());
  static PerDeviceOnce once;
  const int vsmem = static_cast<int>(sizeof(VertSmem<NJ, PB>)) + 128;
  if (once.first()) {
    MHMR_CUDA_CHECK(cudaFuncSetAttribute(smplx_vertex_kernel<NJ, PB>, cudaFuncAttributeMaxDynamicSharedMemorySize, vsmem));
  }
  const int tiles = (bm.V + kTV - 1) / kTV;
  smplx_vertex_kernel<NJ, PB><<<tiles, kVertThreads, vsmem, st>>>(bm.tmPDX, KT, bm.vt, bm.lbs_weights_padded, ws.cf,
                                                             ws.Amat, ws.xf, transl, K_det, count, bm.V, v3d, v2d);
  MHMR_CUDA_CHECK(cudaGetLastError());
  smplx_joints_kernel<NJ, NL><<<max_persons, 128, 0, st>>>(ws.jposed, ws.xf, transl, K_det, v3d, bm.extra_idx,
                                                           bm.lmk_tri, bm.lmk_bary, count, bm.V, j3d, j2d,
                                                           transl_pelvis);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

}  // namespace

// TMA descriptor of PDX [KT, ldp] fp32: boxes of 16 rows x 220 columns, no swizzle.
int smplx_make_tmap(SmplxDeviceModel* bm) {
  return make_tmap_2d(&bm->tmPDX, bm->PDX, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, bm->pose_feat + bm->L, bm->ldp,
                      static_cast<uint64_t>(bm->ldp) * 4, kChunkRows, kPitch, false);
}
int smplx_tile_verts() { return kTV; }

int smplx_build_pdx(const float* posedirs, const float* sdirs_full, int PF, int L, int V, int ldp, float* PDX,
                    cudaStream_t st) {
  build_pdx_kernel<<<dim3(32, PF + L), 256, 0, st>>>(posedirs, sdirs_full, PF, L, V * 3, ldp, PDX);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int smplx_fold_jreg(const float* Jr, const float* M, int NJ, int V, int Q, float* out, cudaStream_t st) {
  fold_jreg_kernel<<<dim3(NJ, Q), 256, 0, st>>>(Jr, M, V, Q, out);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int smplx_forward(const SmplxDeviceModel& bm, const float* rotvec, const float* shape, const float* expr,
                  const float* transl, const float* K_det, const int* count, int max_persons,
                  SmplxScratch& ws, float* v3d, float* v2d, float* j3d, float* j2d, float* transl_pelvis,
                  cudaStream_t st) {
  return body_forward_impl<kNJ, kPoseFeat, 51, 16, false>(bm, rotvec, shape, expr, transl, K_det, count, max_persons, ws,
                                                      v3d, v2d, j3d, j2d, transl_pelvis, st);
}

int body_forward_raw(const SmplxDeviceModel& bm, const float* full_pose, const float* betas, const float* expr,
                     const float* transl, const float* K, const int* count, int max_persons, SmplxScratch& ws,
                     float* v3d, float* v2d, float* j3d, float* j2d, float* transl_pelvis, cudaStream_t st) {
  if (bm.num_joints == 24)
    return body_forward_impl<24, 207, 0, 8, true>(bm, full_pose, betas, expr, transl, K, count, max_persons, ws, v3d,
                                               v2d, j3d, j2d, transl_pelvis, st);
  if (bm.num_joints == kNJ)
    return body_forward_impl<kNJ, kPoseFeat, 51, 16, true>(bm, full_pose, betas, expr, transl, K, count, max_persons, ws,
                                                       v3d, v2d, j3d, j2d, transl_pelvis, st);
  set_last_error("body model: only SMPL (24 joints) and SMPL-X (55 joints) are instantiated");
  return MHMR_ERR_UNSUPPORTED;
}

// ================================================================================================
// Backward: input gradients of the two layers above (DESIGN.md §9).  Stateless: each call recomputes the per-person
// prep with body_prep_kernel into its own scratch, plus the vertex / joint forward when a 2-D upstream gradient needs
// the projected points.  No float atomics: every cross-CTA sum goes through per-tile partials that the person kernel
// adds in tile order, so the bits do not depend on scheduling or on the other persons of the call.
//   1. body_grad_joints_kernel   per person: gJ = g_j3d + proj^T g_j2d (+ g_transl_pelvis on joint 0)
//   2. body_grad_stream_kernel   per 80-vertex tile, 16 persons per pass over the tile's PDX slab:
//        g_o (vertex outputs, incl. the landmark / vertex-picked joints through the vertex->joint table),
//        g_q = R_root^T g_o, T_i = sum_j w_ij A_j, g_vposed = T_i[:3,:3]^T g_q;
//        streamed rows k: v_posed += cf_k PDX_k (forward contraction) and g_cf_k = PDX_k . g_vposed (reduction);
//        then g_A_j = sum_i w_ij g_q_i [v_posed_i; 1]^T, sum_i g_o_i and sum_i g_o_i q_i^T as tile partials
//   3. body_grad_person_kernel   per person: tile sums, placement, A -> G, kinematic chain in reverse, pose
//        features, Rodrigues, J(beta) = Jt + Jdirs beta, loc / dist
// ================================================================================================
namespace {

constexpr int kGTV = 80;            // vertices per CTA: 131 tiles for V = 10475 on 132 SMs
constexpr int kGTC = kGTV * 3;       // 240 columns
constexpr int kGThreads = 256;
constexpr int kGPB = 16;             // persons per pass over the slab
constexpr int kGRows = 16;           // PDX rows per staged chunk: (row, person) = 256 dot products per chunk
constexpr int kGStages = 3;          // cp.async ring depth
constexpr int kGvpPitch = kGTC + 1;  // odd pitch: the 16 persons of one row group read 16 distinct banks
constexpr int kGChunkF4 = kGRows * kGTC / 4;  // 960 float4 per chunk

template <int NJ>
struct GradSmem {
  float stage[kGStages][kGRows][kGTC];
  float pfs[kKTMax][kGPB];
  float Ws[kGTV][NJ];
  float gvp[kGPB][kGvpPitch];
  float go[kGPB][kGTC];
  float vps[kGPB][kGTC];
  float Ts[kGPB][kGTV][12];  // skinning transforms, then the outer products g_q [v_posed; 1]^T
};

__device__ __forceinline__ void cp_async16_zfill(void* smem, const void* gmem, bool pred) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(pred ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// perspective_projection backward at the camera-space point o: out2 = K[:2] . (o / o_z) (o_z / o_z has derivative 0)
__device__ __forceinline__ void proj_grad(const float* o, const float* Kd, float g0, float g1, float* go) {
  const float iz = 1.f / o[2];
  const float gu = Kd[0] * g0 + Kd[3] * g1, gw = Kd[1] * g0 + Kd[4] * g1;
  go[0] += gu * iz;
  go[1] += gw * iz;
  go[2] -= (gu * o[0] + gw * o[1]) * iz * iz;
}

// d<g, R(r)>/dr for R = I + A(a) K(r) + B(a) K(r)^2, A = sin a / a, B = (1 - cos a) / a^2, a = ||r + eps||:
// eps = 1e-8 is smplx.batch_rodrigues, eps = 0 with `roma` is roma.rotvec_to_rotmat (first-order below 1e-6 rad).
// Below a = 0.5 A, B and their derivatives come from their Taylor series (truncation < 1e-9), which keeps the
// a^3 / a^4 cancellations of the closed forms out of fp32 and makes r = 0 exact.
__device__ void rotvec_grad(float rx, float ry, float rz, float eps, bool roma, const float* g, float* out) {
  const float ge[3] = {g[7] - g[5], g[2] - g[6], g[3] - g[1]};  // <g, K(e_k)>
  const float ex = rx + eps, ey = ry + eps, ez = rz + eps;
  const float a = sqrtf(ex * ex + ey * ey + ez * ez);
  if (roma && a < 1e-6f) {
    out[0] = ge[0]; out[1] = ge[1]; out[2] = ge[2];
    return;
  }
  const float a2 = a * a;
  float A, B, Ap, Bp;
  if (a < 0.5f) {
    A = 1.f - a2 / 6.f * (1.f - a2 / 20.f * (1.f - a2 / 42.f * (1.f - a2 / 72.f)));
    B = 0.5f * (1.f - a2 / 12.f * (1.f - a2 / 30.f * (1.f - a2 / 56.f * (1.f - a2 / 90.f))));
    Ap = -a / 3.f * (1.f - a2 / 10.f * (1.f - a2 / 28.f * (1.f - a2 / 54.f)));
    Bp = -a / 12.f * (1.f - a2 / 15.f * (1.f - a2 * (3.f / 112.f) * (1.f - a2 / 67.5f)));
  } else {
    const float s = sinf(a), c = cosf(a), h = sinf(0.5f * a);
    const float omc = 2.f * h * h;
    A = s / a;
    B = omc / a2;
    Ap = (a * c - s) / a2;
    Bp = (a * s - 2.f * omc) / (a2 * a);
  }
  const float Kr[9] = {0.f, -rz, ry, rz, 0.f, -rx, -ry, rx, 0.f};
  float gK = 0.f, gKK = 0.f;
#pragma unroll
  for (int m = 0; m < 3; ++m)
#pragma unroll
    for (int n = 0; n < 3; ++n) {
      const float kk = Kr[m * 3] * Kr[n] + Kr[m * 3 + 1] * Kr[3 + n] + Kr[m * 3 + 2] * Kr[6 + n];
      gK += g[m * 3 + n] * Kr[m * 3 + n];
      gKK += g[m * 3 + n] * kk;
    }
  const float e[3] = {ex, ey, ez};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float E[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // K(e_k)
    if (k == 0) { E[5] = -1.f; E[7] = 1.f; }
    if (k == 1) { E[2] = 1.f; E[6] = -1.f; }
    if (k == 2) { E[1] = -1.f; E[3] = 1.f; }
    float gM = 0.f;  // <g, E K + K E>
#pragma unroll
    for (int m = 0; m < 3; ++m)
#pragma unroll
      for (int n = 0; n < 3; ++n) {
        float v = 0.f;
#pragma unroll
        for (int q = 0; q < 3; ++q) v += E[m * 3 + q] * Kr[q * 3 + n] + Kr[m * 3 + q] * E[q * 3 + n];
        gM += g[m * 3 + n] * v;
      }
    const float dadr = a > 0.f ? e[k] / a : 0.f;
    out[k] = dadr * (Ap * gK + Bp * gKK) + A * ge[k] + B * gM;
  }
}

// 1. per-output-joint upstream gradient (camera space)
__global__ void __launch_bounds__(128)
body_grad_joints_kernel(const float* __restrict__ j3d, const float* __restrict__ K, const float* __restrict__ g_j3d,
                        const float* __restrict__ g_j2d, const float* __restrict__ g_tp, int J, float* __restrict__ gJ) {
  const int p = blockIdx.x, j = threadIdx.x;
  if (j >= J) return;
  const int64_t pj = static_cast<int64_t>(p) * J + j;
  float g[3] = {0.f, 0.f, 0.f};
  if (g_j3d != nullptr) { g[0] = g_j3d[pj * 3]; g[1] = g_j3d[pj * 3 + 1]; g[2] = g_j3d[pj * 3 + 2]; }
  if (g_j2d != nullptr) proj_grad(j3d + pj * 3, K + p * 9, g_j2d[pj * 2], g_j2d[pj * 2 + 1], g);
  if (j == 0 && g_tp != nullptr) { g[0] += g_tp[p * 3]; g[1] += g_tp[p * 3 + 1]; g[2] += g_tp[p * 3 + 2]; }
  gJ[pj * 3] = g[0]; gJ[pj * 3 + 1] = g[1]; gJ[pj * 3 + 2] = g[2];
}

// 2. the streaming pass.  part[tile][p][PS]: [g_A (NJ x 12) | g_cf (KT) | sum g_o (3) | sum g_o q^T (9)]
template <int NJ>
__global__ void __launch_bounds__(kGThreads, 1)
body_grad_stream_kernel(const float* __restrict__ PDX, int ldp, int KT, const float* __restrict__ vt,
                        const float* __restrict__ W, const float* __restrict__ cf, const float* __restrict__ Amat,
                        const float* __restrict__ xf, const float* __restrict__ K, const float* __restrict__ vout,
                        const float* __restrict__ g_v3d, const float* __restrict__ g_v2d,
                        const float* __restrict__ gJ, int J, const int* __restrict__ v2j_ptr,
                        const int* __restrict__ v2j_jt, const float* __restrict__ v2j_w, int P, int V, int PS,
                        float* __restrict__ part) {
  extern __shared__ uint8_t gsm_raw[];
  GradSmem<NJ>& sm = *reinterpret_cast<GradSmem<NJ>*>(gsm_raw + ((16u - (smem_u32(gsm_raw) & 15u)) & 15u));
  const int tid = threadIdx.x, tile = blockIdx.x;
  const int v0 = tile * kGTV, nv = min(kGTV, V - v0), col0 = v0 * 3, ncol = nv * 3;
  const int n_chunks = (KT + kGRows - 1) / kGRows;
  const int brow = tid >> 4, bj = tid & 15;  // (row, person) of the g_cf dot product

  for (int i = tid; i < kGTV * NJ; i += kGThreads) {
    const int v = i / NJ, jj = i - v * NJ;
    sm.Ws[v][jj] = (v < nv) ? W[static_cast<int64_t>(v0 + v) * NJ + jj] : 0.f;
  }
  auto issue = [&](int ch) {
    float* dst = &sm.stage[ch % kGStages][0][0];
    for (int idx = tid; idx < kGChunkF4; idx += kGThreads) {
      const int row = idx / (kGTC / 4), c4 = idx - row * (kGTC / 4);
      const int k = ch * kGRows + row, col = col0 + c4 * 4;
      const bool ok = k < KT && col < ldp;  // ldp is a multiple of 4: a float4 is wholly inside or outside
      cp_async16_zfill(dst + row * kGTC + c4 * 4, ok ? PDX + static_cast<int64_t>(k) * ldp + col : PDX, ok);
    }
  };

  for (int pb0 = 0; pb0 < P; pb0 += kGPB) {
    const int np = min(kGPB, P - pb0);
    __syncthreads();  // the previous pass is done with every buffer
    // the first stages of the slab stream while the per-vertex work below runs
    for (int ch = 0; ch < kGStages - 1; ++ch) {
      if (ch < n_chunks) issue(ch);
      cp_async_commit();
    }
    for (int i = tid; i < kKTMax * kGPB; i += kGThreads) {
      const int k = i / kGPB, j = i - k * kGPB;
      sm.pfs[k][j] = (j < np && k < KT) ? cf[static_cast<int64_t>(pb0 + j) * KT + k] : 0.f;
    }
    // ---- per (person, vertex): output gradient, skinning transform, g_vposed
    for (int i = tid; i < kGPB * kGTV; i += kGThreads) {
      const int j = i / kGTV, v = i - j * kGTV;
      float go[3] = {0.f, 0.f, 0.f}, gv[3] = {0.f, 0.f, 0.f};
      float T[12];
#pragma unroll
      for (int q = 0; q < 12; ++q) T[q] = 0.f;
      if (j < np && v < nv) {
        const int p = pb0 + j;
        const int64_t pv = static_cast<int64_t>(p) * V + v0 + v;
        if (g_v3d != nullptr) { go[0] = g_v3d[pv * 3]; go[1] = g_v3d[pv * 3 + 1]; go[2] = g_v3d[pv * 3 + 2]; }
        if (g_v2d != nullptr) proj_grad(vout + pv * 3, K + p * 9, g_v2d[pv * 2], g_v2d[pv * 2 + 1], go);
        for (int e = v2j_ptr[v0 + v]; e < v2j_ptr[v0 + v + 1]; ++e) {
          const float w = v2j_w[e];
          const float* gj = gJ + (static_cast<int64_t>(p) * J + v2j_jt[e]) * 3;
          go[0] = fmaf(w, gj[0], go[0]); go[1] = fmaf(w, gj[1], go[1]); go[2] = fmaf(w, gj[2], go[2]);
        }
        const float4* A = reinterpret_cast<const float4*>(Amat + static_cast<int64_t>(p) * NJ * 12);
#pragma unroll 4
        for (int jj = 0; jj < NJ; ++jj) {
          const float w = sm.Ws[v][jj];
          const float4 a0 = __ldg(A + jj * 3), a1 = __ldg(A + jj * 3 + 1), a2 = __ldg(A + jj * 3 + 2);
          T[0] = fmaf(w, a0.x, T[0]); T[1] = fmaf(w, a0.y, T[1]); T[2] = fmaf(w, a0.z, T[2]); T[3] = fmaf(w, a0.w, T[3]);
          T[4] = fmaf(w, a1.x, T[4]); T[5] = fmaf(w, a1.y, T[5]); T[6] = fmaf(w, a1.z, T[6]); T[7] = fmaf(w, a1.w, T[7]);
          T[8] = fmaf(w, a2.x, T[8]); T[9] = fmaf(w, a2.y, T[9]); T[10] = fmaf(w, a2.z, T[10]); T[11] = fmaf(w, a2.w, T[11]);
        }
        const float* X = xf + static_cast<int64_t>(p) * 16;
        float gq[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) gq[c] = X[c] * go[0] + X[3 + c] * go[1] + X[6 + c] * go[2];
#pragma unroll
        for (int c = 0; c < 3; ++c) gv[c] = T[c] * gq[0] + T[4 + c] * gq[1] + T[8 + c] * gq[2];
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        sm.go[j][v * 3 + c] = go[c];
        sm.gvp[j][v * 3 + c] = gv[c];
      }
#pragma unroll
      for (int q = 0; q < 12; ++q) sm.Ts[j][v][q] = T[q];
    }

    // ---- stream the slab: v_posed accumulation (column threads) and g_cf dot products ((row, person) threads)
    float acc[kGPB];
#pragma unroll
    for (int j = 0; j < kGPB; ++j) acc[j] = 0.f;
    for (int ch = 0; ch < n_chunks; ++ch) {
      cp_async_wait<kGStages - 2>();
      __syncthreads();  // chunk ch visible to all; everyone is done with the stage refilled next
      if (ch + kGStages - 1 < n_chunks) issue(ch + kGStages - 1);
      cp_async_commit();
      const float(*stg)[kGTC] = sm.stage[ch % kGStages];
      if (tid < kGTC) {
#pragma unroll 4
        for (int row = 0; row < kGRows; ++row) {
          const float w = stg[row][tid];
          const int k = ch * kGRows + row;
#pragma unroll
          for (int q = 0; q < kGPB / 4; ++q) {
            const float4 cc = *reinterpret_cast<const float4*>(&sm.pfs[k][q * 4]);
            acc[q * 4] = fmaf(cc.x, w, acc[q * 4]);
            acc[q * 4 + 1] = fmaf(cc.y, w, acc[q * 4 + 1]);
            acc[q * 4 + 2] = fmaf(cc.z, w, acc[q * 4 + 2]);
            acc[q * 4 + 3] = fmaf(cc.w, w, acc[q * 4 + 3]);
          }
        }
      }
      {
        const float* st = stg[brow];
        const float* gv = sm.gvp[bj];
        float s8[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) s8[u] = 0.f;
#pragma unroll 2
        for (int c = 0; c < kGTC; c += 8)
#pragma unroll
          for (int u = 0; u < 8; ++u) s8[u] = fmaf(st[c + u], gv[c + u], s8[u]);
        const float s = ((s8[0] + s8[1]) + (s8[2] + s8[3])) + ((s8[4] + s8[5]) + (s8[6] + s8[7]));
        const int k = ch * kGRows + brow;
        if (bj < np && k < KT) part[(static_cast<int64_t>(tile) * P + pb0 + bj) * PS + NJ * 12 + k] = s;
      }
    }
    cp_async_wait<0>();
    if (tid < kGTC) {
#pragma unroll
      for (int j = 0; j < kGPB; ++j) sm.vps[j][tid] = (tid < ncol) ? vt[col0 + tid] + acc[j] : 0.f;
    }
    __syncthreads();
    // ---- per (person, vertex): posed vertex q = T [v_posed; 1] and the outer product g_q [v_posed; 1]^T
    for (int i = tid; i < kGPB * kGTV; i += kGThreads) {
      const int j = i / kGTV, v = i - j * kGTV;
      const float* T = sm.Ts[j][v];
      const float vp[4] = {sm.vps[j][v * 3], sm.vps[j][v * 3 + 1], sm.vps[j][v * 3 + 2], 1.f};
      float q[3], gq[3];
      const float* X = xf + static_cast<int64_t>(pb0 + min(j, np - 1)) * 16;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        q[r] = T[r * 4] * vp[0] + T[r * 4 + 1] * vp[1] + T[r * 4 + 2] * vp[2] + T[r * 4 + 3];
        gq[r] = X[r] * sm.go[j][v * 3] + X[3 + r] * sm.go[j][v * 3 + 1] + X[6 + r] * sm.go[j][v * 3 + 2];
      }
      float* M = sm.Ts[j][v];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) M[r * 4 + s] = gq[r] * vp[s];
#pragma unroll
      for (int r = 0; r < 3; ++r) sm.vps[j][v * 3 + r] = q[r];
    }
    __syncthreads();
    // ---- tile partials, each summed over the tile's vertices in vertex order
    const int nE = NJ * 12 + 12;
    for (int i = tid; i < np * nE; i += kGThreads) {
      const int j = i / nE, e = i - j * nE;
      float s4[4] = {0.f, 0.f, 0.f, 0.f};
      int dst;
      if (e < NJ * 12) {
        const int jj = e / 12, q = e - jj * 12;
        for (int v = 0; v < nv; ++v) s4[v & 3] = fmaf(sm.Ws[v][jj], sm.Ts[j][v][q], s4[v & 3]);
        dst = e;
      } else {
        const int e2 = e - NJ * 12;
        if (e2 < 3) {
          for (int v = 0; v < nv; ++v) s4[v & 3] += sm.go[j][v * 3 + e2];
        } else {
          const int r = (e2 - 3) / 3, c = (e2 - 3) - r * 3;
          for (int v = 0; v < nv; ++v) s4[v & 3] = fmaf(sm.go[j][v * 3 + r], sm.vps[j][v * 3 + c], s4[v & 3]);
        }
        dst = NJ * 12 + KT + e2;
      }
      part[(static_cast<int64_t>(tile) * P + pb0 + j) * PS + dst] = (s4[0] + s4[1]) + (s4[2] + s4[3]);
    }
  }
}

// 3. per person: tile sums, placement, A -> G, kinematic chain in reverse, pose features, Rodrigues, J(beta).
// kRaw: d_rot = d_full_pose [P, NJ, 3], d_transl written; else d_rot = d_rotvec [P, 53, 3], d_loc / d_dist written,
// and d_R [P, 53, 9] (nullable) receives the gradient with respect to each rotation matrix, before Rodrigues.
template <int NJ, int PF, bool kRaw>
__global__ void __launch_bounds__(256)
body_grad_person_kernel(const float* __restrict__ rotvec, const float* __restrict__ shape,
                        const float* __restrict__ expr, int n_expr, const float* __restrict__ Jt,
                        const float* __restrict__ Jdirs, const int* __restrict__ parents, int num_betas,
                        int center_idx, int KT, const float* __restrict__ Amat, const float* __restrict__ jposed,
                        const float* __restrict__ xf, const float* __restrict__ gJ, int J,
                        const float* __restrict__ part, int tiles, int P, int PS, const float* __restrict__ loc,
                        const float* __restrict__ dist, const float* __restrict__ K,
                        const float* __restrict__ g_transl, float* __restrict__ d_rot, float* __restrict__ d_shape,
                        float* __restrict__ d_expr, float* __restrict__ d_transl, float* __restrict__ d_loc,
                        float* __restrict__ d_dist, float* __restrict__ d_R) {
  constexpr int kPSMax = NJ * 12 + kKTMax + 12;
  __shared__ float red[kPSMax];
  __shared__ float Rs[NJ][9], GR[NJ][9], Js[NJ][3];
  __shared__ float gGR[NJ][9], gGt[NJ][3], gJl[NJ][3], gR[NJ][9];
  __shared__ float beta[32], gcen[3];
  const int p = blockIdx.x, tid = threadIdx.x;
  const int L = num_betas + n_expr;
  for (int e = tid; e < PS; e += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < tiles; ++t) s += part[(static_cast<int64_t>(t) * P + p) * PS + e];
    red[e] = s;
  }
  if (tid < num_betas) beta[tid] = shape[p * num_betas + tid];
  if (tid >= 32 && tid < 32 + n_expr) beta[num_betas + (tid - 32)] = expr[p * n_expr + (tid - 32)];
  __syncthreads();
  float r3[3] = {0.f, 0.f, 0.f};
  if (tid < NJ) {
    const int j = tid;
    const int src = kRaw ? j : full_pose_source(j);
    if (src >= 0) {
      const float* rv = rotvec + (static_cast<int64_t>(p) * (kRaw ? NJ : 53) + src) * 3;
      r3[0] = rv[0]; r3[1] = rv[1]; r3[2] = rv[2];
    }
    // the forward's rotation (smplx.lbs.batch_rodrigues), its joints and the chain's rotations G_R = A[:, :3]
    const float ex = r3[0] + 1e-8f, ey = r3[1] + 1e-8f, ez = r3[2] + 1e-8f;
    const float ang = sqrtf(ex * ex + ey * ey + ez * ez);
    const float ax = r3[0] / ang, ay = r3[1] / ang, az = r3[2] / ang;
    const float s = sinf(ang), c1 = 1.f - cosf(ang);
    const float Kx[9] = {0.f, -az, ay, az, 0.f, -ax, -ay, ax, 0.f};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float kk = Kx[r * 3] * Kx[c] + Kx[r * 3 + 1] * Kx[3 + c] + Kx[r * 3 + 2] * Kx[6 + c];
        Rs[j][r * 3 + c] = ((r == c) ? 1.f : 0.f) + s * Kx[r * 3 + c] + c1 * kk;
        GR[j][r * 3 + c] = Amat[(static_cast<int64_t>(p) * NJ + j) * 12 + r * 4 + c];
      }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float v = Jt[j * 3 + r];
      for (int l = 0; l < L; ++l) v += Jdirs[(j * 3 + r) * L + l] * beta[l];
      Js[j][r] = v;
    }
  }
  const float* gJp = gJ + static_cast<int64_t>(p) * J * 3;
  const float* X = xf + static_cast<int64_t>(p) * 16;
  const float* jp = jposed + static_cast<int64_t>(p) * NJ * 3;
  if (tid == NJ) {
    // placement: every output point o = R_root (x - J_centre) + transl (the pelvis cancels), x the posed LBS point
    const float* Sv = red + NJ * 12 + KT;
    float S[3] = {Sv[0], Sv[1], Sv[2]};
    for (int j = 0; j < NJ; ++j) {
      S[0] += gJp[j * 3]; S[1] += gJp[j * 3 + 1]; S[2] += gJp[j * 3 + 2];
    }
    if (kRaw) {
      d_transl[p * 3] = S[0]; d_transl[p * 3 + 1] = S[1]; d_transl[p * 3 + 2] = S[2];
    } else {
      const float* Mo = Sv + 3;
      const float* Jc = jp + center_idx * 3;
      float gRr[9];
#pragma unroll
      for (int m = 0; m < 3; ++m)
#pragma unroll
        for (int n = 0; n < 3; ++n) gRr[m * 3 + n] = Mo[m * 3 + n] - Sv[m] * Jc[n];
      for (int j = 0; j < NJ; ++j)
#pragma unroll
        for (int m = 0; m < 3; ++m)
#pragma unroll
          for (int n = 0; n < 3; ++n) gRr[m * 3 + n] += gJp[j * 3 + m] * (jp[j * 3 + n] - Jc[n]);
      const float* rv = rotvec + static_cast<int64_t>(p) * 53 * 3;
      rotvec_grad(rv[0], rv[1], rv[2], 0.f, true, gRr, d_rot + static_cast<int64_t>(p) * 53 * 3);
      if (d_R != nullptr) {
#pragma unroll
        for (int q = 0; q < 9; ++q) d_R[static_cast<int64_t>(p) * 53 * 9 + q] = gRr[q];
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) gcen[c] = -(X[c] * S[0] + X[3 + c] * S[1] + X[6 + c] * S[2]);
      // transl = K^-1 [loc, 1] dist (the inverse as loc_to_transl computes it)
      float gt[3] = {S[0], S[1], S[2]};
      if (g_transl != nullptr) { gt[0] += g_transl[p * 3]; gt[1] += g_transl[p * 3 + 1]; gt[2] += g_transl[p * 3 + 2]; }
      const float* m = K + p * 9;
      const float a = m[0], bb = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
      const float Ac = e * i - f * h, Bc = -(d * i - f * g), Cc = d * h - e * g;
      const float rr = 1.0f / (a * Ac + bb * Bc + c * Cc);
      const float inv[9] = {Ac * rr, -(bb * i - c * h) * rr, (bb * f - c * e) * rr,
                            Bc * rr, (a * i - c * g) * rr, -(a * f - c * d) * rr,
                            Cc * rr, -(a * h - bb * g) * rr, (a * e - bb * d) * rr};
      const float lx = loc[p * 2], ly = loc[p * 2 + 1], dd = dist[p];
      float gd = 0.f;
#pragma unroll
      for (int q = 0; q < 3; ++q) gd += (inv[q * 3] * lx + inv[q * 3 + 1] * ly + inv[q * 3 + 2]) * gt[q];
      d_dist[p] = gd;
      d_loc[p * 2] = (inv[0] * gt[0] + inv[3] * gt[1] + inv[6] * gt[2]) * dd;
      d_loc[p * 2 + 1] = (inv[1] * gt[0] + inv[4] * gt[1] + inv[7] * gt[2]) * dd;
    }
  }
  __syncthreads();
  if (tid < NJ) {
    // A_j = [G_R | G_t - G_R J_j], posed joint = G_t
    const int j = tid;
    float gx[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) gx[c] = X[c] * gJp[j * 3] + X[3 + c] * gJp[j * 3 + 1] + X[6 + c] * gJp[j * 3 + 2];
    if (!kRaw && j == center_idx) { gx[0] += gcen[0]; gx[1] += gcen[1]; gx[2] += gcen[2]; }
    const float* gA = red + j * 12;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      gGt[j][r] = gx[r] + gA[r * 4 + 3];
#pragma unroll
      for (int c = 0; c < 3; ++c) gGR[j][r * 3 + c] = gA[r * 4 + c] - gA[r * 4 + 3] * Js[j][c];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
      gJl[j][c] = -(GR[j][c] * gA[3] + GR[j][3 + c] * gA[7] + GR[j][6 + c] * gA[11]);
  }
  __syncthreads();
  if (tid == 0) {
    // kinematic chain in reverse: G_j = G_par [R_j | J_j - J_par]
    for (int j = NJ - 1; j >= 1; --j) {
      const int par = parents[j];
      const float t[3] = {Js[j][0] - Js[par][0], Js[j][1] - Js[par][1], Js[j][2] - Js[par][2]};
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b)
          gR[j][a * 3 + b] = GR[par][a] * gGR[j][b] + GR[par][3 + a] * gGR[j][3 + b] + GR[par][6 + a] * gGR[j][6 + b];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
          gGR[par][r * 3 + c] += gGR[j][r * 3] * Rs[j][c * 3] + gGR[j][r * 3 + 1] * Rs[j][c * 3 + 1] +
                                 gGR[j][r * 3 + 2] * Rs[j][c * 3 + 2] + gGt[j][r] * t[c];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float u = GR[par][c] * gGt[j][0] + GR[par][3 + c] * gGt[j][1] + GR[par][6 + c] * gGt[j][2];
        gJl[j][c] += u;
        gJl[par][c] -= u;
        gGt[par][c] += gGt[j][c];
      }
    }
#pragma unroll
    for (int q = 0; q < 9; ++q) gR[0][q] = gGR[0][q];
#pragma unroll
    for (int c = 0; c < 3; ++c) gJl[0][c] += gGt[0][c];
  }
  __syncthreads();
  if (tid < NJ) {
    const int j = tid;
    if (j >= 1) {
#pragma unroll
      for (int q = 0; q < 9; ++q) gR[j][q] += red[NJ * 12 + (j - 1) * 9 + q];  // pose feature R_j - I
    }
    float gr[3];
    rotvec_grad(r3[0], r3[1], r3[2], 1e-8f, false, gR[j], gr);
    const int src = kRaw ? j : full_pose_source(j);
    if (src >= 0) {
      float* o = d_rot + (static_cast<int64_t>(p) * (kRaw ? NJ : 53) + src) * 3;
      o[0] = gr[0]; o[1] = gr[1]; o[2] = gr[2];
      if (!kRaw && d_R != nullptr) {
#pragma unroll
        for (int q = 0; q < 9; ++q) d_R[(static_cast<int64_t>(p) * 53 + src) * 9 + q] = gR[j][q];
      }
    }
  }
  if (tid >= 64 && tid < 64 + L) {
    // beta enters the blend shapes (cf rows PF..) and the joints J = Jt + Jdirs beta
    const int l = tid - 64;
    float s = red[NJ * 12 + PF + l];
    for (int q = 0; q < NJ * 3; ++q) s = fmaf(Jdirs[q * L + l], gJl[q / 3][q % 3], s);
    if (l < num_betas) d_shape[p * num_betas + l] = s;
    else if (d_expr != nullptr) d_expr[p * n_expr + (l - num_betas)] = s;
  }
}

__global__ void set_count_kernel(int* count, int P) { *count = P; }

template <int NJ, int PF, int NL, int PB, bool kRaw>
int body_backward_impl(const SmplxDeviceModel& bm, SmplxGradScratch& gs, int P, const float* rotvec,
                       const float* shape, const float* expr, const float* transl, const float* K,
                       const BodyGrads& g, const float* loc, const float* dist, const float* g_transl, float* d_rot,
                       float* d_shape, float* d_expr, float* d_transl, float* d_loc, float* d_dist, float* d_R,
                       cudaStream_t st) {
  const int KT = PF + bm.L, J = NJ + 21 + NL, V = bm.V;
  MHMR_REQUIRE(KT <= kKTMax, "smplx: too many blend-shape coefficients");
  MHMR_REQUIRE(bm.num_joints == NJ && bm.pose_feat == PF && bm.n_lmk == NL, "body model / kernel shape mismatch");
  MHMR_REQUIRE(P <= gs.max_persons, "P exceeds the gradient scratch");
  const int tiles = (V + kGTV - 1) / kGTV;
  const int PS = NJ * 12 + KT + 12;
  set_count_kernel<<<1, 1, 0, st>>>(gs.count, P);
  MHMR_CUDA_CHECK(cudaGetLastError());
  const bool need_fwd = g.v2d != nullptr || g.j2d != nullptr;  // projections need the forward's points
  if (need_fwd) {
    TRY(body_forward_impl<NJ, PF, NL, PB, kRaw>(bm, rotvec, shape, expr, transl, K, gs.count, P, gs.fw, gs.v3d,
                                                nullptr, gs.j3d, gs.j2d, gs.tp, st));
  } else {
    body_prep_kernel<NJ, PF, kRaw><<<P, 64, 0, st>>>(rotvec, shape, expr, bm.L - bm.num_betas, bm.Jt, bm.Jdirs,
                                                     bm.parents, gs.count, bm.num_betas, bm.center_idx, KT, gs.fw.cf,
                                                     gs.fw.Amat, gs.fw.xf, gs.fw.jposed);
    MHMR_CUDA_CHECK(cudaGetLastError());
  }
  body_grad_joints_kernel<<<P, 128, 0, st>>>(gs.j3d, K, g.j3d, g.j2d, g.tp, J, gs.gJ);
  MHMR_CUDA_CHECK(cudaGetLastError());
  static PerDeviceOnce once;
  const int smem = static_cast<int>(sizeof(GradSmem<NJ>)) + 16;
  if (once.first()) {
    MHMR_CUDA_CHECK(cudaFuncSetAttribute(body_grad_stream_kernel<NJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  }
  body_grad_stream_kernel<NJ><<<tiles, kGThreads, smem, st>>>(
      bm.PDX, bm.ldp, KT, bm.vt, bm.lbs_weights_padded, gs.fw.cf, gs.fw.Amat, gs.fw.xf, K, gs.v3d, g.v3d, g.v2d, gs.gJ,
      J, gs.v2j_ptr, gs.v2j_jt, gs.v2j_w, P, V, PS, gs.part);
  MHMR_CUDA_CHECK(cudaGetLastError());
  body_grad_person_kernel<NJ, PF, kRaw><<<P, 256, 0, st>>>(
      rotvec, shape, expr, bm.L - bm.num_betas, bm.Jt, bm.Jdirs, bm.parents, bm.num_betas, bm.center_idx, KT,
      gs.fw.Amat, gs.fw.jposed, gs.fw.xf, gs.gJ, J, gs.part, tiles, P, PS, loc, dist, K, g_transl, d_rot, d_shape,
      d_expr, d_transl, d_loc, d_dist, d_R);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

}  // namespace

int smplx_grad_init(DeviceBody* b, int max_persons, cudaStream_t st) {
  const SmplxDeviceModel& bm = b->bm;
  SmplxGradScratch* gs = &b->gs;
  const int V = bm.V, NJ = bm.num_joints, KT = bm.pose_feat + bm.L, NL = bm.n_lmk, J = NJ + 21 + NL;
  const int Pm = max_persons, tiles = (V + kGTV - 1) / kGTV;
  // vertex -> output-joint table (vertex-picked joints, then the landmark corners), built on the host in joint order
  MHMR_CUDA_CHECK(cudaStreamSynchronize(st));
  std::vector<int32_t> ext(21), tri(3 * NL);
  std::vector<float> bary(3 * NL);
  MHMR_CUDA_CHECK(cudaMemcpy(ext.data(), bm.extra_idx, 21 * 4, cudaMemcpyDeviceToHost));
  if (NL) {
    MHMR_CUDA_CHECK(cudaMemcpy(tri.data(), bm.lmk_tri, 3 * NL * 4, cudaMemcpyDeviceToHost));
    MHMR_CUDA_CHECK(cudaMemcpy(bary.data(), bm.lmk_bary, 3 * NL * 4, cudaMemcpyDeviceToHost));
  }
  std::vector<std::vector<std::pair<int, float>>> rows(V);
  for (int e = 0; e < 21; ++e) rows[ext[e]].push_back({NJ + e, 1.f});
  for (int l = 0; l < NL; ++l)
    for (int f = 0; f < 3; ++f) rows[tri[l * 3 + f]].push_back({NJ + 21 + l, bary[l * 3 + f]});
  std::vector<int32_t> rp(V + 1, 0), jt;
  std::vector<float> w;
  for (int v = 0; v < V; ++v) {
    for (const auto& e : rows[v]) { jt.push_back(e.first); w.push_back(e.second); }
    rp[v + 1] = static_cast<int32_t>(jt.size());
  }
  const size_t ne = jt.size();
  gs->max_persons = Pm;
  gs->part_bytes = static_cast<size_t>(tiles) * Pm * (NJ * 12 + KT + 12) * 4;
  TRY(b->alloc(&gs->fw.cf, static_cast<size_t>(Pm) * KT, st));
  TRY(b->alloc(&gs->fw.Amat, static_cast<size_t>(Pm) * NJ * 12, st));
  TRY(b->alloc(&gs->fw.xf, static_cast<size_t>(Pm) * 16, st));
  TRY(b->alloc(&gs->fw.jposed, static_cast<size_t>(Pm) * NJ * 3, st));
  TRY(b->alloc(&gs->v3d, static_cast<size_t>(Pm) * V * 3, st));
  TRY(b->alloc(&gs->j3d, static_cast<size_t>(Pm) * J * 3, st));
  TRY(b->alloc(&gs->j2d, static_cast<size_t>(Pm) * J * 2, st));
  TRY(b->alloc(&gs->tp, static_cast<size_t>(Pm) * 3, st));
  TRY(b->alloc(&gs->transl, static_cast<size_t>(Pm) * 3, st));
  TRY(b->alloc(&gs->gJ, static_cast<size_t>(Pm) * J * 3, st));
  TRY(b->alloc(&gs->part, gs->part_bytes / 4, st));
  TRY(b->alloc(&gs->count, 1, st));
  TRY(b->alloc(&gs->v2j_ptr, V + 1, st));
  TRY(b->alloc(&gs->v2j_jt, ne > 0 ? ne : 1, st));
  TRY(b->alloc(&gs->v2j_w, ne > 0 ? ne : 1, st));
  // on `st`, after the zero-fills; the host tables live until the synchronisation
  MHMR_CUDA_CHECK(cudaMemcpyAsync(gs->v2j_ptr, rp.data(), (V + 1) * 4, cudaMemcpyHostToDevice, st));
  if (ne) {
    MHMR_CUDA_CHECK(cudaMemcpyAsync(gs->v2j_jt, jt.data(), ne * 4, cudaMemcpyHostToDevice, st));
    MHMR_CUDA_CHECK(cudaMemcpyAsync(gs->v2j_w, w.data(), ne * 4, cudaMemcpyHostToDevice, st));
  }
  MHMR_CUDA_CHECK(cudaStreamSynchronize(st));
  return MHMR_OK;
}

int smplx_backward(const SmplxDeviceModel& bm, SmplxGradScratch& gs, int P, const float* rotvec, const float* shape,
                   const float* expr, const float* loc, const float* dist, const float* K_det, const BodyGrads& g,
                   const float* g_transl, float* d_rotvec, float* d_shape, float* d_expr, float* d_loc, float* d_dist,
                   cudaStream_t st, float* d_rotmat) {
  TRY(loc_to_transl(loc, dist, K_det, P, gs.transl, st));
  return body_backward_impl<kNJ, kPoseFeat, 51, 16, false>(bm, gs, P, rotvec, shape, expr, gs.transl, K_det, g, loc,
                                                           dist, g_transl, d_rotvec, d_shape, d_expr, nullptr, d_loc,
                                                           d_dist, d_rotmat, st);
}

int body_backward_raw(const SmplxDeviceModel& bm, SmplxGradScratch& gs, int P, const float* full_pose,
                      const float* betas, const float* expr, const float* transl, const float* K, const BodyGrads& g,
                      float* d_full_pose, float* d_betas, float* d_expr, float* d_transl, cudaStream_t st) {
  if (bm.num_joints == 24)
    return body_backward_impl<24, 207, 0, 8, true>(bm, gs, P, full_pose, betas, expr, transl, K, g, nullptr, nullptr,
                                                   nullptr, d_full_pose, d_betas, d_expr, d_transl, nullptr, nullptr,
                                                   nullptr, st);
  if (bm.num_joints == kNJ)
    return body_backward_impl<kNJ, kPoseFeat, 51, 16, true>(bm, gs, P, full_pose, betas, expr, transl, K, g, nullptr,
                                                            nullptr, nullptr, d_full_pose, d_betas, d_expr, d_transl,
                                                            nullptr, nullptr, nullptr, st);
  set_last_error("body model: only SMPL (24 joints) and SMPL-X (55 joints) are instantiated");
  return MHMR_ERR_UNSUPPORTED;
}

}  // namespace mhmr
