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

}  // namespace mhmr
