// Training loss of the SMPL-X head (reference loss.py:47-115, scored on a forced-index forward as train.py:292-300 does)
// and its gradient with respect to the head's last Linears (DESIGN.md §10):
//
//   loss_partials_kernel   one CTA per chunk of one term: fp64 sums of |d| (and of the 2-D validity counts, of the
//                          focal loss' positive / negative parts and positives) in a fixed thread mapping
//   loss_finalize_kernel   one warp: each term's chunks summed in chunk order, nan_to_num, the weighted total, and the
//                          per-term gradient scale (alpha / count, 0 for a replaced term or a 2-D term before its epoch)
//   point_grad_kernel      upstream gradients of v3d / j3d / v2d / j2d for the SMPL-X backward
//   person_grad_kernel     per person: the pelvis gradient (sign counts, exact in int), transl, K_det
//   (smplx_backward)       the SMPL-X layer's backward, with the gradient of each joint's rotation matrix
//   dec_grad_kernel        per person: Gram-Schmidt backward of the 53 6D rows, betas, cam (dist chain), expression,
//                          offset (+ 14 d_loc)
//   logit_grad_kernel      focal-loss gradient through the clamped sigmoid of every cell
// No float atomics: every sum has a fixed order, so repeated calls are bitwise identical.
#include "kernels.cuh"

using namespace mhmr;

namespace {

constexpr int kJ = 127, kRot = 53, kThreads = 256, kChunk = 8192;
enum Term { T_BCE, T_OFFSET, T_ROTMAT, T_SHAPE, T_DIST, T_TRANSL, T_J3D, T_V3D, T_J2D, T_V2D, T_N };

struct Chunks {
  int64_t n[T_N];   // work units of each term
  int first[T_N + 1];  // first chunk of each term; first[T_N] = all chunks
};

struct LossPtrs {
  const float *s_hat, *s_gt, *off_hat, *off_gt, *R_hat, *R_gt, *sh_hat, *sh_gt, *dpp_hat, *dpp_gt, *tr_hat, *tr_gt,
      *tp_hat, *tp_gt, *j3_hat, *j3_gt, *v3_hat, *v3_gt, *j2_hat, *j2_gt, *v2_hat, *v2_gt;
  int nb, nb_gt, nb_min, V;
  float img_size;
};

__device__ __forceinline__ float sgnf(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }
// d|d|/d(pred) scaled by the term's coefficient; a zero coefficient (replaced term) gives 0 even for non-finite d
__device__ __forceinline__ float l1g(float coef, float d) { return coef != 0.f ? coef * sgnf(d) : 0.f; }
// strictly inside (0, img_size) on both axes (loss.py:70,72)
__device__ __forceinline__ bool valid2d(float x, float y, float S) { return x > 0.f && x < S && y > 0.f && y < S; }

__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < (blockDim.x >> 5); ++i) s += red[i];
  return s;  // valid on thread 0
}

// 3-D points relative to their own pelvis (loss.py:63-67): pred - target
__device__ __forceinline__ float d3(const float* hat, const float* gt, const float* tph, const float* tpg, int64_t e,
                                    int per) {
  const int64_t p = e / per;
  const int c = static_cast<int>(e % 3);
  return (hat[e] - tph[p * 3 + c]) - (gt[e] - tpg[p * 3 + c]);
}

__global__ void __launch_bounds__(kThreads)
loss_partials_kernel(LossPtrs a, Chunks ch, double* __restrict__ part) {
  __shared__ double red[kThreads / 32];
  const int c = blockIdx.x;
  int t = 0;
  while (c >= ch.first[t + 1]) ++t;
  const int64_t u0 = static_cast<int64_t>(c - ch.first[t]) * kChunk;
  const int64_t u1 = min(u0 + kChunk, ch.n[t]);
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  for (int64_t u = u0 + threadIdx.x; u < u1; u += blockDim.x) {
    switch (t) {
      case T_BCE: {  // _neg_loss (loss.py:8-40) with the binary target scores >= 1
        const float s = a.s_hat[u];
        if (a.s_gt[u] >= 1.f) {
          const float q = 1.f - s;
          s0 += static_cast<double>(logf(s + 1e-7f) * (q * q));
          s2 += 1.0;
        } else {
          s1 += static_cast<double>(logf(1.f - s + 1e-7f) * (s * s));
        }
        break;
      }
      case T_OFFSET: s0 += fabsf(a.off_hat[u] - a.off_gt[u]); break;
      case T_ROTMAT: s0 += fabsf(a.R_hat[u] - a.R_gt[u]); break;
      case T_SHAPE: {
        const int64_t p = u / a.nb_min, k = u % a.nb_min;
        s0 += fabsf(a.sh_hat[p * a.nb + k] - a.sh_gt[p * a.nb_gt + k]);
        break;
      }
      case T_DIST: s0 += fabsf(a.dpp_hat[u] - a.dpp_gt[u]); break;
      case T_TRANSL: s0 += fabsf(a.tr_hat[u] - a.tr_gt[u]); break;
      case T_J3D: s0 += fabsf(d3(a.j3_hat, a.j3_gt, a.tp_hat, a.tp_gt, u, kJ * 3)); break;
      case T_V3D: s0 += fabsf(d3(a.v3_hat, a.v3_gt, a.tp_hat, a.tp_gt, u, a.V * 3)); break;
      case T_J2D:
      case T_V2D: {
        const float* h = t == T_J2D ? a.j2_hat : a.v2_hat;
        const float* g = t == T_J2D ? a.j2_gt : a.v2_gt;
        if (valid2d(g[2 * u], g[2 * u + 1], a.img_size)) {
          s0 += static_cast<double>(fabsf(h[2 * u] - g[2 * u]) + fabsf(h[2 * u + 1] - g[2 * u + 1]));
          s1 += 1.0;
        }
        break;
      }
    }
  }
  s0 = block_sum(s0, red);
  s1 = block_sum(s1, red);
  s2 = block_sum(s2, red);
  if (threadIdx.x == 0) {
    part[c * 3] = s0; part[c * 3 + 1] = s1; part[c * 3 + 2] = s2;
  }
}

// loss [11] = total, terms in loss.py's dict order; coef [T_N] = d total / d (per-element |d|) of each term.
__global__ void loss_finalize_kernel(const double* __restrict__ part, Chunks ch, LossWeights w, int P, int V,
                                     int use_2d, float* __restrict__ loss, float* __restrict__ coef) {
  __shared__ double val[T_N], cf[T_N];
  const int t = threadIdx.x;
  if (t < T_N) {
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int c = ch.first[t]; c < ch.first[t + 1]; ++c) {
      s0 += part[c * 3]; s1 += part[c * 3 + 1]; s2 += part[c * 3 + 2];
    }
    const float alpha[T_N] = {w.bce, w.offset, w.rotmat, w.shape, w.dist, w.transl, w.j3d, w.v3d, w.j2d, w.v2d};
    double v, g;  // the term, and its derivative with respect to one element's |d| (bce: to pos / neg parts)
    if (t == T_BCE) {
      g = s2 == 0.0 ? -1.0 : -1.0 / s2;
      v = (s0 + s1) * g;
    } else {
      double n = static_cast<double>(P);  // mean over persons
      if (t == T_J3D) n *= kJ;
      if (t == T_V3D) n *= V;
      if (t == T_J2D || t == T_V2D) n = s1;  // mean over the valid points of all persons
      g = 1.0 / n;                           // n = 0: NaN below, replaced
      v = s0 * g;
    }
    const bool finite = isfinite(v);
    const bool on = t < T_J2D || use_2d;
    val[t] = finite ? v : 0.0;
    cf[t] = (finite && on) ? alpha[t] * g : 0.0;
    coef[t] = static_cast<float>(cf[t]);
    loss[1 + t] = static_cast<float>(val[t]);
  }
  __syncthreads();
  if (t == 0) {
    const float alpha[T_N] = {w.bce, w.offset, w.rotmat, w.shape, w.dist, w.transl, w.j3d, w.v3d, w.j2d, w.v2d};
    double total = 0.0;
    for (int k = 0; k < T_N; ++k)
      if (k < T_J2D || use_2d) total += static_cast<double>(alpha[k]) * val[k];
    loss[0] = static_cast<float>(total);
  }
}

// g_j3d [P,127,3], g_v3d [P,V,3], g_j2d [P,127,2], g_v2d [P,V,2] (2-D only when given)
__global__ void point_grad_kernel(LossPtrs a, const float* __restrict__ coef, int P, float* __restrict__ g_j3d,
                                  float* __restrict__ g_v3d, float* __restrict__ g_j2d, float* __restrict__ g_v2d) {
  const int64_t nj3 = static_cast<int64_t>(P) * kJ * 3, nv3 = static_cast<int64_t>(P) * a.V * 3;
  const int64_t nj2 = static_cast<int64_t>(P) * kJ, nv2 = static_cast<int64_t>(P) * a.V;
  const int64_t n = nj3 + nv3 + (g_j2d != nullptr ? nj2 + nv2 : 0);
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < n;
       e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    if (e < nj3) {
      g_j3d[e] = l1g(coef[T_J3D], d3(a.j3_hat, a.j3_gt, a.tp_hat, a.tp_gt, e, kJ * 3));
    } else if (e < nj3 + nv3) {
      const int64_t u = e - nj3;
      g_v3d[u] = l1g(coef[T_V3D], d3(a.v3_hat, a.v3_gt, a.tp_hat, a.tp_gt, u, a.V * 3));
    } else {
      int64_t u = e - nj3 - nv3;
      const bool j = u < nj2;
      if (!j) u -= nj2;
      const float* h = j ? a.j2_hat : a.v2_hat;
      const float* g = j ? a.j2_gt : a.v2_gt;
      float* o = j ? g_j2d : g_v2d;
      const float cf = valid2d(g[2 * u], g[2 * u + 1], a.img_size) ? coef[j ? T_J2D : T_V2D] : 0.f;
      o[2 * u] = l1g(cf, h[2 * u] - g[2 * u]);
      o[2 * u + 1] = l1g(cf, h[2 * u + 1] - g[2 * u + 1]);
    }
  }
}

// Per person: g_tp = -(sum of the 3-D points' gradients) (each point is taken relative to the pelvis); the sums are
// sign counts, exact in int32.  g_transl, and K_det[p] = K[det_b[p]] for the backward.
__global__ void __launch_bounds__(kThreads)
person_grad_kernel(LossPtrs a, const float* __restrict__ coef, const float* __restrict__ K,
                   const int* __restrict__ det_b, float* __restrict__ g_tp, float* __restrict__ g_tr,
                   float* __restrict__ K_det) {
  __shared__ int cnt[2][3];
  const int p = blockIdx.x;
  if (threadIdx.x < 6) cnt[threadIdx.x / 3][threadIdx.x % 3] = 0;
  __syncthreads();
  int cj[3] = {0, 0, 0}, cv[3] = {0, 0, 0};
  const int64_t base_j = static_cast<int64_t>(p) * kJ * 3, base_v = static_cast<int64_t>(p) * a.V * 3;
  for (int e = threadIdx.x; e < kJ * 3; e += blockDim.x)
    cj[e % 3] += static_cast<int>(sgnf(d3(a.j3_hat, a.j3_gt, a.tp_hat, a.tp_gt, base_j + e, kJ * 3)));
  for (int e = threadIdx.x; e < a.V * 3; e += blockDim.x)
    cv[e % 3] += static_cast<int>(sgnf(d3(a.v3_hat, a.v3_gt, a.tp_hat, a.tp_gt, base_v + e, a.V * 3)));
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    atomicAdd(&cnt[0][c], cj[c]);  // integer sums: the result does not depend on the order
    atomicAdd(&cnt[1][c], cv[c]);
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    const int c = threadIdx.x;
    const float cfj = coef[T_J3D], cfv = coef[T_V3D];
    g_tp[p * 3 + c] = -((cfj != 0.f ? cfj * static_cast<float>(cnt[0][c]) : 0.f) +
                        (cfv != 0.f ? cfv * static_cast<float>(cnt[1][c]) : 0.f));
    g_tr[p * 3 + c] = l1g(coef[T_TRANSL], a.tr_hat[p * 3 + c] - a.tr_gt[p * 3 + c]);
  } else if (threadIdx.x >= 32 && threadIdx.x < 41) {
    const int i = threadIdx.x - 32;
    K_det[p * 9 + i] = K[det_b[p] * 9 + i];
  }
}

// Backward of the engine's gram_schmidt (head.cu, roma.special_gramschmidt of utils/humans.py:12-22): 6D row x =
// (a, b), R = [e1 e2 e3] (columns), gradient G [3][3] row-major -> dx [6].
__device__ __forceinline__ void gram_schmidt_grad(const float* x, const float* G, float* dx) {
  float e1[3] = {x[0], x[1], x[2]}, b[3] = {x[3], x[4], x[5]};
  const float na = sqrtf(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
  e1[0] /= na; e1[1] /= na; e1[2] /= na;
  const float dp = e1[0] * b[0] + e1[1] * b[1] + e1[2] * b[2];
  float e2[3] = {b[0] - dp * e1[0], b[1] - dp * e1[1], b[2] - dp * e1[2]};
  const float nb = sqrtf(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
  e2[0] /= nb; e2[1] /= nb; e2[2] /= nb;
  const float g1[3] = {G[0], G[3], G[6]}, g2[3] = {G[1], G[4], G[7]}, g3[3] = {G[2], G[5], G[8]};
  // e3 = e1 x e2: <g3, de1 x e2> = <e2 x g3, de1>, <g3, e1 x de2> = <g3 x e1, de2>
  float ge1[3] = {g1[0] + (e2[1] * g3[2] - e2[2] * g3[1]), g1[1] + (e2[2] * g3[0] - e2[0] * g3[2]),
                  g1[2] + (e2[0] * g3[1] - e2[1] * g3[0])};
  const float ge2[3] = {g2[0] + (g3[1] * e1[2] - g3[2] * e1[1]), g2[1] + (g3[2] * e1[0] - g3[0] * e1[2]),
                        g2[2] + (g3[0] * e1[1] - g3[1] * e1[0])};
  // e2 = b' / |b'|, b' = b - (e1.b) e1
  const float q2 = ge2[0] * e2[0] + ge2[1] * e2[1] + ge2[2] * e2[2];
  float gbp[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) gbp[i] = (ge2[i] - q2 * e2[i]) / nb;
  const float q = e1[0] * gbp[0] + e1[1] * gbp[1] + e1[2] * gbp[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    dx[3 + i] = gbp[i] - q * e1[i];
    ge1[i] -= dp * gbp[i] + q * b[i];
  }
  // e1 = a / |a|
  const float q1 = ge1[0] * e1[0] + ge1[1] * e1[1] + ge1[2] * e1[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) dx[i] = (ge1[i] - q1 * e1[i]) / na;
}

// d_dec [P, ld] and d_offset [P, 2] of one person per CTA.
__global__ void __launch_bounds__(128)
dec_grad_kernel(LossPtrs a, const float* __restrict__ coef, const float* __restrict__ dec, int ld,
                const float* __restrict__ K_det, float focal_norm, const float* __restrict__ dR,
                const float* __restrict__ d_shape, const float* __restrict__ d_expr, const float* __restrict__ d_loc,
                const float* __restrict__ d_dist, float* __restrict__ d_dec, float* __restrict__ d_offset) {
  const int p = blockIdx.x, t = threadIdx.x, nb = a.nb;
  const float* x = dec + static_cast<int64_t>(p) * ld;
  float* o = d_dec + static_cast<int64_t>(p) * ld;
  if (t < kRot) {
    const int64_t r = (static_cast<int64_t>(p) * kRot + t) * 9;
    float G[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) G[q] = dR[r + q] + l1g(coef[T_ROTMAT], a.R_hat[r + q] - a.R_gt[r + q]);
    float dx[6];
    gram_schmidt_grad(x + t * 6, G, dx);
#pragma unroll
    for (int i = 0; i < 6; ++i) o[t * 6 + i] = dx[i];
  } else if (t == kRot) {
    // dist = clamp(exp(cam0 f / fn) - 1e-10, 0, 50) as person_post computes it; zero gradient where clamped
    const float cam0 = x[318 + nb];
    const float sc = K_det[p * 9] / focal_norm;
    const float ex = expf(cam0 * sc);
    const float dd = ex - 1e-10f;
    const float chain = (dd >= 0.f && dd <= 50.f) ? d_dist[p] * ex * sc : 0.f;
    o[318 + nb] = chain + l1g(coef[T_DIST], cam0 - a.dpp_gt[p]);
    o[319 + nb] = 0.f;
    o[320 + nb] = 0.f;
    // loc = (cell + 0.5 + offset) * 14
#pragma unroll
    for (int c = 0; c < 2; ++c)
      d_offset[p * 2 + c] = l1g(coef[T_OFFSET], a.off_hat[p * 2 + c] - a.off_gt[p * 2 + c]) + 14.f * d_loc[p * 2 + c];
  } else if (t >= 64 && t < 64 + nb) {
    const int k = t - 64;
    const float direct =
        k < a.nb_min ? l1g(coef[T_SHAPE], a.sh_hat[p * nb + k] - a.sh_gt[p * a.nb_gt + k]) : 0.f;
    o[318 + k] = d_shape[p * nb + k] + direct;
  } else if (t >= 96 && t < 106) {
    o[321 + nb + (t - 96)] = d_expr[p * 10 + (t - 96)];
  }
}

// d_logits of every cell: focal loss through sigmoid clamped to [1e-4, 1 - 1e-4] (model.py:641-643)
__global__ void logit_grad_kernel(const float* __restrict__ s_hat, const float* __restrict__ s_gt,
                                  const float* __restrict__ coef, int n, float* __restrict__ d_logits) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float s = s_hat[i], cf = coef[T_BCE];
  float g = 0.f;
  if (cf != 0.f && s != 1e-4f && s != 1.0f - 1e-4f) {
    const float q = 1.f - s;
    const float ds = s_gt[i] >= 1.f ? q * q / (s + 1e-7f) - 2.f * q * logf(s + 1e-7f)
                                    : -(s * s) / (q + 1e-7f) + 2.f * s * logf(q + 1e-7f);
    g = cf * ds * (s * q);
  }
  d_logits[i] = g;
}

}  // namespace

namespace mhmr {

int train_loss_smplx(const SmplxDeviceModel& bm, SmplxGradScratch& gs, const TrainLossArgs& A, cudaStream_t st) {
  const mhmr_outputs& yh = *A.y_hat;
  const TrainTargets& y = A.y;
  const int P = A.P, V = bm.V, nb = bm.num_betas, BN = A.B * A.res * A.res;
  LossPtrs a;
  a.s_hat = yh.scores_map; a.s_gt = y.scores; a.off_hat = yh.offset; a.off_gt = y.offset;
  a.R_hat = yh.rotmat; a.R_gt = y.rotmat; a.sh_hat = yh.shape; a.sh_gt = y.shape;
  a.dpp_hat = yh.dist_pp; a.dpp_gt = y.dist_pp; a.tr_hat = yh.transl; a.tr_gt = y.transl;
  a.tp_hat = yh.transl_pelvis; a.tp_gt = y.transl_pelvis; a.j3_hat = yh.j3d; a.j3_gt = y.j3d;
  a.v3_hat = yh.v3d; a.v3_gt = y.v3d; a.j2_hat = yh.j2d; a.j2_gt = y.j2d; a.v2_hat = yh.v2d; a.v2_gt = y.v2d;
  a.nb = nb; a.nb_gt = y.shape_dim; a.nb_min = nb < y.shape_dim ? nb : y.shape_dim; a.V = V;
  a.img_size = static_cast<float>(A.img_size);

  // the SMPL-X backward's own requirements, before any launch
  MHMR_REQUIRE(P <= gs.max_persons, "P exceeds the gradient scratch");
  MHMR_REQUIRE(bm.num_joints == 55 && bm.n_lmk == 51, "mhmr_train_loss needs the SMPL-X layer (55 joints, 51 landmarks)");
  Chunks ch;
  const int64_t n[T_N] = {BN, 2ll * P, 9ll * kRot * P, static_cast<int64_t>(a.nb_min) * P, P, 3ll * P,
                          3ll * kJ * P, 3ll * V * P, static_cast<int64_t>(kJ) * P, static_cast<int64_t>(V) * P};
  ch.first[0] = 0;
  for (int t = 0; t < T_N; ++t) {
    ch.n[t] = n[t];
    ch.first[t + 1] = ch.first[t] + static_cast<int>((n[t] + kChunk - 1) / kChunk);
  }
  const int chunks = ch.first[T_N];

  // stream-ordered scratch: fp64 partials, then fp32 coefficients, upstream and intermediate gradients
  const size_t Pz = static_cast<size_t>(P);
  CallScratch ws(st);
  const size_t r_part = ws.region(chunks * 3 * sizeof(double));
  auto f32 = [&ws](size_t n) { return ws.region(n * 4); };
  const size_t r_coef = f32(16), r_j3d = f32(Pz * kJ * 3), r_v3d = f32(Pz * V * 3), r_j2d = f32(Pz * kJ * 2),
               r_v2d = f32(Pz * V * 2), r_tp = f32(Pz * 3), r_tr = f32(Pz * 3), r_K = f32(Pz * 9),
               r_rotvec = f32(Pz * kRot * 3), r_dR = f32(Pz * kRot * 9), r_shape = f32(Pz * nb), r_expr = f32(Pz * 10),
               r_loc = f32(Pz * 2), r_dist = f32(Pz);
  TRY(ws.allocate());
  double* part = ws.dev<double>(r_part);
  float *coef = ws.dev<float>(r_coef), *g_j3d = ws.dev<float>(r_j3d), *g_v3d = ws.dev<float>(r_v3d),
        *g_j2d = ws.dev<float>(r_j2d), *g_v2d = ws.dev<float>(r_v2d), *g_tp = ws.dev<float>(r_tp),
        *g_tr = ws.dev<float>(r_tr), *K_det = ws.dev<float>(r_K), *d_rotvec = ws.dev<float>(r_rotvec),
        *dR = ws.dev<float>(r_dR), *d_shape = ws.dev<float>(r_shape), *d_expr = ws.dev<float>(r_expr),
        *d_loc = ws.dev<float>(r_loc), *d_dist = ws.dev<float>(r_dist);

  loss_partials_kernel<<<chunks, kThreads, 0, st>>>(a, ch, part);
  MHMR_CUDA_CHECK(cudaGetLastError());
  loss_finalize_kernel<<<1, 32, 0, st>>>(part, ch, A.w, P, V, A.use_2d, A.loss, coef);
  MHMR_CUDA_CHECK(cudaGetLastError());
  logit_grad_kernel<<<(BN + 255) / 256, 256, 0, st>>>(a.s_hat, a.s_gt, coef, BN, A.d_logits);
  MHMR_CUDA_CHECK(cudaGetLastError());
  if (P > 0) {
    const bool two_d = A.use_2d != 0;
    point_grad_kernel<<<1056, 256, 0, st>>>(a, coef, P, g_j3d, g_v3d, two_d ? g_j2d : nullptr,
                                             two_d ? g_v2d : nullptr);
    MHMR_CUDA_CHECK(cudaGetLastError());
    person_grad_kernel<<<P, kThreads, 0, st>>>(a, coef, A.K, yh.det_idx, g_tp, g_tr, K_det);
    MHMR_CUDA_CHECK(cudaGetLastError());
    BodyGrads g;
    g.v3d = g_v3d; g.j3d = g_j3d; g.tp = g_tp;
    if (two_d) { g.v2d = g_v2d; g.j2d = g_j2d; }
    TRY(smplx_backward(bm, gs, P, yh.rotvec, yh.shape, yh.expression, yh.loc, yh.dist, K_det, g, g_tr, d_rotvec, d_shape,
                       d_expr, d_loc, d_dist, st, dR));
    const float focal_norm = static_cast<float>(A.img_size / (2.0 * tan(30.0 * 3.14159265358979323846 / 180.0)));
    dec_grad_kernel<<<P, 128, 0, st>>>(a, coef, yh.dec, 318 + nb + 13, K_det, focal_norm, dR, d_shape, d_expr, d_loc,
                                       d_dist, A.d_dec, A.d_offset);
    MHMR_CUDA_CHECK(cudaGetLastError());
  }
  return ws.release();
}

}  // namespace mhmr
