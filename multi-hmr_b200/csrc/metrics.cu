// Evaluation metrics of the caller that turns Model.forward outputs into the README's numbers
// (reference Trainer.evaluate, train.py:336-482; helpers utils/training.py:9-193): SURVEY.md §8(f) row 3.
//
//   mhmr_eval_match_2d      greedy matching of predicted to ground-truth persons on 2-D joints
//                           (utils/training.py:25-147 `match_2d_greedy` with valid=None, IoU gate :149-193)
//   mhmr_eval_points_error  per matched pair: mean point error in mm (PVE / MPJPE, train.py:387,419) and the same
//                           after the Procrustes similarity alignment (PA-PVE / PA-MPJPE, train.py:391-393,
//                           roma.rigid_points_registration(compute_scaling=True))
//   mhmr_eval_regress       per matched pair: a sparse regressor applied to the centred points (SMPL-X -> SMPL
//                           transfer, train.py:383-384; H36M joints, :406-415; EHF joints, :73)
// The matched pairs stay on the device between the two calls (no host round trip inside one image's evaluation).
// Latency-bound kernels on a few persons: one CTA for the matching, one CTA per matched pair for the errors.
#include "kernels.cuh"

using namespace mhmr;

namespace {

constexpr int kMaxPersons = 48;  // per image, predictions and ground truths (static smem: 48 KB)

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// err[p*G+g] = largest singular value of the [J,2] matrix of joint differences (np.linalg.norm(D, 2) of a MATRIX,
// utils/training.py:50); iou[p*G+g] = IoU of the joint bounding boxes with the +1 pixel convention (:149-193).
__global__ void __launch_bounds__(256)
match_2d_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const uint8_t* __restrict__ vmask,
                int P, int G, int J, float iou_thresh, int* __restrict__ pairs, int* __restrict__ n_pairs,
                int* __restrict__ pred_to_gt, int* __restrict__ gt_to_pred) {
  __shared__ double err[kMaxPersons * kMaxPersons];
  __shared__ float iou[kMaxPersons * kMaxPersons];
  __shared__ float box[2 * kMaxPersons][4];  // x1, y1, x2, y2 of every prediction then every ground truth
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int i = warp; i < P + G; i += nw) {
    const float* pts = (i < P) ? pred + static_cast<int64_t>(i) * J * 2 : gt + static_cast<int64_t>(i - P) * J * 2;
    float x1 = INFINITY, y1 = INFINITY, x2 = -INFINITY, y2 = -INFINITY;
    for (int j = lane; j < J; j += 32) {
      const float x = pts[2 * j], y = pts[2 * j + 1];
      x1 = fminf(x1, x); x2 = fmaxf(x2, x); y1 = fminf(y1, y); y2 = fmaxf(y2, y);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      x1 = fminf(x1, __shfl_xor_sync(0xffffffffu, x1, o));
      y1 = fminf(y1, __shfl_xor_sync(0xffffffffu, y1, o));
      x2 = fmaxf(x2, __shfl_xor_sync(0xffffffffu, x2, o));
      y2 = fmaxf(y2, __shfl_xor_sync(0xffffffffu, y2, o));
    }
    if (lane == 0) { box[i][0] = x1; box[i][1] = y1; box[i][2] = x2; box[i][3] = y2; }
  }
  for (int c = warp; c < P * G; c += nw) {
    const int p = c / G, g = c - p * G;
    const float* a = pred + static_cast<int64_t>(p) * J * 2;
    const float* b = gt + static_cast<int64_t>(g) * J * 2;
    double sxx = 0.0, sxy = 0.0, syy = 0.0;
    for (int j = lane; j < J; j += 32) {
      if (vmask != nullptr && vmask[g * J + j] == 0) continue;
      const double dx = static_cast<double>(a[2 * j]) - b[2 * j], dy = static_cast<double>(a[2 * j + 1]) - b[2 * j + 1];
      sxx += dx * dx; sxy += dx * dy; syy += dy * dy;
    }
    sxx = warp_sum_d(sxx); sxy = warp_sum_d(sxy); syy = warp_sum_d(syy);
    if (lane == 0) {
      const double h = 0.5 * (sxx - syy);
      err[c] = sqrt(0.5 * (sxx + syy) + sqrt(h * h + sxy * sxy));  // sqrt of the largest eigenvalue of D^T D
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < P * G; c += blockDim.x) {
    const int p = c / G, g = c - p * G;
    const float* b1 = box[p];
    const float* b2 = box[P + g];
    const float xl = fmaxf(b1[0], b2[0]), yt = fmaxf(b1[1], b2[1]), xr = fminf(b1[2], b2[2]), yb = fminf(b1[3], b2[3]);
    const float inter = fmaxf(0.f, xr - xl + 1.f) * fmaxf(0.f, yb - yt + 1.f);
    const float a1 = (b1[2] - b1[0] + 1.f) * (b1[3] - b1[1] + 1.f), a2 = (b2[2] - b2[0] + 1.f) * (b2[3] - b2[1] + 1.f);
    iou[c] = inter / (a1 + a2 - inter);
  }
  for (int p = threadIdx.x; p < P; p += blockDim.x) pred_to_gt[p] = -1;
  for (int g = threadIdx.x; g < G; g += blockDim.x) gt_to_pred[g] = -1;
  __syncthreads();
  if (threadIdx.x != 0) return;
  // the sequential greedy loop of utils/training.py:60-109 (valid=None)
  int n_gt = 0, n_op = 0, n_fp = 0, n = 0;
  while (n_gt < G && n_op + n_fp < P) {
    bool found = false, false_positive = false;
    int p = -1, g = -1;
    while (!found) {
      int best = -1;
      double bv = INFINITY;
      for (int c = 0; c < P * G; ++c)
        if (err[c] < bv) { bv = err[c]; best = c; }  // first minimum, like np.argmin
      if (best < 0) break;  // every pair consumed (the reference would spin here)
      p = best / G; g = best - p * G;
      err[best] = INFINITY;
      if (pred_to_gt[p] < 0 && gt_to_pred[g] < 0 && iou[best] >= iou_thresh) {
        found = true;
      } else if (iou[best] < iou_thresh) {
        found = true; false_positive = true; ++n_fp;
      }
    }
    if (!found) break;
    if (!false_positive) {
      pairs[2 * n] = p; pairs[2 * n + 1] = g; ++n;
      pred_to_gt[p] = g; gt_to_pred[g] = p;
      ++n_op; ++n_gt;
    }
  }
  *n_pairs = n;
}

// Symmetric 3x3 eigen-decomposition (cyclic Jacobi, double): A = V diag(w) V^T, eigenvalues sorted descending.
__device__ void eig_sym3(double A[3][3], double V[3][3], double w[3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; ++sweep) {
    const double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
    if (off < 1e-300) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (fabs(A[p][q]) < 1e-300) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = ((theta >= 0) ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < 3; ++i) w[i] = A[i][i];
  for (int i = 0; i < 2; ++i)
    for (int j = i + 1; j < 3; ++j)
      if (w[j] > w[i]) {
        const double tw = w[i]; w[i] = w[j]; w[j] = tw;
        for (int k = 0; k < 3; ++k) { const double tv = V[k][i]; V[k][i] = V[k][j]; V[k][j] = tv; }
      }
}

__device__ __forceinline__ double det3(const double M[3][3]) {
  return M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0]) +
         M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
}

// Similarity (R, t, s) minimising sum |s R x_i + t - y_i|^2 from the centred cross-covariance M = sum yhat xhat^T
// and sxx = sum |xhat|^2 (roma.rigid_points_registration + special_procrustes: SVD with the reflection fix on the
// smallest singular direction).
__device__ void procrustes_from_cov(double M[3][3], double sxx, const double xm[3], const double ym[3], double R[3][3],
                                    double t[3], double* s) {
  double A[3][3], V[3][3], w[3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A[i][j] = M[0][i] * M[0][j] + M[1][i] * M[1][j] + M[2][i] * M[2][j];  // M^T M
  eig_sym3(A, V, w);
  double sig[3], U[3][3];
  for (int k = 0; k < 3; ++k) sig[k] = sqrt(fmax(w[k], 0.0));
  for (int k = 0; k < 2; ++k) {  // u_k = M v_k / sigma_k (the two leading directions)
    double n = 0.0, u[3];
    for (int i = 0; i < 3; ++i) { u[i] = M[i][0] * V[0][k] + M[i][1] * V[1][k] + M[i][2] * V[2][k]; n += u[i] * u[i]; }
    n = sqrt(n);
    for (int i = 0; i < 3; ++i) U[i][k] = (n > 0) ? u[i] / n : ((i == k) ? 1.0 : 0.0);
  }
  // Gram-Schmidt the second against the first (degenerate inputs), third = +-cross so that the reflection is explicit
  double d01 = U[0][0] * U[0][1] + U[1][0] * U[1][1] + U[2][0] * U[2][1], n1 = 0.0;
  for (int i = 0; i < 3; ++i) { U[i][1] -= d01 * U[i][0]; n1 += U[i][1] * U[i][1]; }
  n1 = sqrt(n1);
  for (int i = 0; i < 3; ++i) U[i][1] = (n1 > 0) ? U[i][1] / n1 : U[i][1];
  // with R = U diag(1, 1, det(U) det(V)) V^T the sign of the third column of U cancels: take u3 = u1 x u2
  U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
  U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
  U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
  // sign of the third singular value in the DECOMPOSITION M = U S V^T with this U: (u3^T M v3) may be negative
  double u3Mv3 = 0.0;
  for (int i = 0; i < 3; ++i) u3Mv3 += U[i][2] * (M[i][0] * V[0][2] + M[i][1] * V[1][2] + M[i][2] * V[2][2]);
  const double detV = det3(V);  // det(U) = +1 by construction
  // LAPACK's U would have u3 flipped when u3Mv3 < 0 (singular values are non-negative): det(U_lapack) = sign(u3Mv3)
  const double su = (u3Mv3 < 0) ? -1.0 : 1.0;
  const double d = su * detV;  // det(U_lapack) * det(V)
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      R[i][j] = U[i][0] * V[j][0] + U[i][1] * V[j][1] + d * su * U[i][2] * V[j][2];
  *s = (sig[0] + sig[1] + d * sig[2]) / sxx;
  for (int i = 0; i < 3; ++i) t[i] = ym[i] - (*s) * (R[i][0] * xm[0] + R[i][1] * xm[1] + R[i][2] * xm[2]);
}

__device__ __forceinline__ double block_sum_d(double v, double* red) {
  v = warp_sum_d(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double tot = 0.0;
  for (int w = 0; w < (blockDim.x >> 5); ++w) tot += red[w];
  return tot;
}

// one CTA per matched pair m < *n_pairs
__global__ void __launch_bounds__(256)
points_error_kernel(const float* __restrict__ pred, const float* __restrict__ pred_center,
                    const float* __restrict__ gt, const float* __restrict__ gt_center,
                    const int* __restrict__ pairs, const int* __restrict__ n_pairs, int n,
                    float* __restrict__ err_mm, float* __restrict__ pa_err_mm) {
  __shared__ double red[8];
  __shared__ double tr[13];  // R (9), t (3), s
  const int m = blockIdx.x;
  if (m >= *n_pairs) return;
  const int pid = pairs[2 * m], gid = pairs[2 * m + 1];
  const float* X = pred + static_cast<int64_t>(pid) * n * 3;
  const float* Y = gt + static_cast<int64_t>(gid) * n * 3;
  float cx[3] = {0.f, 0.f, 0.f}, cy[3] = {0.f, 0.f, 0.f};
  if (pred_center != nullptr) for (int i = 0; i < 3; ++i) cx[i] = pred_center[pid * 3 + i];
  if (gt_center != nullptr) for (int i = 0; i < 3; ++i) cy[i] = gt_center[gid * 3 + i];
  double sx[3] = {0, 0, 0}, sy[3] = {0, 0, 0}, e = 0.0;
  for (int v = threadIdx.x; v < n; v += blockDim.x) {
    float x[3], y[3];
    for (int i = 0; i < 3; ++i) { x[i] = X[3 * v + i] - cx[i]; y[i] = Y[3 * v + i] - cy[i]; sx[i] += x[i]; sy[i] += y[i]; }
    const float dx = y[0] - x[0], dy = y[1] - x[1], dz = y[2] - x[2];
    e += sqrtf(dx * dx + dy * dy + dz * dz);
  }
  double xm[3], ym[3];
  for (int i = 0; i < 3; ++i) { xm[i] = block_sum_d(sx[i], red) / n; ym[i] = block_sum_d(sy[i], red) / n; }
  e = block_sum_d(e, red);
  double M[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, sxx = 0.0;
  for (int v = threadIdx.x; v < n; v += blockDim.x) {
    double x[3], y[3];
    for (int i = 0; i < 3; ++i) { x[i] = (X[3 * v + i] - cx[i]) - xm[i]; y[i] = (Y[3 * v + i] - cy[i]) - ym[i]; }
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) M[i][j] += y[i] * x[j];
    sxx += x[0] * x[0] + x[1] * x[1] + x[2] * x[2];
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) M[i][j] = block_sum_d(M[i][j], red);
  sxx = block_sum_d(sxx, red);
  if (threadIdx.x == 0) {
    double R[3][3], t[3], s;
    procrustes_from_cov(M, sxx, xm, ym, R, t, &s);
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) tr[i * 3 + j] = R[i][j];
      tr[9 + i] = t[i];
    }
    tr[12] = s;
    err_mm[m] = static_cast<float>(e / n * 1000.0);
  }
  __syncthreads();
  double pe = 0.0;
  for (int v = threadIdx.x; v < n; v += blockDim.x) {
    double x[3], d2 = 0.0;
    for (int i = 0; i < 3; ++i) x[i] = X[3 * v + i] - cx[i];
    for (int i = 0; i < 3; ++i) {
      const double a = tr[12] * (tr[i * 3] * x[0] + tr[i * 3 + 1] * x[1] + tr[i * 3 + 2] * x[2]) + tr[9 + i];
      const double d = (Y[3 * v + i] - cy[i]) - a;
      d2 += d * d;
    }
    pe += sqrt(d2);
  }
  pe = block_sum_d(pe, red);
  if (threadIdx.x == 0) pa_err_mm[m] = static_cast<float>(pe / n * 1000.0);
}

// One warp per output row i of pair m: y_r = sum_k A[r, k] (X[src, k] - c[src]) for r = rows[i] (or i), minus y_root when
// root >= 0; src = pairs[2m + side].  Optional projection out2d[m, i] = (K[src] . (y / y_z))[:2] (utils/camera.py:14-27).
__device__ __forceinline__ void regress_row(const int* __restrict__ rowptr, const int* __restrict__ col,
                                            const float* __restrict__ val, int r, const float* __restrict__ X,
                                            const float c[3], int lane, float y[3]) {
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int e = rowptr[r] + lane; e < rowptr[r + 1]; e += 32) {
    const int k = col[e];
    const float w = val[e];
    a0 = fmaf(w, X[3 * k] - c[0], a0);
    a1 = fmaf(w, X[3 * k + 1] - c[1], a1);
    a2 = fmaf(w, X[3 * k + 2] - c[2], a2);
  }
  y[0] = warp_sum(a0);
  y[1] = warp_sum(a1);
  y[2] = warp_sum(a2);
}

__global__ void __launch_bounds__(256)
regress_pairs_kernel(const int* __restrict__ rowptr, const int* __restrict__ col, const float* __restrict__ val,
                     const int* __restrict__ rows, int R_out, int root, int N, const float* __restrict__ X,
                     const float* __restrict__ center, const int* __restrict__ pairs, int side,
                     const int* __restrict__ n_pairs, const float* __restrict__ K, float* __restrict__ out,
                     float* __restrict__ out2d) {
  const int m = blockIdx.y;
  if (m >= *n_pairs) return;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= R_out) return;
  const int src = pairs[2 * m + side];
  const float* Xs = X + static_cast<int64_t>(src) * N * 3;
  float c[3] = {0.f, 0.f, 0.f};
  if (center != nullptr) for (int q = 0; q < 3; ++q) c[q] = center[src * 3 + q];
  float y[3];
  regress_row(rowptr, col, val, rows != nullptr ? rows[i] : i, Xs, c, lane, y);
  if (root >= 0) {
    float y0[3];
    regress_row(rowptr, col, val, root, Xs, c, lane, y0);
    for (int q = 0; q < 3; ++q) y[q] -= y0[q];
  }
  if (lane != 0) return;
  float* o = out + (static_cast<int64_t>(m) * R_out + i) * 3;
  o[0] = y[0]; o[1] = y[1]; o[2] = y[2];
  if (out2d != nullptr) {
    const float* Kd = K + src * 9;
    const float u = y[0] / y[2], w = y[1] / y[2], one = y[2] / y[2];
    out2d[(static_cast<int64_t>(m) * R_out + i) * 2] = Kd[0] * u + Kd[1] * w + Kd[2] * one;
    out2d[(static_cast<int64_t>(m) * R_out + i) * 2 + 1] = Kd[3] * u + Kd[4] * w + Kd[5] * one;
  }
}

}  // namespace

extern "C" {

int mhmr_eval_regress(const int32_t* rowptr, const int32_t* col, const float* val, int R, int N, const int32_t* rows,
                      int R_out, int root, const float* X, const float* center, const int32_t* pairs, int side,
                      const int32_t* n_pairs, int max_pairs, const float* K, float* out, float* out2d, void* stream) {
  MHMR_REQUIRE(rowptr != nullptr && col != nullptr && val != nullptr && X != nullptr && pairs != nullptr &&
                   n_pairs != nullptr && out != nullptr, "null argument");
  MHMR_REQUIRE(R >= 1 && N >= 1 && R_out >= 1, "empty regressor");
  MHMR_REQUIRE(rows != nullptr || R_out == R, "without a row list every row of A is an output row");
  MHMR_REQUIRE(root >= -1 && root < R, "root row out of range");
  MHMR_REQUIRE(side == 0 || side == 1, "side selects the prediction (0) or ground-truth (1) column of pairs");
  MHMR_REQUIRE(max_pairs >= 1 && max_pairs <= kMaxPersons, "regression handles up to 48 pairs per image");
  MHMR_REQUIRE((out2d == nullptr) == (K == nullptr), "K and out2d go together");
  const dim3 grid((R_out + 7) / 8, max_pairs);
  regress_pairs_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      rowptr, col, val, rows, R_out, root, N, X, center, pairs, side, n_pairs, K, out, out2d);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}


int mhmr_eval_match_2d(const float* pred_j2d, const float* gt_j2d, const uint8_t* valid_mask, int P, int G, int J,
                       float iou_thresh, int32_t* pairs, int32_t* n_pairs, int32_t* pred_to_gt, int32_t* gt_to_pred,
                       void* stream) {
  MHMR_REQUIRE(gt_j2d != nullptr && pairs != nullptr && n_pairs != nullptr && pred_to_gt != nullptr &&
                   gt_to_pred != nullptr, "null argument");
  MHMR_REQUIRE(P >= 0 && G >= 1 && J >= 1 && P <= kMaxPersons && G <= kMaxPersons,
               "matching handles up to 48 predictions x 48 ground truths per image");
  MHMR_REQUIRE(P == 0 || pred_j2d != nullptr, "null predictions");
  match_2d_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(pred_j2d, gt_j2d, valid_mask, P, G, J, iou_thresh,
                                                                    pairs, n_pairs, pred_to_gt, gt_to_pred);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int mhmr_eval_points_error(const float* pred, const float* pred_center, const float* gt, const float* gt_center,
                           const int32_t* pairs, const int32_t* n_pairs, int max_pairs, int n_points, float* err_mm,
                           float* pa_err_mm, void* stream) {
  MHMR_REQUIRE(pred != nullptr && gt != nullptr && pairs != nullptr && n_pairs != nullptr && err_mm != nullptr &&
                   pa_err_mm != nullptr, "null argument");
  MHMR_REQUIRE(max_pairs >= 1 && n_points >= 3, "need at least one pair slot and three points");
  points_error_kernel<<<max_pairs, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      pred, pred_center, gt, gt_center, pairs, n_pairs, n_points, err_mm, pa_err_mm);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

}  // extern "C"
