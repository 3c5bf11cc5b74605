// Detection head, camera embedding and the HPH cross-attention decoder (query side) of Multi-HMR.
//
// Everything after the backbone that is not a big GEMM: these kernels are latency/HBM-bound, work on fp32
// activations with fp32 weights (the per-person path has ~26 MFLOP/person), keep the person count on the
// device (no host sync: grids are sized for max_persons and exit early) and emit persons in the
// reference's torch.where order (b, y, x).
//
// Reference call sites: model.py:133-158 (detection), :160-187 (embedd_camera), :246-283 (gathers),
// :479-593 (HPH), blocks/cross_attn_transformer.py:129-261, utils/humans.py:12-22, model.py:189-203,291.
#include "kernels.cuh"

namespace mhmr {

namespace {

constexpr float kPi = 3.14159274101257324219f;  // fp32(np.pi), blocks/camera_embed.py:53

__device__ __forceinline__ float sigmoid_clamped(float x) {
  const float s = 1.0f / (1.0f + expf(-x));
  return fminf(fmaxf(s, 1e-4f), 1.0f - 1e-4f);  // model.py:641-643
}

// ----------------------------------------------------------------------------------------------
// scores[r] = clamp(sigmoid(hidden[r,:] . w + b))   — second Linear of mlp_classif (model.py:135)
// ----------------------------------------------------------------------------------------------
__global__ void rowdot_sigmoid_kernel(const __half* __restrict__ hid, int64_t ld, const float* __restrict__ w,
                                      const float* __restrict__ b, float* __restrict__ scores,
                                      float* __restrict__ logits, int clamp, int M, int D) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const __half* hr = hid + static_cast<int64_t>(row) * ld;
  float acc = 0.f;
  for (int k = lane * 8; k < D; k += 256) {
    const uint4 pk = *reinterpret_cast<const uint4*>(hr + k);
    const __half2* h2 = reinterpret_cast<const __half2*>(&pk);
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + k));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(w + k + 4));
    const float2 a = __half22float2(h2[0]), c = __half22float2(h2[1]);
    const float2 d = __half22float2(h2[2]), e = __half22float2(h2[3]);
    acc += a.x * w0.x + a.y * w0.y + c.x * w0.z + c.y * w0.w + d.x * w1.x + d.y * w1.y + e.x * w1.z + e.y * w1.w;
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    const float l = acc + b[0];
    if (logits != nullptr) logits[row] = l;
    scores[row] = clamp ? sigmoid_clamped(l) : 1.0f / (1.0f + expf(-l));  // Anny: no clamp (encoder.py:59-60)
  }
}

// ----------------------------------------------------------------------------------------------
// NMS (max-pool k x k, stride 1, keep where equal) + threshold + ORDERED compaction (model.py:145-149,
// :612-638).  Single CTA: B*N is at most a few 10^5 cells; order = flattened (b, y, x) = torch.where order.
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024, 1)
nms_compact_kernel(const float* __restrict__ scores, float* __restrict__ scores_out, int B, int res,
                   int nms_k, float thresh, int max_persons, int* __restrict__ det_b,
                   int* __restrict__ det_y, int* __restrict__ det_x, float* __restrict__ det_score,
                   int* __restrict__ count, int* __restrict__ count_clamped, int* __restrict__ img_off) {
  __shared__ int warp_tot[32];
  __shared__ int base_s;
  const int N = res * res;
  const int total = B * N;
  const int tid = threadIdx.x;
  const int chunk = (total + blockDim.x - 1) / blockDim.x;
  const int beg = min(tid * chunk, total), end = min(beg + chunk, total);
  int pad = (nms_k - 1) / 2;
  if (nms_k == 2) pad = 1;
  if (nms_k == 4) pad = 2;

  auto nms_value = [&](int i) -> float {
    const float v = scores[i];
    if (nms_k <= 1) return v;
    const int b = i / N, n = i - b * N, y = n / res, x = n - y * res;
    float mx = -INFINITY;
    for (int dy = 0; dy < nms_k; ++dy) {
      const int yy = y - pad + dy;
      if (yy < 0 || yy >= res) continue;
      for (int dx = 0; dx < nms_k; ++dx) {
        const int xx = x - pad + dx;
        if (xx < 0 || xx >= res) continue;
        mx = fmaxf(mx, scores[b * N + yy * res + xx]);
      }
    }
    return (mx == v) ? v : 0.0f;  // heat * keep
  };

  int mine = 0;
  for (int i = beg; i < end; ++i) {
    const float v = nms_value(i);
    scores_out[i] = v;
    mine += (v >= thresh) ? 1 : 0;
  }
  // block exclusive scan of `mine`
  const int lane = tid & 31, wid = tid >> 5;
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int t = (lane < (blockDim.x >> 5)) ? warp_tot[lane] : 0;
    int inc2 = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, inc2, o);
      if (lane >= o) inc2 += u;
    }
    warp_tot[lane] = inc2 - t;  // exclusive warp offsets
    if (lane == 31) base_s = inc2;
  }
  __syncthreads();
  int pos = warp_tot[wid] + incl - mine;
  const int P = base_s;
  if (tid == 0) {
    *count = P;                               // true count: the host turns P > max_persons into an error
    *count_clamped = min(P, max_persons);     // what the per-person kernels may touch
  }
  for (int i = beg; i < end; ++i) {
    const float v = scores_out[i];
    if (v >= thresh) {
      if (pos < max_persons) {
        const int b = i / N, n = i - b * N;
        det_b[pos] = b;
        det_y[pos] = n / res;
        det_x[pos] = n - (n / res) * res;
        det_score[pos] = v;
      }
      ++pos;
    }
  }
  __syncthreads();
  // per-image offsets (persons are sorted by image): img_off[b] = first person of image b
  const int Pc = min(P, max_persons);
  for (int b = tid; b <= B; b += blockDim.x) {
    int lo = 0, hi = Pc;  // lower bound of b in det_b[0..Pc)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (det_b[mid] < b) lo = mid + 1; else hi = mid;
    }
    img_off[b] = lo;
  }
}

// Training-style forced detections (model.py:150-151): scores are NOT suppressed, idx comes from the caller.
__global__ void forced_idx_kernel(const float* __restrict__ scores, float* __restrict__ scores_out, int B,
                                  int res, const int64_t* __restrict__ idx4, int P, int* __restrict__ det_b,
                                  int* __restrict__ det_y, int* __restrict__ det_x,
                                  float* __restrict__ det_score, int* __restrict__ count,
                                  int* __restrict__ count_clamped, int* __restrict__ img_off) {
  const int N = res * res;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * N; i += gridDim.x * blockDim.x)
    scores_out[i] = scores[i];
  if (blockIdx.x == 0) {
    for (int p = threadIdx.x; p < P; p += blockDim.x) {
      const int b = static_cast<int>(idx4[p]), y = static_cast<int>(idx4[P + p]),
                x = static_cast<int>(idx4[2 * P + p]);
      det_b[p] = b; det_y[p] = y; det_x[p] = x;
      det_score[p] = scores[b * N + y * res + x];
    }
    if (threadIdx.x == 0) {
      *count = P;
      *count_clamped = P;  // forced_P <= max_persons is checked on the host
    }
    for (int b = threadIdx.x; b <= B; b += blockDim.x) {
      int c = 0;
      for (int p = 0; p < P; ++p) c += (static_cast<int>(idx4[p]) < b) ? 1 : 0;
      img_off[b] = c;
    }
  }
}

// ----------------------------------------------------------------------------------------------
// Camera: K^-1 per image (torch.inverse in utils/camera.py:43) and Fourier ray features
// (model.py:160-187, blocks/camera_embed.py:39-58).
// ----------------------------------------------------------------------------------------------
__global__ void invert_K_kernel(const float* __restrict__ K, float* __restrict__ Kinv, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* m = K + b * 9;
  const float a = m[0], bb = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
  const float A = e * i - f * h, Bc = -(d * i - f * g), C = d * h - e * g;
  const float det = a * A + bb * Bc + c * C;
  const float r = 1.0f / det;
  float* o = Kinv + b * 9;
  o[0] = A * r;  o[1] = -(bb * i - c * h) * r; o[2] = (bb * f - c * e) * r;
  o[3] = Bc * r; o[4] = (a * i - c * g) * r;   o[5] = -(a * f - c * d) * r;
  o[6] = C * r;  o[7] = -(a * h - bb * g) * r; o[8] = (a * e - bb * d) * r;
}

// Feature j of the 99-dim camera embedding at token (gy, gx): the (row, col) grid is passed as (x, y)
// to the un-projection, exactly as model.py:164-178 does.
__device__ __forceinline__ float camera_feature(const float* __restrict__ Kinv, const float* __restrict__ freqs,
                                                int gy, int gx, int j) {
  const float px = static_cast<float>(gy * 14 + 7), py = static_cast<float>(gx * 14 + 7);
  float ray[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) ray[r] = Kinv[r * 3 + 0] * px + Kinv[r * 3 + 1] * py + Kinv[r * 3 + 2];
  if (j < 3) return ray[j];
  const int t = (j - 3) % 48, d = t / 16, k = t % 16;
  const float arg = kPi * (ray[d] * freqs[k]);
  return (j < 51) ? sinf(arg) : cosf(arg);
}

// ctx16[b*N + n, D + j] = fp16(feature j), zero padding up to the row pitch.
__global__ void ctx_fourier_kernel(const float* __restrict__ Kinv, const float* __restrict__ freqs,
                                   __half* __restrict__ ctx, int64_t ld, int B, int res, int D, int pad_cols) {
  const int row = blockIdx.x;  // b*N + n
  const int N = res * res;
  const int b = row / N, n = row - b * N;
  const int j = threadIdx.x;
  if (j >= pad_cols) return;
  float v = 0.f;
  if (j < 99) v = camera_feature(Kinv + b * 9, freqs, n / res, n - (n / res) * res, j);
  ctx[static_cast<int64_t>(row) * ld + D + j] = __float2half_rn(v);
}

// Block-wide sum over 256 threads (all threads receive the result).
__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) t += red[w];
  return t;
}

// Per person: z_central, query = cat(z_central, z_K) + cross_queries_x[y] + cross_queries_y[x]
// (model.py:252-265, :500-504; note queries_x is indexed with y and queries_y with x, as in the reference),
// and the learned value embedding that the reference adds into the context at this cell (model.py:514-517).
// z_central is either the fp32 feature row of the bulk pass (z32) or, when `xr` is given, the final LayerNorm
// (eps 1e-6) of the person's REFINED residual stream (central-stream refinement, refine_* below).
__global__ void __launch_bounds__(256)
person_gather_kernel(const float* __restrict__ z32, const float* __restrict__ xr,
                     const float* __restrict__ norm_g, const float* __restrict__ norm_b,
                     const float* __restrict__ Kinv, const float* __restrict__ freqs,
                     const float* __restrict__ cq_x, const float* __restrict__ cq_y,
                     const float* __restrict__ cv_x, const float* __restrict__ cv_y,
                     const int* __restrict__ det_b, const int* __restrict__ det_y,
                     const int* __restrict__ det_x, const int* __restrict__ count, int res, int D,
                     float* __restrict__ zc, float* __restrict__ query, float* __restrict__ vals, int ldq) {
  __shared__ float red[8];
  const int p = blockIdx.x;
  if (p >= *count) return;
  const int b = det_b[p], y = det_y[p], x = det_x[p];
  const int N = res * res, C = D + 99;
  const float* zr = z32 + (static_cast<int64_t>(b) * N + y * res + x) * D;
  float mean = 0.f, rstd = 1.f;
  if (xr != nullptr) {
    const float* r = xr + static_cast<int64_t>(p) * D;
    float s = 0.f;
    for (int c = threadIdx.x; c < D; c += 256) s += r[c];
    mean = block_sum_256(s, red) / D;
    float q = 0.f;
    for (int c = threadIdx.x; c < D; c += 256) { const float d = r[c] - mean; q += d * d; }
    rstd = rsqrtf(block_sum_256(q, red) / D + 1e-6f);
  }
  for (int c = threadIdx.x; c < ldq; c += blockDim.x) {
    float v = 0.f, val = 0.f;
    if (c < C) {
      float base;
      if (c < D) {
        base = (xr != nullptr) ? (xr[static_cast<int64_t>(p) * D + c] - mean) * rstd * norm_g[c] + norm_b[c] : zr[c];
        zc[static_cast<int64_t>(p) * D + c] = base;
      } else {
        base = camera_feature(Kinv + b * 9, freqs, y, x, c - D);
      }
      v = base + cq_x[static_cast<int64_t>(y) * C + c] + cq_y[static_cast<int64_t>(x) * C + c];
      val = cv_x[static_cast<int64_t>(y) * C + c] + cv_y[static_cast<int64_t>(x) * C + c];
    }
    query[static_cast<int64_t>(p) * ldq + c] = v;
    vals[static_cast<int64_t>(p) * ldq + c] = val;
  }
}

// Central-stream refinement, step 0: per detected person, the token row index of its cell in the [B*T, .]
// token matrices (cls row skipped), its 14x14x3 input patch in the order of the patch-embed weight
// (c, ky, kx: dinov2 PatchEmbed Conv2d) and the fp32 (pos_embed + bias) row of its cell.
// With n_cls > 0 the first n_cls refined rows are the cls tokens of images 0..n_cls-1 (start value cls_token +
// pos_embed[0], a zero patch, so the patch embedding adds nothing) and person p is row n_cls + p;
// rows_out = n_cls + *count.
__global__ void __launch_bounds__(256)
refine_prepare_kernel(const float* __restrict__ img, const uint8_t* __restrict__ img_u8,
                      const float* __restrict__ lut, int S, const float* __restrict__ rowadd, int D,
                      const int* __restrict__ det_b, const int* __restrict__ det_y,
                      const int* __restrict__ det_x, const int* __restrict__ count, int res, int n_cls,
                      const float* __restrict__ cls_pos, int* __restrict__ rows_out,
                      int* __restrict__ rowidx, float* __restrict__ patch, int ldp, float* __restrict__ xr) {
  const int r = blockIdx.x;
  const int N = res * res;
  if (r == 0 && threadIdx.x == 0 && rows_out != nullptr) *rows_out = n_cls + *count;
  if (r < n_cls) {
    if (threadIdx.x == 0) rowidx[r] = r * (N + 1);
    for (int k = threadIdx.x; k < ldp; k += 256) patch[static_cast<int64_t>(r) * ldp + k] = 0.f;
    for (int c = threadIdx.x; c < D; c += 256) xr[static_cast<int64_t>(r) * D + c] = cls_pos[c];
    return;
  }
  const int p = r - n_cls;
  if (p >= *count) return;
  rowidx += n_cls; patch += static_cast<int64_t>(n_cls) * ldp; xr += static_cast<int64_t>(n_cls) * D;
  const int b = det_b[p], y = det_y[p], x = det_x[p];
  const int n = y * res + x;
  if (threadIdx.x == 0) rowidx[p] = b * (N + 1) + 1 + n;
  for (int k = threadIdx.x; k < ldp; k += 256) {
    float v = 0.f;
    if (k < 588) {
      const int c = k / 196, r = k - c * 196, ky = r / 14, kx = r - ky * 14;
      if (img_u8 != nullptr)  // fused uint8 loader: the fp32 pixel is the table entry (normalize_rgb, bit-exact)
        v = lut[c * 256 + img_u8[((static_cast<int64_t>(b) * S + y * 14 + ky) * S + x * 14 + kx) * 3 + c]];
      else
        v = img[((static_cast<int64_t>(b) * 3 + c) * S + y * 14 + ky) * S + x * 14 + kx];
    }
    patch[static_cast<int64_t>(p) * ldp + k] = v;
  }
  for (int c = threadIdx.x; c < D; c += 256) xr[static_cast<int64_t>(p) * D + c] = rowadd[static_cast<int64_t>(n) * D + c];
}

// KV[b*N + cell(p), :] += dKV[p, :]   (context += learned values at detected cells, model.py:517)
// The reference's `xx[idx] += values` is a non-accumulating index_put: a cell that several (forced) persons share
// receives the values once.  Their dKV rows are equal (the values depend on the cell only), so only the first person
// of a cell adds; the others leave, and no row is updated by two CTAs.
__global__ void kv_add_rows_kernel(float* __restrict__ KV, int64_t ldkv, const float* __restrict__ dKV,
                                   int ncols, const int* __restrict__ det_b, const int* __restrict__ det_y,
                                   const int* __restrict__ det_x, const int* __restrict__ count, int res) {
  const int p = blockIdx.x;
  if (p >= *count) return;
  const int b = det_b[p], y = det_y[p], x = det_x[p];
  int dup = 0;
  for (int q = threadIdx.x; q < p; q += blockDim.x) dup |= (det_b[q] == b && det_y[q] == y && det_x[q] == x);
  if (__syncthreads_or(dup)) return;
  const int N = res * res;
  float* row = KV + (static_cast<int64_t>(b) * N + y * res + x) * ldkv;
  for (int c = threadIdx.x; c < ncols; c += blockDim.x) row[c] += dKV[static_cast<int64_t>(p) * ncols + c];
}

// ----------------------------------------------------------------------------------------------
// Skinny linear: out[p, n] = resid[p, n] + act( LN?(x[p, :]) . W[n, :] + bias[n] ),  p < *count.
// fp32 weights streamed once per chunk of 8 persons (from L2 after the first chunk).  out may be resid (the
// residual updates of the HPH): each element is read and then written by the same thread.
//   grid = (ceil(Nout / (8 CPW)), ceil(max_persons / 8)), block = 256: 8 warps x CPW output columns each.
//   The 8 input rows are staged K-tile by K-tile (1024 floats per person, 32 KB static smem, 128-bit loads, LayerNorm
//   applied on the way in from per-row statistics computed once) so that several CTAs share an SM whatever K is;
//   every staged x value is used for CPW columns; the 8 CPW partial sums per lane are reduced with a butterfly
//   (31 shuffles for 32 values) that leaves lane (column, person) with its total.
// (r02: the first version staged whole rows with scalar loads in every CTA and used one column per warp: 25-37 us per
// launch for 4-16 MB of weights; 90 such launches per forward.)
// ----------------------------------------------------------------------------------------------
constexpr int kSkinnyPT = 8;
constexpr int kSkinnyKT = 1024;

template <int CPW>
__global__ void __launch_bounds__(256)
skinny_linear_kernel(const float* __restrict__ x, int ldx, const int* __restrict__ count, int K,
                     const float* __restrict__ W, int ldw, const float* __restrict__ bias, int Nout,
                     const float* __restrict__ ln_g, const float* __restrict__ ln_b, float ln_eps, int act,
                     const float* resid, int ldr, float* out, int ldo) {
  __shared__ __align__(16) float xs[kSkinnyPT][kSkinnyKT];
  __shared__ float stats[kSkinnyPT][2];
  constexpr int COLS = 8 * CPW;
  const int Kp = (K + 3) & ~3;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_base = blockIdx.x * COLS + warp * CPW;
  // Programmatic dependent launch: the weights do not depend on the preceding kernel, so this CTA's weight rows are
  // pulled into L2 while that kernel drains; everything it produced (count, activations) is read after the wait.
  griddep_launch_dependents();
  if (blockIdx.y == 0) {
#pragma unroll
    for (int c = 0; c < CPW; ++c) {
      const int n = n_base + c;
      if (n < Nout) {
        const char* wr = reinterpret_cast<const char*>(W + static_cast<int64_t>(n) * ldw);
        for (int b = lane * 128; b < Kp * 4; b += 32 * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(wr + b));
      }
    }
  }
  griddep_wait();
  const int P = *count;
  const int p0 = blockIdx.y * kSkinnyPT;
  if (p0 >= P) return;
  const int np = min(kSkinnyPT, P - p0);

  // LayerNorm statistics of the (fp32) input rows: one warp per person, two passes over the row
  if (ln_g != nullptr) {
    if (warp < np) {
      const float* src = x + static_cast<int64_t>(p0 + warp) * ldx;
      float sum = 0.f;
      for (int k = lane; k < K; k += 32) sum += src[k];
      const float mean = warp_sum(sum) / K;
      float q = 0.f;
      for (int k = lane; k < K; k += 32) { const float d = src[k] - mean; q += d * d; }
      const float rstd = rsqrtf(warp_sum(q) / K + ln_eps);
      if (lane == 0) { stats[warp][0] = mean; stats[warp][1] = rstd; }
    }
    __syncthreads();
  }

  float acc[CPW][kSkinnyPT];
#pragma unroll
  for (int c = 0; c < CPW; ++c)
#pragma unroll
    for (int j = 0; j < kSkinnyPT; ++j) acc[c][j] = 0.f;
  const bool vec_x = (ldx & 3) == 0;  // 128-bit loads need 16-byte aligned rows

  for (int k0 = 0; k0 < Kp; k0 += kSkinnyKT) {
    const int kt = min(kSkinnyKT, Kp - k0);  // multiple of 4
    const int q4 = kt >> 2;
    // ---- stage the K tile of the 8 rows (zeros for absent persons and for k >= K)
    for (int idx = threadIdx.x; idx < kSkinnyPT * q4; idx += 256) {
      const int j = idx / q4, q = idx - j * q4, k = k0 + 4 * q;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j < np) {
        const float* src = x + static_cast<int64_t>(p0 + j) * ldx + k;
        if (vec_x) {
          v = *reinterpret_cast<const float4*>(src);
        } else {
          v.x = src[0];
          if (k + 1 < K) v.y = src[1];
          if (k + 2 < K) v.z = src[2];
          if (k + 3 < K) v.w = src[3];
        }
        if (ln_g != nullptr) {
          const float mean = stats[j][0], rstd = stats[j][1];
          const float4 g = __ldg(reinterpret_cast<const float4*>(ln_g + k));
          const float4 bb = __ldg(reinterpret_cast<const float4*>(ln_b + k));
          v.x = (v.x - mean) * rstd * g.x + bb.x;
          v.y = (v.y - mean) * rstd * g.y + bb.y;
          v.z = (v.z - mean) * rstd * g.z + bb.z;
          v.w = (v.w - mean) * rstd * g.w + bb.w;
        }
        if (k + 3 >= K) {  // the padding of the last group must not contribute
          if (k + 1 >= K) v.y = 0.f;
          if (k + 2 >= K) v.z = 0.f;
          if (k + 3 >= K) v.w = 0.f;
        }
      }
      *reinterpret_cast<float4*>(&xs[j][4 * q]) = v;
    }
    __syncthreads();
    // ---- partial dot products of this warp's CPW columns with the 8 staged rows
    for (int k = lane * 4; k < kt; k += 128) {
      float4 w4[CPW];
#pragma unroll
      for (int c = 0; c < CPW; ++c) {
        const int n = min(n_base + c, Nout - 1);
        w4[c] = __ldg(reinterpret_cast<const float4*>(W + static_cast<int64_t>(n) * ldw + k0 + k));
      }
#pragma unroll
      for (int j = 0; j < kSkinnyPT; ++j) {
        const float4 x4 = *reinterpret_cast<const float4*>(&xs[j][k]);
#pragma unroll
        for (int c = 0; c < CPW; ++c)
          acc[c][j] += w4[c].x * x4.x + w4[c].y * x4.y + w4[c].z * x4.z + w4[c].w * x4.w;
      }
    }
    __syncthreads();
  }

  // ---- butterfly reduction: NV = 8 CPW values per lane -> lane L holds the total of value L (mod NV)
  constexpr int NV = CPW * kSkinnyPT;
  float a[NV];
#pragma unroll
  for (int c = 0; c < CPW; ++c)
#pragma unroll
    for (int j = 0; j < kSkinnyPT; ++j) a[c * kSkinnyPT + j] = acc[c][j];
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
  const int vi = lane & (NV - 1);
  const int c = vi / kSkinnyPT, j = vi - c * kSkinnyPT;
  const int n = n_base + c;
  if (lane < NV && j < np && n < Nout) {
    float v = a[0];
    if (bias != nullptr) v += bias[n];
    if (act == 1) v = fmaxf(v, 0.f);
    if (act == 2) v = gelu_erf(v);
    if (resid != nullptr) v += resid[static_cast<int64_t>(p0 + j) * ldr + n];
    out[static_cast<int64_t>(p0 + j) * ldo + n] = v;
  }
}

// ----------------------------------------------------------------------------------------------
// HPH self-attention among the persons of one image (Attention.forward,
// cross_attn_transformer.py:129-159): one warp per (person, head), dim_head = 32 = one lane per channel.
// Padded slots of the reference contribute exactly zero weight (-1e11 before softmax), so only the real
// persons of the image are visited.
// ----------------------------------------------------------------------------------------------
__global__ void hph_self_attn_kernel(const float* __restrict__ qkv, int ld, const int* __restrict__ det_b,
                                     const int* __restrict__ img_off, const int* __restrict__ count,
                                     int heads, float scale, float* __restrict__ out, int ldo) {
  const int p = blockIdx.x, h = blockIdx.y, lane = threadIdx.x;
  if (p >= *count) return;
  const int inner = heads * 32;
  const int b = det_b[p];
  const int beg = img_off[b], end = img_off[b + 1];
  const float q = qkv[static_cast<int64_t>(p) * ld + h * 32 + lane];
  float m = -INFINITY, l = 0.f, acc = 0.f;
  for (int o = beg; o < end; ++o) {
    const float k = qkv[static_cast<int64_t>(o) * ld + inner + h * 32 + lane];
    const float v = qkv[static_cast<int64_t>(o) * ld + 2 * inner + h * 32 + lane];
    const float s = warp_sum(q * k) * scale;
    const float mn = fmaxf(m, s);
    const float a = expf(m - mn), e = expf(s - mn);
    l = l * a + e;
    acc = acc * a + e * v;
    m = mn;
  }
  out[static_cast<int64_t>(p) * ldo + h * 32 + lane] = acc / l;
}

// ----------------------------------------------------------------------------------------------
// HPH cross-attention (CrossAttention.forward, cross_attn_transformer.py:185-205): one CTA per
// (person, head); keys/values are rows of the per-image KV matrix (fp32, produced by the to_kv GEMM).
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
hph_cross_attn_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ KV, int64_t ldkv,
                      int k_col, int v_col, const int* __restrict__ det_b, const int* __restrict__ count,
                      int N, float scale, float* __restrict__ out, int ldo) {
  const int p = blockIdx.x, h = blockIdx.y;
  if (p >= *count) return;
  __shared__ float red_m[8], red_l[8], red_acc[8][32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float qr[32];
#pragma unroll
  for (int d = 0; d < 32; ++d) qr[d] = q[static_cast<int64_t>(p) * ldq + h * 32 + d];
  const float* base = KV + static_cast<int64_t>(det_b[p]) * N * ldkv;
  float m = -INFINITY, l = 0.f, acc[32];
#pragma unroll
  for (int d = 0; d < 32; ++d) acc[d] = 0.f;
  for (int n = tid; n < N; n += 256) {
    const float4* kr = reinterpret_cast<const float4*>(base + static_cast<int64_t>(n) * ldkv + k_col + h * 32);
    const float4* vr = reinterpret_cast<const float4*>(base + static_cast<int64_t>(n) * ldkv + v_col + h * 32);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 k4 = kr[i];
      s += qr[4 * i] * k4.x + qr[4 * i + 1] * k4.y + qr[4 * i + 2] * k4.z + qr[4 * i + 3] * k4.w;
    }
    s *= scale;
    const float mn = fmaxf(m, s);
    const float a = expf(m - mn), e = expf(s - mn);
    l = l * a + e;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 v4 = vr[i];
      acc[4 * i] = acc[4 * i] * a + e * v4.x;
      acc[4 * i + 1] = acc[4 * i + 1] * a + e * v4.y;
      acc[4 * i + 2] = acc[4 * i + 2] * a + e * v4.z;
      acc[4 * i + 3] = acc[4 * i + 3] * a + e * v4.w;
    }
    m = mn;
  }
  // merge the 256 partial softmax states: warp shuffle, then across the 8 warps through smem
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
    const float l2 = __shfl_xor_sync(0xffffffffu, l, o);
    const float mn = fmaxf(m, m2);
    const float a = (m == -INFINITY) ? 0.f : expf(m - mn);
    const float b = (m2 == -INFINITY) ? 0.f : expf(m2 - mn);
    l = l * a + l2 * b;
#pragma unroll
    for (int d = 0; d < 32; ++d) {
      const float c2 = __shfl_xor_sync(0xffffffffu, acc[d], o);
      acc[d] = acc[d] * a + c2 * b;
    }
    m = mn;
  }
  if (lane == 0) {
    red_m[warp] = m;
    red_l[warp] = l;
#pragma unroll
    for (int d = 0; d < 32; ++d) red_acc[warp][d] = acc[d];
  }
  __syncthreads();
  if (warp == 0) {
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < 8; ++w) M = fmaxf(M, red_m[w]);
    float L = 0.f, A = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      const float a = (red_m[w] == -INFINITY) ? 0.f : expf(red_m[w] - M);
      L += red_l[w] * a;
      A += red_acc[w][lane] * a;
    }
    out[static_cast<int64_t>(p) * ldo + h * 32 + lane] = A / L;
  }
}

// ----------------------------------------------------------------------------------------------
// Rotation helpers (roma.special_gramschmidt, roma.rotmat_to_rotvec)
// ----------------------------------------------------------------------------------------------
// R = [e1 e2 e1 x e2] (columns) from the two 3-vectors a, b by Gram-Schmidt; R[r][c]
__device__ __forceinline__ void gram_schmidt(float a0, float a1, float a2, float b0, float b1, float b2,
                                             float (&R)[3][3]) {
  const float na = sqrtf(a0 * a0 + a1 * a1 + a2 * a2);
  a0 /= na; a1 /= na; a2 /= na;
  const float dp = a0 * b0 + a1 * b1 + a2 * b2;
  b0 -= dp * a0; b1 -= dp * a1; b2 -= dp * a2;
  const float nb = sqrtf(b0 * b0 + b1 * b1 + b2 * b2);
  b0 /= nb; b1 /= nb; b2 /= nb;
  const float c0 = a1 * b2 - a2 * b1, c1 = a2 * b0 - a0 * b2, c2 = a0 * b1 - a1 * b0;
  R[0][0] = a0; R[0][1] = b0; R[0][2] = c0;
  R[1][0] = a1; R[1][1] = b1; R[1][2] = c1;
  R[2][0] = a2; R[2][1] = b2; R[2][2] = c2;
}

// rotation matrix -> unit quaternion (xyzw, largest of diagonal / trace) -> rotation vector rv[3]
__device__ __forceinline__ void rotmat_to_rotvec(const float (&R)[3][3], float* rv) {
  const float tr = R[0][0] + R[1][1] + R[2][2];
  int choice = 0;
  float best = R[0][0];
  if (R[1][1] > best) { best = R[1][1]; choice = 1; }
  if (R[2][2] > best) { best = R[2][2]; choice = 2; }
  if (tr > best) { choice = 3; }
  float q[4];
  if (choice != 3) {
    const int i = choice, jj = (i + 1) % 3, k = (jj + 1) % 3;
    q[i] = 1.f - tr + 2.f * R[i][i];
    q[jj] = R[jj][i] + R[i][jj];
    q[k] = R[k][i] + R[i][k];
    q[3] = R[k][jj] - R[jj][k];
  } else {
    q[0] = R[2][1] - R[1][2];
    q[1] = R[0][2] - R[2][0];
    q[2] = R[1][0] - R[0][1];
    q[3] = 1.f + tr;
  }
  const float nq = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= nq; q[1] /= nq; q[2] /= nq; q[3] /= nq;
  if (q[3] < 0.f) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
  const float half = atan2f(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]), q[3]);
  const float ang = 2.f * half;
  float sc;
  if (fabsf(ang) <= 1e-3f) {
    const float a2_ = ang * ang;
    sc = 2.f + a2_ / 12.f + 7.f * a2_ * a2_ / 2880.f;
  } else {
    sc = ang / sinf(ang / 2.f);
  }
  rv[0] = sc * q[0]; rv[1] = sc * q[1]; rv[2] = sc * q[2];
}

// ----------------------------------------------------------------------------------------------
// Per-person post-processing: 6D -> rotation matrix (utils/humans.py:12-22, roma.special_gramschmidt),
// rotation matrix -> rotation vector (model.py:291, roma.rotmat_to_rotvec), distance (model.py:189-203),
// location (model.py:272-275), translation K^-1 [loc,1] dist (blocks/smpl_layer.py:123).
// dec[p, :] = [pose6 (318) | betas (nb) | cam (3) | expr (10)]  (decoder outputs + init, model.py:571-575)
// ----------------------------------------------------------------------------------------------
__global__ void person_post_kernel(const float* __restrict__ dec, int ld_dec, int num_betas,
                                   const float* __restrict__ offset, const float* __restrict__ K,
                                   const float* __restrict__ Kinv, const int* __restrict__ det_b,
                                   const int* __restrict__ det_y, const int* __restrict__ det_x,
                                   const int* __restrict__ count, float focal_norm,
                                   float* __restrict__ rotmat, float* __restrict__ rotvec,
                                   float* __restrict__ shape, float* __restrict__ expr,
                                   float* __restrict__ dist_pp, float* __restrict__ dist,
                                   float* __restrict__ loc, float* __restrict__ transl,
                                   float* __restrict__ K_det) {
  const int p = blockIdx.x;
  if (p >= *count) return;
  const float* d = dec + static_cast<int64_t>(p) * ld_dec;
  const int j = threadIdx.x;
  if (j < 53) {
    const float* x6 = d + j * 6;
    float R[3][3];
    gram_schmidt(x6[0], x6[1], x6[2], x6[3], x6[4], x6[5], R);
    float* Ro = rotmat + (static_cast<int64_t>(p) * 53 + j) * 9;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) Ro[r * 3 + c] = R[r][c];
    rotmat_to_rotvec(R, rotvec + (static_cast<int64_t>(p) * 53 + j) * 3);
  } else if (j == 53) {
    const int b = det_b[p];
    const float* Kb = K + b * 9;
    const float* Ki = Kinv + b * 9;
    for (int i = 0; i < 9; ++i) K_det[p * 9 + i] = Kb[i];
    const float cam0 = d[318 + num_betas];
    dist_pp[p] = cam0;
    float dd = cam0 * (Kb[0] / focal_norm);          // undo_focal_length_normalization
    dd = expf(dd) - 1e-10f;                          // undo_log_depth
    dd = fminf(fmaxf(dd, 0.f), 50.f);                // clamp (clip_dist tuple is always truthy)
    dist[p] = dd;
    const float lx = (static_cast<float>(det_x[p]) + 0.5f + offset[p * 2 + 0]) * 14.f;
    const float ly = (static_cast<float>(det_y[p]) + 0.5f + offset[p * 2 + 1]) * 14.f;
    loc[p * 2 + 0] = lx;
    loc[p * 2 + 1] = ly;
#pragma unroll
    for (int r = 0; r < 3; ++r) transl[p * 3 + r] = (Ki[r * 3] * lx + Ki[r * 3 + 1] * ly + Ki[r * 3 + 2]) * dd;
  } else if (j >= 64 && j < 64 + num_betas) {
    shape[p * num_betas + (j - 64)] = d[318 + (j - 64)];
  } else if (j >= 96 && j < 106) {
    expr[p * 10 + (j - 96)] = d[318 + num_betas + 3 + (j - 96)];
  }
}

// transl = K^-1 [loc, 1] * dist per person (blocks/smpl_layer.py:123), K inverted per person.
__global__ void loc_to_transl_kernel(const float* __restrict__ loc, const float* __restrict__ dist,
                                     const float* __restrict__ K_det, int P, float* __restrict__ transl) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const float* m = K_det + p * 9;
  const float a = m[0], bb = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
  const float A = e * i - f * h, Bc = -(d * i - f * g), C = d * h - e * g;
  const float r = 1.0f / (a * A + bb * Bc + c * C);
  const float inv[9] = {A * r, -(bb * i - c * h) * r, (bb * f - c * e) * r,
                        Bc * r, (a * i - c * g) * r, -(a * f - c * d) * r,
                        C * r, -(a * h - bb * g) * r, (a * e - bb * d) * r};
  const float lx = loc[p * 2], ly = loc[p * 2 + 1], dd = dist[p];
#pragma unroll
  for (int q = 0; q < 3; ++q) transl[p * 3 + q] = (inv[q * 3] * lx + inv[q * 3 + 1] * ly + inv[q * 3 + 2]) * dd;
}

}  // namespace

int loc_to_transl(const float* loc, const float* dist, const float* K_det, int P, float* transl,
                  cudaStream_t st) {
  loc_to_transl_kernel<<<(P + 63) / 64, 64, 0, st>>>(loc, dist, K_det, P, transl);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

// ------------------------------------------------------------------------------------------------
// Host launchers
// ------------------------------------------------------------------------------------------------
int rowdot_sigmoid(const __half* hid, int64_t ld, const float* w, const float* b, float* scores, float* logits,
                   bool clamp, int M, int D, cudaStream_t st) {
  MHMR_REQUIRE(D % 8 == 0 && ld % 8 == 0, "rowdot: D and pitch must be multiples of 8");
  rowdot_sigmoid_kernel<<<(M + 7) / 8, 256, 0, st>>>(hid, ld, w, b, scores, logits, clamp ? 1 : 0, M, D);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int nms_compact(const float* scores, float* scores_out, int B, int res, int nms_k, float thresh,
                int max_persons, int* det_b, int* det_y, int* det_x, float* det_score, int* count,
                int* count_clamped, int* img_off, cudaStream_t st) {
  MHMR_REQUIRE(nms_k >= 1 && nms_k <= 15, "nms kernel size out of range");
  nms_compact_kernel<<<1, 1024, 0, st>>>(scores, scores_out, B, res, nms_k, thresh, max_persons, det_b,
                                         det_y, det_x, det_score, count, count_clamped, img_off);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int forced_detections(const float* scores, float* scores_out, int B, int res, const int64_t* idx4, int P,
               int* det_b, int* det_y, int* det_x, float* det_score, int* count, int* count_clamped,
               int* img_off, cudaStream_t st) {
  forced_idx_kernel<<<64, 256, 0, st>>>(scores, scores_out, B, res, idx4, P, det_b, det_y, det_x, det_score,
                                        count, count_clamped, img_off);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int invert_K(const float* K, float* Kinv, int B, cudaStream_t st) {
  invert_K_kernel<<<(B + 63) / 64, 64, 0, st>>>(K, Kinv, B);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int ctx_fourier(const float* Kinv, const float* freqs, __half* ctx, int64_t ld, int B, int res, int D,
                int pad_cols, cudaStream_t st) {
  MHMR_REQUIRE(pad_cols >= 99 && pad_cols <= 128, "ctx_fourier: pad_cols must be in [99,128]");
  ctx_fourier_kernel<<<B * res * res, 128, 0, st>>>(Kinv, freqs, ctx, ld, B, res, D, pad_cols);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int person_gather(const float* z32, const float* xr, const float* norm_g, const float* norm_b, const float* Kinv,
                  const float* freqs, const float* cq_x, const float* cq_y, const float* cv_x, const float* cv_y,
                  const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons, int res,
                  int D, float* zc, float* query, float* vals, int ldq, cudaStream_t st) {
  person_gather_kernel<<<max_persons, 256, 0, st>>>(z32, xr, norm_g, norm_b, Kinv, freqs, cq_x, cq_y, cv_x, cv_y,
                                                    det_b, det_y, det_x, count, res, D, zc, query, vals, ldq);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int refine_prepare(const float* img, const uint8_t* img_u8, const float* lut, int S, const float* rowadd, int D,
                   const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons, int res,
                   int n_cls, const float* cls_pos, int* rows_out, int* rowidx, float* patch, int ldp, float* xr,
                   cudaStream_t st) {
  MHMR_REQUIRE(ldp >= 588 && ldp % 4 == 0, "refine_prepare: patch pitch must be >= 588 and a multiple of 4");
  MHMR_REQUIRE((img != nullptr) != (img_u8 != nullptr), "refine_prepare: exactly one image source");
  MHMR_REQUIRE(n_cls == 0 || cls_pos != nullptr, "refine_prepare: cls rows need cls_token + pos_embed[0]");
  refine_prepare_kernel<<<n_cls + max_persons, 256, 0, st>>>(img, img_u8, lut, S, rowadd, D, det_b, det_y, det_x, count,
                                                             res, n_cls, cls_pos, rows_out, rowidx, patch, ldp, xr);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int kv_add_rows(float* KV, int64_t ldkv, const float* dKV, int ncols, const int* det_b, const int* det_y,
                const int* det_x, const int* count, int max_persons, int res, cudaStream_t st) {
  kv_add_rows_kernel<<<max_persons, 256, 0, st>>>(KV, ldkv, dKV, ncols, det_b, det_y, det_x, count, res);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int skinny_linear_ex(const float* x, int ldx, int cols, const int* count, int max_persons, int K, const float* W, int ldw,
                     const float* bias, int Nout, const float* ln_g, const float* ln_b, float ln_eps, int act,
                     const float* resid, int ldr, float* out, int ldo, cudaStream_t st) {
  const int Kp = (K + 3) & ~3;
  MHMR_REQUIRE(ldw % 4 == 0 && ldw >= Kp, "skinny_linear: weight pitch must be >= K rounded to 4");
  MHMR_REQUIRE(x != nullptr && ldx >= K && (ldx % 4 != 0 || ldx >= Kp),
               "skinny_linear: input pitch must cover K (rounded to 4 when it is a multiple of 4)");
  MHMR_REQUIRE(ln_g == nullptr || K % 4 == 0, "skinny_linear: LayerNorm needs K % 4 == 0");
  MHMR_REQUIRE(cols == 0 || cols == 16 || cols == 32, "skinny_linear: cols must be 0 (pick), 16 or 32");
  // columns per warp: 4 (32 per CTA) by default, 2 when that leaves fewer CTAs than SMs for one 8-person chunk
  int cpw = (cols == 16) ? 2 : 4;
  if (cols == 0 && (Nout + 31) / 32 < device_sm_count()) cpw = 2;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((Nout + 8 * cpw - 1) / (8 * cpw), (max_persons + kSkinnyPT - 1) / kSkinnyPT);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  if (cpw == 4) {
    MHMR_CUDA_CHECK(cudaLaunchKernelEx(&cfg, skinny_linear_kernel<4>, x, ldx, count, K, W, ldw, bias, Nout, ln_g, ln_b,
                                       ln_eps, act, resid, ldr, out, ldo));
  } else {
    MHMR_CUDA_CHECK(cudaLaunchKernelEx(&cfg, skinny_linear_kernel<2>, x, ldx, count, K, W, ldw, bias, Nout, ln_g, ln_b,
                                       ln_eps, act, resid, ldr, out, ldo));
  }
  return MHMR_OK;
}

int skinny_linear(const float* x, int ldx, const int* count, int max_persons, int K, const float* W, int ldw,
                  const float* bias, int Nout, const float* ln_g, const float* ln_b, float ln_eps, int act,
                  const float* resid, int ldr, float* out, int ldo, cudaStream_t st) {
  return skinny_linear_ex(x, ldx, 0, count, max_persons, K, W, ldw, bias, Nout, ln_g, ln_b, ln_eps, act, resid, ldr, out,
                          ldo, st);
}

int hph_self_attn(const float* qkv, int ld, const int* det_b, const int* img_off, const int* count,
                  int max_persons, int heads, float* out, int ldo, cudaStream_t st) {
  hph_self_attn_kernel<<<dim3(max_persons, heads), 32, 0, st>>>(qkv, ld, det_b, img_off, count, heads,
                                                                0.17677669529663687f, out, ldo);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int hph_cross_attn(const float* q, int ldq, const float* KV, int64_t ldkv, int k_col, int v_col,
                   const int* det_b, const int* count, int max_persons, int heads, int N, float* out,
                   int ldo, cudaStream_t st) {
  MHMR_REQUIRE(ldkv % 4 == 0 && k_col % 4 == 0 && v_col % 4 == 0, "cross_attn: KV layout must be float4-aligned");
  hph_cross_attn_kernel<<<dim3(max_persons, heads), 256, 0, st>>>(q, ldq, KV, ldkv, k_col, v_col, det_b, count,
                                                                  N, 0.17677669529663687f, out, ldo);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int person_post(const float* dec, int ld_dec, int num_betas, const float* offset, const float* K,
                const float* Kinv, const int* det_b, const int* det_y, const int* det_x, const int* count,
                int max_persons, float focal_norm, float* rotmat, float* rotvec, float* shape, float* expr,
                float* dist_pp, float* dist, float* loc, float* transl, float* K_det, cudaStream_t st) {
  person_post_kernel<<<max_persons, 128, 0, st>>>(dec, ld_dec, num_betas, offset, K, Kinv, det_b, det_y, det_x,
                                                  count, focal_norm, rotmat, rotvec, shape, expr, dist_pp,
                                                  dist, loc, transl, K_det);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

// ------------------------------------------------------------------------------------------------
// Anny variant (multi_hmr_anny/): camera from the cls token, decoder inputs, per-person post-processing and the
// placement of the body model's output.  Same conventions as above: fp32, persons in (b, y, x) order, grids sized
// for the capacity and the device-side count.
// ------------------------------------------------------------------------------------------------
namespace {

__global__ void cls_gather_kernel(const void* __restrict__ X, const __half* __restrict__ Xlo, int64_t ld, int T, int D,
                                  float* __restrict__ out) {
  const int b = blockIdx.x;
  const int64_t row = static_cast<int64_t>(b) * T * ld;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float v;
    if (Xlo != nullptr)
      v = __half2float(static_cast<const __half*>(X)[row + c]) + __half2float(Xlo[row + c]);
    else
      v = static_cast<const float*>(X)[row + c];
    out[static_cast<int64_t>(b) * D + c] = v;
  }
}

// One warp per image: fov = fov_max * sigmoid(h . w2 + b2), f = (S/2) / tan(fov/2), K_regressed = [[f,0,S/2],
// [0,f,S/2],[0,0,1]] (encoder.py:50-56), K_use = K given, else K_regressed.
__global__ void anny_camera_kernel(const float* __restrict__ hid, int ldh, const float* __restrict__ w2,
                                   const float* __restrict__ b2, const float* __restrict__ fov_max,
                                   const float* __restrict__ K, int B, int D, float half_s, float* __restrict__ fov,
                                   float* __restrict__ K_reg, float* __restrict__ K_use) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  float acc = 0.f;
  for (int k = lane; k < D; k += 32) acc += hid[static_cast<int64_t>(b) * ldh + k] * w2[k];
  acc = warp_sum(acc);
  const float a = fov_max[0] * (1.0f / (1.0f + expf(-(acc + b2[0]))));
  const float f = half_s / tanf(a / 2.0f);
  const float kr[9] = {f, 0.f, half_s, 0.f, f, half_s, 0.f, 0.f, 1.f};
  if (lane < 9) {
    K_reg[b * 9 + lane] = kr[lane];
    K_use[b * 9 + lane] = (K != nullptr) ? K[b * 9 + lane] : kr[lane];
  }
  if (lane == 0) fov[b] = a;
}

__global__ void __launch_bounds__(256)
anny_gather_kernel(const float* __restrict__ z32, const float* __restrict__ xr, const float* __restrict__ norm_g,
                   const float* __restrict__ norm_b, const float* __restrict__ pos, const int* __restrict__ det_b,
                   const int* __restrict__ det_y, const int* __restrict__ det_x, const int* __restrict__ count,
                   int res, int D, int dim, float* __restrict__ zc, float* __restrict__ xa) {
  __shared__ float red[8];
  const int p = blockIdx.x;
  if (p >= *count) return;
  const int n = det_y[p] * res + det_x[p];
  const float* zr = z32 + (static_cast<int64_t>(det_b[p]) * res * res + n) * D;
  float mean = 0.f, rstd = 1.f;
  if (xr != nullptr) {
    const float* r = xr + static_cast<int64_t>(p) * D;
    float s = 0.f;
    for (int c = threadIdx.x; c < D; c += 256) s += r[c];
    mean = block_sum_256(s, red) / D;
    float q = 0.f;
    for (int c = threadIdx.x; c < D; c += 256) { const float d = r[c] - mean; q += d * d; }
    rstd = rsqrtf(block_sum_256(q, red) / D + 1e-6f);
  }
  for (int c = threadIdx.x; c < D; c += 256)
    zc[static_cast<int64_t>(p) * D + c] =
        (xr != nullptr) ? (xr[static_cast<int64_t>(p) * D + c] - mean) * rstd * norm_g[c] + norm_b[c] : zr[c];
  for (int c = threadIdx.x; c < dim; c += 256) xa[static_cast<int64_t>(p) * dim + c] = pos[static_cast<int64_t>(n) * dim + c];
}

// multi_hmr.py:143-175: thread j < J: 6D (rot6d.reshape(3, 2): columns (x0, x2, x4), (x1, x3, x5)) -> R by
// Gram-Schmidt, R <- u_j R + (1 - u_j) I, rotvec, [[R, 0], [0, 1]]; then the per-person scalars and shape.
__global__ void anny_person_post_kernel(const float* __restrict__ rot6d, int ld6, int J, const float* __restrict__ useful,
                                        float* __restrict__ shape, int num_betas, const float* __restrict__ offset,
                                        const float* __restrict__ dist_pp, const float* __restrict__ K_use,
                                        const float* __restrict__ Kinv, const int* __restrict__ det_b,
                                        const int* __restrict__ det_y, const int* __restrict__ det_x,
                                        const int* __restrict__ count, float* __restrict__ rotmat,
                                        float* __restrict__ rotmat_homo, float* __restrict__ rotvec,
                                        float* __restrict__ dist, float* __restrict__ loc, float* __restrict__ transl,
                                        float* __restrict__ K_det) {
  const int p = blockIdx.x;
  if (p >= *count) return;
  for (int j = threadIdx.x; j < J; j += blockDim.x) {
    const float* x6 = rot6d + static_cast<int64_t>(p) * ld6 + j * 6;
    float R[3][3];
    gram_schmidt(x6[0], x6[2], x6[4], x6[1], x6[3], x6[5], R);
    const float u = useful[j];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) R[r][c] = u * R[r][c] + (1.0f - u) * (r == c ? 1.0f : 0.0f);
    const int64_t pj = static_cast<int64_t>(p) * J + j;
    float* Ro = rotmat + pj * 9;
    float* Ho = rotmat_homo + pj * 16;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float v = (r < 3 && c < 3) ? R[r][c] : (r == 3 && c == 3 ? 1.0f : 0.0f);
        if (r < 3 && c < 3) Ro[r * 3 + c] = v;
        Ho[r * 4 + c] = v;
      }
    rotmat_to_rotvec(R, rotvec + pj * 3);
  }
  for (int i = threadIdx.x; i < num_betas; i += blockDim.x) {
    const float v = shape[p * num_betas + i];
    shape[p * num_betas + i] = 1.0f / (1.0f + expf(-v));
  }
  if (threadIdx.x == 0) {
    const int b = det_b[p];
    const float* Kb = K_use + b * 9;
    const float* Ki = Kinv + b * 9;
    for (int i = 0; i < 9; ++i) K_det[p * 9 + i] = Kb[i];
    const float dd = Kb[0] / fmaxf(expf(dist_pp[p]), 1e-5f);
    dist[p] = dd;
    const float lx = (static_cast<float>(det_x[p]) + 0.5f + offset[p * 2 + 0]) * 14.f;
    const float ly = (static_cast<float>(det_y[p]) + 0.5f + offset[p * 2 + 1]) * 14.f;
    loc[p * 2 + 0] = lx;
    loc[p * 2 + 1] = ly;
#pragma unroll
    for (int r = 0; r < 3; ++r) transl[p * 3 + r] = (Ki[r * 3] * lx + Ki[r * 3 + 1] * ly + Ki[r * 3 + 2]) * dd;
  }
}

// multi_hmr.py:180-186: x <- (x - bone(center)) + transl for every vertex and bone, then K_det (x / x_z)
__global__ void anny_place_kernel(const float* __restrict__ bone_poses, const float* __restrict__ transl,
                                  const float* __restrict__ K_det, int center, int V, int J, float* __restrict__ v3d,
                                  float* __restrict__ j3d, float* __restrict__ v2d, float* __restrict__ j2d,
                                  float* __restrict__ transl_pelvis) {
  const int p = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V + J) return;
  const float* bp = bone_poses + static_cast<int64_t>(p) * J * 16;
  const float c0 = bp[center * 16 + 3], c1 = bp[center * 16 + 7], c2 = bp[center * 16 + 11];
  const float t0 = transl[p * 3], t1 = transl[p * 3 + 1], t2 = transl[p * 3 + 2];
  float x, y, z;
  float *o3, *o2;
  if (i < V) {
    o3 = v3d + (static_cast<int64_t>(p) * V + i) * 3;
    o2 = (v2d != nullptr) ? v2d + (static_cast<int64_t>(p) * V + i) * 2 : nullptr;
    x = o3[0]; y = o3[1]; z = o3[2];
  } else {
    const int j = i - V;
    o3 = j3d + (static_cast<int64_t>(p) * J + j) * 3;
    o2 = j2d + (static_cast<int64_t>(p) * J + j) * 2;
    x = bp[j * 16 + 3]; y = bp[j * 16 + 7]; z = bp[j * 16 + 11];
  }
  x = (x - c0) + t0; y = (y - c1) + t1; z = (z - c2) + t2;
  o3[0] = x; o3[1] = y; o3[2] = z;
  if (i == V) { transl_pelvis[p * 3] = x; transl_pelvis[p * 3 + 1] = y; transl_pelvis[p * 3 + 2] = z; }
  if (o2 != nullptr) {
    const float* K = K_det + p * 9;
    const float u = x / z, v = y / z, w = z / z;
    o2[0] = K[0] * u + K[1] * v + K[2] * w;
    o2[1] = K[3] * u + K[4] * v + K[5] * w;
  }
}

}  // namespace

int cls_gather(const void* X, const __half* Xlo, int64_t ld, int T, int B, int D, float* out, cudaStream_t st) {
  cls_gather_kernel<<<B, 256, 0, st>>>(X, Xlo, ld, T, D, out);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int anny_camera(const float* hid, int ldh, const float* w2, const float* b2, const float* fov_max, const float* K,
                int B, int S, float* fov, float* K_reg, float* K_use, float* Kinv, cudaStream_t st) {
  anny_camera_kernel<<<(B + 7) / 8, 256, 0, st>>>(hid, ldh, w2, b2, fov_max, K, B, ldh, static_cast<float>(S) / 2.0f,
                                                  fov, K_reg, K_use);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return invert_K(K_use, Kinv, B, st);
}

int anny_gather(const float* z32, const float* xr, const float* norm_g, const float* norm_b, const float* pos,
                const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons, int res,
                int D, int dim, float* zc, float* xa, cudaStream_t st) {
  anny_gather_kernel<<<max_persons, 256, 0, st>>>(z32, xr, norm_g, norm_b, pos, det_b, det_y, det_x, count, res, D,
                                                  dim, zc, xa);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int anny_person_post(const float* rot6d, int ld6, int J, const float* useful, float* shape, int num_betas,
                     const float* offset, const float* dist_pp, const float* K_use, const float* Kinv,
                     const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons,
                     float* rotmat, float* rotmat_homo, float* rotvec, float* dist, float* loc, float* transl,
                     float* K_det, cudaStream_t st) {
  anny_person_post_kernel<<<max_persons, 192, 0, st>>>(rot6d, ld6, J, useful, shape, num_betas, offset, dist_pp, K_use,
                                                       Kinv, det_b, det_y, det_x, count, rotmat, rotmat_homo, rotvec,
                                                       dist, loc, transl, K_det);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int anny_place(const float* bone_poses, const float* transl, const float* K_det, int center, int P, int V, int J,
               float* v3d, float* j3d, float* v2d, float* j2d, float* transl_pelvis, cudaStream_t st) {
  MHMR_REQUIRE(P >= 0 && P <= 65535 && V >= 0 && J >= 1 && center >= 0 && center < J, "anny_place: bad sizes");
  if (P == 0) return MHMR_OK;
  anny_place_kernel<<<dim3((V + J + 255) / 256, P), 256, 0, st>>>(bone_poses, transl, K_det, center, V, J, v3d, j3d,
                                                                  v2d, j2d, transl_pelvis);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

}  // namespace mhmr
