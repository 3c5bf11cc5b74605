// Stage-level C-ABI entry points (unit parity + ncu targets). See include/mhmr.h.
#include "../../include/mhmr.h"
#include "gemm_tc.cuh"
#include "kernels.cuh"

using namespace mhmr;

namespace {
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
}  // namespace

extern "C" {

const char* mhmr_last_error(void) { return get_last_error(); }

int mhmr_op_gemm_f16(const void* A, int64_t lda, const void* W, int64_t ldw, int M, int N, int K,
                     int epilogue, const float* bias, const float* gamma, const float* rowadd,
                     void* out, int64_t ldo, int rows_in, int rows_out, int row_off, int block_n,
                     void* stream) {
  GemmEpi ep;
  ep.bias = bias;
  ep.gamma = gamma;
  ep.rowadd = rowadd;
  ep.out = out;
  ep.ldo = ldo;
  ep.rows_in = rows_in;
  ep.rows_out = rows_out;
  ep.row_off = row_off;
  MHMR_REQUIRE(epilogue >= 0 && epilogue < EPI_NUM_PUBLIC_KINDS, "gemm: bad epilogue kind");
  GemmPlan plan;
  int rc = gemm_plan_init(&plan, static_cast<const __half*>(A), lda, static_cast<const __half*>(W),
                          ldw, M, N, K, epilogue, ep, block_n);
  if (rc != MHMR_OK) return rc;
  return gemm_plan_run(&plan, static_cast<cudaStream_t>(stream));
}

int mhmr_op_resid_ln_linear_f16(const void* A, int64_t lda, const void* Wp, int64_t ldwp, const float* bp,
                                const float* ls, float* X, int M, int D, int Ka, const float* ln_g,
                                const float* ln_b, const float* W, const float* b, int N, int gelu, void* out16,
                                int64_t ldo, void* stream) {
  MHMR_REQUIRE(A && Wp && bp && ls && X && ln_g && ln_b && W && b && out16, "null argument");
  MHMR_REQUIRE(D % 128 == 0 && D <= 1024 && N % 32 == 0, "resid_ln_linear: D must be a multiple of 128 (<= 1024)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int bn_d = (D % 256 == 0) ? 512 : 128, bn_n = (N % 256 == 0) ? 512 : 128;
  const int slots = gemm_stat_slots(D, bn_d);
  CallScratch ws(st);
  const size_t r_x16 = ws.region(static_cast<size_t>(M) * D * 2), r_xlo = ws.region(static_cast<size_t>(M) * D * 2),
               r_W16 = ws.region(static_cast<size_t>(N) * D * 2),
               r_stats = ws.region(static_cast<size_t>(M) * slots * sizeof(float2)),
               r_bias2 = ws.region(static_cast<size_t>(N) * 4);
  TRY(ws.allocate());
  __half *x16 = ws.dev<__half>(r_x16), *xlo = ws.dev<__half>(r_xlo), *W16 = ws.dev<__half>(r_W16);
  float2* stats = ws.dev<float2>(r_stats);
  float* bias2 = ws.dev<float>(r_bias2);
  TRY(fold_ln_linear(W, b, ln_g, ln_b, W16, bias2, N, D, st));
  TRY(split_rowstats(X, x16, xlo, D, stats, slots, M, D, st));  // the stream enters as (hi, lo)
  GemmEpi p;
  p.bias = bp; p.gamma = ls;
  p.x16 = x16; p.xlo = xlo; p.ldx16 = D; p.stats = stats; p.stat_slots = slots;
  GemmPlan pp;
  TRY(gemm_plan_init(&pp, static_cast<const __half*>(A), lda, static_cast<const __half*>(Wp), ldwp, M, D, Ka,
                     EPI_LS_RESID_SPLIT, p, bn_d));
  TRY(gemm_plan_run(&pp, st));
  GemmEpi c;
  c.bias = bias2; c.stats = stats; c.stat_slots = slots; c.out = out16; c.ldo = ldo;
  GemmPlan cp;
  TRY(gemm_plan_init(&cp, x16, D, W16, D, M, N, D, gelu ? EPI_LN_GELU_F16 : EPI_LN_BIAS_F16, c, bn_n));
  TRY(gemm_plan_run(&cp, st));
  TRY(merge_split(x16, xlo, X, static_cast<int64_t>(M) * D, st));
  return ws.release();
}

int mhmr_op_attention(const void* qkv, int64_t ld_qkv, void* out, int64_t ldo, int B, int T, int D,
                      void* stream) {
  return attention_forward(static_cast<const __half*>(qkv), ld_qkv, static_cast<__half*>(out), ldo, B, T,
                           D, static_cast<cudaStream_t>(stream));
}

int mhmr_op_normalize_u8(const void* img_u8, const float* lut, float* out, int B, int H, int W, void* stream) {
  MHMR_REQUIRE(img_u8 != nullptr && lut != nullptr && out != nullptr, "null argument");
  return normalize_u8(static_cast<const uint8_t*>(img_u8), lut, out, B, H, W, static_cast<cudaStream_t>(stream));
}

// ---- person-decoder kernels (head.cu, refine.cu): the launchers the engine calls, unchanged ----------------------

int mhmr_op_skinny_linear(const float* x, int ldx, const int* count, int max_persons, int K, const float* W, int ldw,
                          const float* bias, int Nout, const float* ln_g, const float* ln_b, float ln_eps, int act,
                          const float* resid, int ldr, float* out, int ldo, int cols, void* stream) {
  MHMR_REQUIRE(x && count && W && out, "null argument");
  MHMR_REQUIRE(max_persons >= 0 && K >= 1 && Nout >= 1 && act >= 0 && act <= 2, "skinny_linear: bad sizes or act");
  MHMR_REQUIRE(ldo >= Nout && (resid == nullptr || ldr >= Nout), "skinny_linear: output pitches must cover Nout");
  MHMR_REQUIRE((ln_g == nullptr) == (ln_b == nullptr), "skinny_linear: LayerNorm needs both ln_g and ln_b");
  MHMR_REQUIRE(aligned16(W) && (ldx % 4 != 0 || aligned16(x)) && (ln_g == nullptr || (aligned16(ln_g) && aligned16(ln_b))),
               "skinny_linear: W, LayerNorm vectors and x (when ldx % 4 == 0) must be 16-byte aligned");
  if (max_persons == 0) return MHMR_OK;
  return skinny_linear_ex(x, ldx, cols, count, max_persons, K, W, ldw, bias, Nout, ln_g, ln_b, ln_eps, act, resid, ldr,
                          out, ldo, static_cast<cudaStream_t>(stream));
}

int mhmr_op_hph_self_attn(const float* qkv, int ld, const int* det_b, const int* img_off, const int* count,
                          int max_persons, int heads, float* out, int ldo, void* stream) {
  MHMR_REQUIRE(qkv && det_b && img_off && count && out, "null argument");
  MHMR_REQUIRE(max_persons >= 0 && heads >= 1 && ld >= 3 * 32 * heads && ldo >= 32 * heads,
               "hph_self_attn: pitches must cover 3 * heads * 32 (qkv) and heads * 32 (out)");
  if (max_persons == 0) return MHMR_OK;
  return hph_self_attn(qkv, ld, det_b, img_off, count, max_persons, heads, out, ldo, static_cast<cudaStream_t>(stream));
}

int mhmr_op_hph_cross_attn(const float* q, int ldq, const float* KV, int64_t ldkv, int k_col, int v_col,
                           const int* det_b, const int* count, int max_persons, int heads, int N, float* out, int ldo,
                           void* stream) {
  MHMR_REQUIRE(q && KV && det_b && count && out, "null argument");
  MHMR_REQUIRE(max_persons >= 0 && heads >= 1 && N >= 1 && ldq >= 32 * heads && ldo >= 32 * heads && k_col >= 0 &&
                   v_col >= 0 && k_col + 32 * heads <= ldkv && v_col + 32 * heads <= ldkv,
               "hph_cross_attn: bad sizes or column offsets");
  MHMR_REQUIRE(aligned16(KV), "hph_cross_attn: KV must be 16-byte aligned");
  if (max_persons == 0) return MHMR_OK;
  return hph_cross_attn(q, ldq, KV, ldkv, k_col, v_col, det_b, count, max_persons, heads, N, out, ldo,
                        static_cast<cudaStream_t>(stream));
}

int mhmr_op_detect(const float* scores, int B, int res, int nms_k, float thresh, int max_persons, float* scores_out,
                   int* det_b, int* det_y, int* det_x, float* det_score, int* count, int* count_clamped, int* img_off,
                   void* stream) {
  MHMR_REQUIRE(scores && scores_out && det_b && det_y && det_x && det_score && count && count_clamped && img_off,
               "null argument");
  MHMR_REQUIRE(scores != scores_out, "detect: scores_out must not alias scores (neighbours are read while writing)");
  MHMR_REQUIRE(B >= 1 && res >= 1 && max_persons >= 0, "detect: bad sizes");
  return nms_compact(scores, scores_out, B, res, nms_k, thresh, max_persons, det_b, det_y, det_x, det_score, count,
                     count_clamped, img_off, static_cast<cudaStream_t>(stream));
}

int mhmr_op_person_post(const float* dec, int ld_dec, int num_betas, const float* offset, const float* K, int B,
                        const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons,
                        float focal_norm, float* rotmat, float* rotvec, float* shape, float* expr, float* dist_pp,
                        float* dist, float* loc, float* transl, float* K_det, void* stream) {
  MHMR_REQUIRE(dec && offset && K && det_b && det_y && det_x && count && rotmat && rotvec && shape && expr && dist_pp &&
                   dist && loc && transl && K_det, "null argument");
  MHMR_REQUIRE(B >= 1 && max_persons >= 0 && num_betas >= 1 && num_betas <= 32 && ld_dec >= 318 + num_betas + 13,
               "person_post: bad sizes (num_betas in [1, 32], decoder row = 318 + num_betas + 3 + 10)");
  if (max_persons == 0) return MHMR_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallScratch ws(st);
  const size_t r_Kinv = ws.region(static_cast<size_t>(B) * 9 * sizeof(float));
  TRY(ws.allocate());
  float* Kinv = ws.dev<float>(r_Kinv);
  TRY(invert_K(K, Kinv, B, st));
  TRY(person_post(dec, ld_dec, num_betas, offset, K, Kinv, det_b, det_y, det_x, count, max_persons, focal_norm, rotmat,
                  rotvec, shape, expr, dist_pp, dist, loc, transl, K_det, st));
  return ws.release();
}

int mhmr_op_anny_person_post(const float* hid, int D, const float* w2, const float* b2, const float* fov_max,
                             const float* K, int B, int img_size, float* fov, float* K_regressed, float* K_use,
                             const float* rot6d, int ld6, int J, const float* useful, float* shape, int num_betas,
                             const float* offset, const float* dist_pp, const int* det_b, const int* det_y,
                             const int* det_x, const int* count, int max_persons, float* rotmat, float* rotmat_homo,
                             float* rotvec, float* dist, float* loc, float* transl, float* K_det, void* stream) {
  MHMR_REQUIRE(hid && w2 && b2 && fov_max && fov && K_regressed && K_use && rot6d && useful && shape && offset &&
                   dist_pp && det_b && det_y && det_x && count && rotmat && rotmat_homo && rotvec && dist && loc &&
                   transl && K_det, "null argument");
  MHMR_REQUIRE(B >= 1 && D >= 1 && img_size >= 1 && J >= 1 && ld6 >= 6 * J && num_betas >= 0 && max_persons >= 0,
               "anny_person_post: bad sizes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallScratch ws(st);
  const size_t r_Kinv = ws.region(static_cast<size_t>(B) * 9 * sizeof(float));
  TRY(ws.allocate());
  float* Kinv = ws.dev<float>(r_Kinv);
  TRY(anny_camera(hid, D, w2, b2, fov_max, K, B, img_size, fov, K_regressed, K_use, Kinv, st));
  if (max_persons > 0)
    TRY(anny_person_post(rot6d, ld6, J, useful, shape, num_betas, offset, dist_pp, K_use, Kinv, det_b, det_y, det_x,
                         count, max_persons, rotmat, rotmat_homo, rotvec, dist, loc, transl, K_det, st));
  return ws.release();
}

int mhmr_op_refine_chain(int depth, int D, const int* count, int max_persons, const float* Wproj, const float* bproj,
                         const float* ls1, const float* ln2_g, const float* ln2_b, const float* Wfc1, const float* bfc1,
                         const float* Wfc2, const float* bfc2, const float* ls2, const void* O16, int64_t rows_o16,
                         const int* rowidx, float* x, void* stream) {
  MHMR_REQUIRE(count && Wproj && bproj && ls1 && ln2_g && ln2_b && Wfc1 && bfc1 && Wfc2 && bfc2 && ls2 && O16 && rowidx &&
                   x, "null argument");
  MHMR_REQUIRE(depth >= 1 && D >= 4 && D % 4 == 0 && max_persons >= 0 && rows_o16 >= 1, "refine_chain: bad sizes");
  // the chain stages 8 hidden rows of 4D floats plus a 8 x 256 reduction buffer in (at most 200 KB of) shared memory
  MHMR_REQUIRE((8 * 4 * D + 8 * 256) * 4 <= 200 * 1024, "refine_chain: D must be at most 1536");
  MHMR_REQUIRE(aligned16(x) && aligned16(O16) && aligned16(Wproj) && aligned16(Wfc1) && aligned16(Wfc2) &&
                   aligned16(ln2_g) && aligned16(ln2_b), "refine_chain: x, O16, weights and ln2 must be 16-byte aligned");
  if (max_persons == 0) return MHMR_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t DD = static_cast<int64_t>(D) * D;
  CallScratch ws(st);
  const size_t r_layers = ws.region(depth * sizeof(RefineLayer), true),
               r_term = ws.region(static_cast<size_t>(depth) * max_persons * D * sizeof(float)),
               r_h = ws.region(static_cast<size_t>(max_persons) * 4 * D * sizeof(float)),
               r_barrier = ws.region(sizeof(unsigned int));
  RefineLayer* rl = ws.host<RefineLayer>(r_layers);
  for (int l = 0; l < depth; ++l)
    rl[l] = RefineLayer{static_cast<const __half*>(O16) + l * rows_o16 * D, Wproj + l * DD, bproj + l * D, ls1 + l * D,
                        ln2_g + l * D, ln2_b + l * D, Wfc1 + l * 4 * DD, bfc1 + l * 4 * D, Wfc2 + l * 4 * DD,
                        bfc2 + l * D, ls2 + l * D};
  TRY(ws.allocate());
  TRY(ws.upload());
  const RefineLayer* layers = ws.dev<const RefineLayer>(r_layers);
  float *term = ws.dev<float>(r_term), *h = ws.dev<float>(r_h);
  TRY(refine_proj_terms(layers, depth, rowidx, count, D, max_persons, term, st));
  TRY(refine_mlp_chain(layers, depth, count, D, max_persons, term, x, h, ws.dev<unsigned int>(r_barrier), st));
  return ws.release();
}

// ---- backbone entry, folded LayerNorm and the gathers of the heads (vit_misc.cu, gemm_tc.cu, head.cu) --------------

int mhmr_op_im2col_patch14(const float* img, const void* img_u8, const float* lut, int B, int S, void* A, int ldA,
                           void* stream) {
  MHMR_REQUIRE(A != nullptr && (img != nullptr) != (img_u8 != nullptr) && (img_u8 == nullptr) == (lut == nullptr),
               "im2col: exactly one image source (fp32 CHW, or uint8 HWC with its table)");
  MHMR_REQUIRE(B >= 1 && S >= 14 && S % 14 == 0 && ldA >= 588, "im2col: bad geometry");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (img_u8 != nullptr)
    return im2col_u8_patch14(static_cast<const uint8_t*>(img_u8), lut, static_cast<__half*>(A), B, S, ldA, st);
  return im2col_patch14(img, static_cast<__half*>(A), B, S, ldA, st);
}

int mhmr_op_layernorm(const void* X, const void* Xlo, const float* gamma, const float* beta, void* out16, int64_t ld16,
                      float* out32, int64_t ld32, int M, int D, float eps, int rows_in, int skip, void* stream) {
  MHMR_REQUIRE(X && gamma && beta && (out16 || out32), "null argument");
  MHMR_REQUIRE(M >= 0 && D >= 128 && D % 128 == 0 && D <= 1024, "layernorm: D must be a multiple of 128 (<= 1024)");
  MHMR_REQUIRE(rows_in == 0 ? skip == 0 : (rows_in > 0 && skip >= 0 && skip < rows_in && M % rows_in == 0),
               "layernorm: rows_in must divide M and exceed skip");
  MHMR_REQUIRE((out16 == nullptr || (ld16 >= D && ld16 % 4 == 0)) && (out32 == nullptr || (ld32 >= D && ld32 % 4 == 0)),
               "layernorm: output pitches must cover D and be multiples of 4");
  MHMR_REQUIRE(aligned16(X) && aligned16(gamma) && aligned16(beta) && (Xlo == nullptr || aligned16(Xlo)) &&
                   (out16 == nullptr || aligned16(out16)) && (out32 == nullptr || aligned16(out32)),
               "layernorm: every buffer must be 16-byte aligned");
  if (M == 0) return MHMR_OK;
  return layernorm_split(X, static_cast<const __half*>(Xlo), gamma, beta, static_cast<__half*>(out16), ld16, out32,
                         ld32, M, D, eps, rows_in, skip, static_cast<cudaStream_t>(stream));
}

int mhmr_op_split_rowstats(const float* X, void* xhi, void* xlo, int64_t ld16, float* stats, int slots, int M, int D,
                           void* stream) {
  MHMR_REQUIRE(X && xhi && xlo && stats, "null argument");
  MHMR_REQUIRE(M >= 0 && D >= 128 && D % 128 == 0 && D <= 1024 && slots >= 1 && slots <= 32 && ld16 >= D &&
                   ld16 % 4 == 0, "split_rowstats: bad sizes");
  MHMR_REQUIRE(aligned16(X) && aligned16(xhi) && aligned16(xlo) && (reinterpret_cast<uintptr_t>(stats) & 7u) == 0,
               "split_rowstats: X and the planes must be 16-byte aligned, stats 8-byte aligned");
  if (M == 0) return MHMR_OK;
  return split_rowstats(X, static_cast<__half*>(xhi), static_cast<__half*>(xlo), ld16, reinterpret_cast<float2*>(stats),
                        slots, M, D, static_cast<cudaStream_t>(stream));
}

int mhmr_op_fold_ln_linear(const float* W, const float* bias, const float* ln_g, const float* ln_b, void* W16,
                           float* bias2, int N, int K, void* stream) {
  MHMR_REQUIRE(W && bias && ln_g && ln_b && W16 && bias2, "null argument");
  MHMR_REQUIRE(N >= 1 && K >= 1, "fold_ln_linear: bad sizes");
  return fold_ln_linear(W, bias, ln_g, ln_b, static_cast<__half*>(W16), bias2, N, K, static_cast<cudaStream_t>(stream));
}

int mhmr_op_gemm_internal(const void* A, int64_t lda, const void* W, int64_t ldw, int M, int N, int K, int epilogue,
                          const float* bias, const float* gamma, void* x16, void* xlo, int64_t ldx16, float* stats,
                          int stat_slots, const float* rowadd, int rows_in, int rows_out, int row_off, void* out,
                          int64_t ldo, int block_n, int M_run, void* stream) {
  MHMR_REQUIRE(epilogue >= 0 && epilogue < EPI_NUM_KINDS, "gemm_internal: epilogue must be a kind in 0..9");
  MHMR_REQUIRE(epilogue != EPI_LS_RESID_SPLIT || (ldx16 >= N && aligned16(x16) && aligned16(xlo)),
               "gemm_internal: the split planes must cover N columns and be 16-byte aligned");
  MHMR_REQUIRE(epilogue == EPI_LS_RESID_SPLIT || (ldo >= N && aligned16(out)),
               "gemm_internal: the output must cover N columns and be 16-byte aligned");
  MHMR_REQUIRE(stats == nullptr || aligned16(stats), "gemm_internal: stats must be 16-byte aligned");
  MHMR_REQUIRE(rowadd == nullptr || aligned16(rowadd), "gemm_internal: rowadd must be 16-byte aligned");
  MHMR_REQUIRE(M_run >= 0 && M_run <= M, "gemm_internal: M_run must be in [0, M] (0 runs all M rows)");
  GemmEpi ep;
  ep.bias = bias;
  ep.gamma = gamma;
  ep.rowadd = rowadd;
  ep.rows_in = rows_in;
  ep.rows_out = rows_out;
  ep.row_off = row_off;
  ep.out = out;
  ep.ldo = ldo;
  ep.x16 = static_cast<__half*>(x16);
  ep.xlo = static_cast<__half*>(xlo);
  ep.ldx16 = ldx16;
  ep.stats = reinterpret_cast<float2*>(stats);
  ep.stat_slots = stat_slots;
  GemmPlan plan;
  int rc = gemm_plan_init(&plan, static_cast<const __half*>(A), lda, static_cast<const __half*>(W), ldw, M, N, K,
                          epilogue, ep, block_n);
  if (rc != MHMR_OK) return rc;
  return gemm_plan_run_rows(&plan, M_run > 0 ? M_run : M, static_cast<cudaStream_t>(stream));
}

int mhmr_op_camera_ctx(const float* K, int B, const float* freqs, float* Kinv, void* ctx, int64_t ld, int res, int col0,
                       int pad_cols, void* stream) {
  MHMR_REQUIRE(K && freqs && Kinv && ctx, "null argument");
  MHMR_REQUIRE(B >= 1 && res >= 1 && col0 >= 0 && pad_cols >= 99 && pad_cols <= 128 && ld >= col0 + pad_cols,
               "camera_ctx: bad sizes (pad_cols in [99, 128], ld >= col0 + pad_cols)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rc = invert_K(K, Kinv, B, st);
  if (rc != MHMR_OK) return rc;
  return ctx_fourier(Kinv, freqs, static_cast<__half*>(ctx), ld, B, res, col0, pad_cols, st);
}

int mhmr_op_rowdot_sigmoid(const void* hid, int64_t ld, const float* w, const float* b, float* scores, float* logits,
                           int clamp, int M, int D, void* stream) {
  MHMR_REQUIRE(hid && w && b && scores, "null argument");
  MHMR_REQUIRE(M >= 0 && D >= 8 && D % 8 == 0 && ld >= D && ld % 8 == 0, "rowdot_sigmoid: bad sizes");
  MHMR_REQUIRE(aligned16(hid) && aligned16(w), "rowdot_sigmoid: hid and w must be 16-byte aligned");
  if (M == 0) return MHMR_OK;
  return rowdot_sigmoid(static_cast<const __half*>(hid), ld, w, b, scores, logits, clamp != 0, M, D,
                        static_cast<cudaStream_t>(stream));
}

int mhmr_op_person_gather(const float* z32, const float* xr, const float* norm_g, const float* norm_b, const float* Kinv,
                          const float* freqs, const float* cq_x, const float* cq_y, const float* cv_x, const float* cv_y,
                          const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons,
                          int res, int D, float* zc, float* query, float* vals, int ldq, void* stream) {
  MHMR_REQUIRE(max_persons >= 0 && res >= 1 && D >= 1 && ldq >= D + 99, "person_gather: bad sizes (ldq >= D + 99)");
  if (max_persons == 0) return MHMR_OK;
  MHMR_REQUIRE(z32 && Kinv && freqs && cq_x && cq_y && cv_x && cv_y && det_b && det_y && det_x && count && zc && query &&
                   vals, "null argument");
  MHMR_REQUIRE(xr == nullptr || (norm_g && norm_b), "person_gather: the refined rows need the final norm");
  return person_gather(z32, xr, norm_g, norm_b, Kinv, freqs, cq_x, cq_y, cv_x, cv_y, det_b, det_y, det_x, count,
                       max_persons, res, D, zc, query, vals, ldq, static_cast<cudaStream_t>(stream));
}

int mhmr_op_refine_prepare(const float* img, const void* img_u8, const float* lut, int S, const float* rowadd, int D,
                           const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons,
                           int n_cls, const float* cls_pos, int* rows_out, int* rowidx, float* patch, int ldp, float* xr,
                           void* stream) {
  MHMR_REQUIRE(S >= 14 && S % 14 == 0 && D >= 1 && max_persons >= 0 && n_cls >= 0, "refine_prepare: bad sizes");
  if (n_cls + max_persons == 0) return MHMR_OK;
  MHMR_REQUIRE(rowadd && det_b && det_y && det_x && count && rowidx && patch && xr, "null argument");
  MHMR_REQUIRE(img_u8 == nullptr || lut != nullptr, "refine_prepare: the uint8 image needs its table");
  return refine_prepare(img, static_cast<const uint8_t*>(img_u8), lut, S, rowadd, D, det_b, det_y, det_x, count,
                        max_persons, S / 14, n_cls, cls_pos, rows_out, rowidx, patch, ldp, xr,
                        static_cast<cudaStream_t>(stream));
}

int mhmr_op_kv_add_rows(float* KV, int64_t ldkv, const float* dKV, int ncols, const int* det_b, const int* det_y,
                        const int* det_x, const int* count, int max_persons, int res, void* stream) {
  MHMR_REQUIRE(max_persons >= 0 && res >= 1 && ncols >= 1 && ldkv >= ncols, "kv_add_rows: bad sizes");
  if (max_persons == 0) return MHMR_OK;
  MHMR_REQUIRE(KV && dKV && det_b && det_y && det_x && count, "null argument");
  return kv_add_rows(KV, ldkv, dKV, ncols, det_b, det_y, det_x, count, max_persons, res,
                     static_cast<cudaStream_t>(stream));
}

int mhmr_op_cls_gather(const void* X, const void* Xlo, int64_t ld, int T, int B, int D, float* out, void* stream) {
  MHMR_REQUIRE(X && out, "null argument");
  MHMR_REQUIRE(B >= 1 && T >= 1 && D >= 1 && ld >= D, "cls_gather: bad sizes");
  return cls_gather(X, static_cast<const __half*>(Xlo), ld, T, B, D, out, static_cast<cudaStream_t>(stream));
}

int mhmr_op_anny_gather(const float* z32, const float* xr, const float* norm_g, const float* norm_b, const float* pos,
                        const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons, int res,
                        int D, int dim, float* zc, float* xa, void* stream) {
  MHMR_REQUIRE(max_persons >= 0 && res >= 1 && D >= 1 && dim >= 1, "anny_gather: bad sizes");
  if (max_persons == 0) return MHMR_OK;
  MHMR_REQUIRE(z32 && pos && det_b && det_y && det_x && count && zc && xa, "null argument");
  MHMR_REQUIRE(xr == nullptr || (norm_g && norm_b), "anny_gather: the refined rows need the final norm");
  return anny_gather(z32, xr, norm_g, norm_b, pos, det_b, det_y, det_x, count, max_persons, res, D, dim, zc, xa,
                     static_cast<cudaStream_t>(stream));
}

int mhmr_op_anny_place(const float* bone_poses, const float* transl, const float* K_det, int center, int P, int V, int J,
                       float* v3d, float* j3d, float* v2d, float* j2d, float* transl_pelvis, void* stream) {
  MHMR_REQUIRE(P >= 0 && P <= 65535 && V >= 0 && J >= 1 && center >= 0 && center < J, "anny_place: bad sizes");
  if (P == 0) return MHMR_OK;
  MHMR_REQUIRE(bone_poses && transl && K_det && (V == 0 || v3d) && j3d && j2d && transl_pelvis, "null argument");
  return anny_place(bone_poses, transl, K_det, center, P, V, J, v3d, j3d, v2d, j2d, transl_pelvis,
                    static_cast<cudaStream_t>(stream));
}

}  // extern "C"
