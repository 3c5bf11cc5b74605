// Host-callable launchers of the non-GEMM kernels (one translation unit each).
#pragma once
#include <vector>

#include "common.cuh"

namespace mhmr {

// ---- attn_tc.cu ------------------------------------------------------------------------------
int attention_forward(const __half* qkv, int64_t ld_qkv, __half* out, int64_t ldo, int B, int T, int D,
                      cudaStream_t stream);

// ---- vit_misc.cu -----------------------------------------------------------------------------
int im2col_patch14(const float* x, __half* A, int B, int S, int ldA, cudaStream_t stream);
int normalize_u8(const uint8_t* img, const float* lut, float* out, int B, int H, int W, cudaStream_t stream);
int im2col_u8_patch14(const uint8_t* img, const float* lut, __half* A, int B, int S, int ldA, cudaStream_t stream);
int cls_rows(float* X, const float* cls_pos, int B, int T, int D, cudaStream_t stream);
int layernorm(const float* X, const float* gamma, const float* beta, __half* out16, int64_t ld16,
              float* out32, int64_t ld32, int M, int D, float eps, int rows_in, int skip,
              cudaStream_t stream);
int f32_to_f16_2d(const float* src, int64_t lds, __half* dst, int64_t ldd, int rows, int cols,
                  cudaStream_t stream);
// folded LayerNorm (gemm_tc.cuh): entry kernel of the chain and the load-time weight folding
int split_rowstats(const float* X, __half* xhi, __half* xlo, int64_t ld16, float2* stats, int slots, int M, int D,
                   cudaStream_t stream);
int merge_split(const __half* xhi, const __half* xlo, float* X, int64_t n, cudaStream_t stream);
// LayerNorm of a two-term fp16 stream (X = hi plane, Xlo = lo plane; Xlo == nullptr: X is fp32)
int layernorm_split(const void* X, const __half* Xlo, const float* gamma, const float* beta, __half* out16,
                    int64_t ld16, float* out32, int64_t ld32, int M, int D, float eps, int rows_in, int skip,
                    cudaStream_t stream);
int fold_ln_linear(const float* W, const float* bias, const float* ln_g, const float* ln_b, __half* W16,
                   float* bias2, int N, int K, cudaStream_t stream);
int repack_f32(const float* src, int64_t lds, int scol, float* dst, int64_t ldd, int dcol, int rows,
               int cols, bool zero_fill, cudaStream_t stream);
int add_vec(const float* a, const float* b, float* out, int64_t n, int64_t b_period, cudaStream_t stream);

// ---- head.cu ---------------------------------------------------------------------------------
// scores[r] = sigmoid(hid[r,:] . w + b), clamped to [1e-4, 1-1e-4] when `clamp` (SMPL-X head); logits nullable
int rowdot_sigmoid(const __half* hid, int64_t ld, const float* w, const float* b, float* scores, float* logits,
                   bool clamp, int M, int D, cudaStream_t st);
int nms_compact(const float* scores, float* scores_out, int B, int res, int nms_k, float thresh,
                int max_persons, int* det_b, int* det_y, int* det_x, float* det_score, int* count,
                int* count_clamped, int* img_off, cudaStream_t st);
int forced_detections(const float* scores, float* scores_out, int B, int res, const int64_t* idx4, int P,
               int* det_b, int* det_y, int* det_x, float* det_score, int* count, int* count_clamped,
               int* img_off, cudaStream_t st);
int loc_to_transl(const float* loc, const float* dist, const float* K_det, int P, float* transl,
                  cudaStream_t st);
int invert_K(const float* K, float* Kinv, int B, cudaStream_t st);
int ctx_fourier(const float* Kinv, const float* freqs, __half* ctx, int64_t ld, int B, int res, int D,
                int pad_cols, cudaStream_t st);
int person_gather(const float* z32, const float* xr, const float* norm_g, const float* norm_b, const float* Kinv,
                  const float* freqs, const float* cq_x, const float* cq_y, const float* cv_x, const float* cv_y,
                  const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons, int res,
                  int D, float* zc, float* query, float* vals, int ldq, cudaStream_t st);
// central-stream refinement (engine.cu:refine_streams): row indices, input patches and pos-embed rows of the
// detected cells, after n_cls leading cls rows (rows_out, nullable: n_cls + persons)
int refine_prepare(const float* img, const uint8_t* img_u8, const float* lut, int S, const float* rowadd, int D, const int* det_b, const int* det_y,
                   const int* det_x, const int* count, int max_persons, int res, int n_cls, const float* cls_pos,
                   int* rows_out, int* rowidx, float* patch, int ldp, float* xr, cudaStream_t st);
// each distinct cell once: persons that share a cell with an earlier person add nothing (their dKV rows are equal)
int kv_add_rows(float* KV, int64_t ldkv, const float* dKV, int ncols, const int* det_b, const int* det_y,
                const int* det_x, const int* count, int max_persons, int res, cudaStream_t st);
int skinny_linear(const float* x, int ldx, const int* count, int max_persons, int K, const float* W, int ldw,
                  const float* bias, int Nout, const float* ln_g, const float* ln_b, float ln_eps, int act,
                  const float* resid, int ldr, float* out, int ldo, cudaStream_t st);
// cols: columns per CTA, 16 or 32 (2 or 4 per warp); 0 picks 16 when 32 would leave SMs idle for one person chunk
int skinny_linear_ex(const float* x, int ldx, int cols, const int* count, int max_persons, int K, const float* W, int ldw,
                     const float* bias, int Nout, const float* ln_g, const float* ln_b, float ln_eps, int act,
                     const float* resid, int ldr, float* out, int ldo, cudaStream_t st);
// ---- refine.cu: central-stream refinement (DESIGN.md §3) -----------------------------------------
struct RefineLayer {
  const __half* O16;  // this block's attention output of the bulk pass [B*T, D]
  const float *Wproj, *bproj, *ls1, *ln2_g, *ln2_b, *Wfc1, *bfc1, *Wfc2, *bfc2, *ls2;  // fp32 masters
};
// term[l][p][:] = ls1_l * (W_proj_l . O16_l[rowidx[p], :] + b_proj_l) for every block l: ONE launch
int refine_proj_terms(const RefineLayer* layers, int depth, const int* rowidx, const int* count, int D,
                      int max_persons, float* term, cudaStream_t st);
// x[p][:] <- for every block: (x + term_l) + ls2_l * MLP_l(LN2_l(x + term_l)): ONE persistent cooperative launch
int refine_mlp_chain(const RefineLayer* layers, int depth, const int* count, int D, int max_persons, const float* term,
                     float* x, float* h, unsigned int* barrier, cudaStream_t st);
int hph_self_attn(const float* qkv, int ld, const int* det_b, const int* img_off, const int* count,
                  int max_persons, int heads, float* out, int ldo, cudaStream_t st);
int hph_cross_attn(const float* q, int ldq, const float* KV, int64_t ldkv, int k_col, int v_col,
                   const int* det_b, const int* count, int max_persons, int heads, int N, float* out,
                   int ldo, cudaStream_t st);
int person_post(const float* dec, int ld_dec, int num_betas, const float* offset, const float* K,
                const float* Kinv, const int* det_b, const int* det_y, const int* det_x, const int* count,
                int max_persons, float focal_norm, float* rotmat, float* rotvec, float* shape, float* expr,
                float* dist_pp, float* dist, float* loc, float* transl, float* K_det, cudaStream_t st);

// ---- head.cu: Anny variant (multi_hmr_anny/) -------------------------------------------------------
// out[b, :] = fp32 row b*T of the residual stream (X fp32, or the two-term split hi = X, lo = Xlo)
int cls_gather(const void* X, const __half* Xlo, int64_t ld, int T, int B, int D, float* out, cudaStream_t st);
// field of view, K_regressed, the intrinsics used (K or K_regressed) and their inverse from the hidden layer of
// mlp_fov_unique (encoder.py:50-56)
int anny_camera(const float* hid, int ldh, const float* w2, const float* b2, const float* fov_max, const float* K,
                int B, int S, float* fov, float* K_reg, float* K_use, float* Kinv, cudaStream_t st);
// per person: zc = final-normed feature (LN of the refined row xr, or the bulk row of z32), xa = dec_pos_emb[cell]
int anny_gather(const float* z32, const float* xr, const float* norm_g, const float* norm_b, const float* pos,
                const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons, int res,
                int D, int dim, float* zc, float* xa, cudaStream_t st);
// 6D -> R (J joints), useful_rotmat blend, rotvec, homogeneous 4x4; loc, dist, transl, sigmoid(shape), K_det
int anny_person_post(const float* rot6d, int ld6, int J, const float* useful, float* shape, int num_betas,
                     const float* offset, const float* dist_pp, const float* K_use, const float* Kinv,
                     const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons,
                     float* rotmat, float* rotmat_homo, float* rotvec, float* dist, float* loc, float* transl,
                     float* K_det, cudaStream_t st);
// after the body model: centre bone, translation, projection
int anny_place(const float* bone_poses, const float* transl, const float* K_det, int center, int P, int V, int J,
               float* v3d, float* j3d, float* v2d, float* j2d, float* transl_pelvis, cudaStream_t st);

// ---- smplx_lbs.cu ----------------------------------------------------------------------------
struct SmplxDeviceModel {
  int V = 0;            // vertices
  int L = 0;            // num_betas + expression coefficients (10 for SMPL-X, 0 for SMPL)
  int num_betas = 10;
  int center_idx = 15;  // person_center joint ('head')
  int num_joints = 55;  // kinematic joints (SMPL-X 55, SMPL 24)
  int pose_feat = 486;  // pose-corrective features = 9 (num_joints - 1)
  int n_lmk = 51;       // static face landmarks appended to the joints (SMPL: 0)
  int ldp = 0;          // PDX / vt row pitch: 3V rounded up to 4
  const float* PDX = nullptr;          // [pose_feat + L, ldp]
  const float* vt = nullptr;           // [ldp] v_template flattened
  const float* lbs_weights_padded = nullptr;  // [ceil(V/72)*72, num_joints], zero rows beyond V
  CUtensorMap tmPDX;                   // TMA descriptor of PDX (boxes of 16 rows x 220 columns)
  const float* Jt = nullptr;           // [num_joints, 3]   J_regressor . v_template
  const float* Jdirs = nullptr;        // [num_joints*3, L] J_regressor . shapedirs
  const int* parents = nullptr;        // [num_joints]
  const int* extra_idx = nullptr;      // [21] vertex-picked joints
  const int* lmk_tri = nullptr;        // [n_lmk, 3] vertex ids of the landmark faces
  const float* lmk_bary = nullptr;     // [n_lmk, 3]
};
struct SmplxScratch {
  float* cf = nullptr;      // [max_persons, pose_feat + L]
  float* Amat = nullptr;    // [max_persons, num_joints, 12]
  float* xf = nullptr;      // [max_persons, 16]
  float* jposed = nullptr;  // [max_persons, num_joints, 3]
};
int smplx_make_tmap(SmplxDeviceModel* bm);
int smplx_tile_verts();
int smplx_build_pdx(const float* posedirs, const float* sdirs_full, int PF, int L, int V, int ldp, float* PDX,
                    cudaStream_t st);
int smplx_fold_jreg(const float* Jr, const float* M, int NJ, int V, int Q, float* out, cudaStream_t st);
int smplx_forward(const SmplxDeviceModel& bm, const float* rotvec, const float* shape, const float* expr,
                  const float* transl, const float* K_det, const int* count, int max_persons,
                  SmplxScratch& ws, float* v3d, float* v2d, float* j3d, float* j2d, float* transl_pelvis,
                  cudaStream_t st);
// The raw body model (smplx.SMPL / smplx.SMPLX forward with transl): full_pose [P, num_joints, 3] in smplx order,
// betas [P, num_betas], expr [P, L - num_betas] (nullable when that is 0), transl [P, 3], K [P, 3, 3] for j2d / v2d.
int body_forward_raw(const SmplxDeviceModel& bm, const float* full_pose, const float* betas, const float* expr,
                     const float* transl, const float* K, const int* count, int max_persons, SmplxScratch& ws,
                     float* v3d, float* v2d, float* j3d, float* j2d, float* transl_pelvis, cudaStream_t st);

// Backward of the two layers (DESIGN.md §9).  Scratch sized by max_persons at create / finalize; each call
// recomputes what it needs from the inputs, so it does not depend on an earlier forward or its scratch.
struct SmplxGradScratch {
  int max_persons = 0;
  SmplxScratch fw;                  // recomputed prep (cf, A, placement, posed joints)
  float* v3d = nullptr;             // [Pm, V, 3] recomputed vertices (only when a 2-D upstream gradient is given)
  float *j3d = nullptr, *j2d = nullptr, *tp = nullptr;  // [Pm, J, 3], [Pm, J, 2], [Pm, 3]
  float* transl = nullptr;          // [Pm, 3] placed layer: K^-1 [loc, 1] dist
  float* gJ = nullptr;              // [Pm, J, 3] per-output-joint upstream gradient
  float* part = nullptr;            // [tiles, Pm, NJ*12 + KT + 12] per-tile partial sums
  size_t part_bytes = 0;
  int* count = nullptr;
  int *v2j_ptr = nullptr, *v2j_jt = nullptr;  // vertex -> output-joint table (CSR over vertices)
  float* v2j_w = nullptr;
};
// Upstream gradients; each nullable (= zero).  v3d [P,V,3], v2d [P,V,2], j3d [P,J,3], j2d [P,J,2], tp [P,3].
struct BodyGrads {
  const float *v3d = nullptr, *v2d = nullptr, *j3d = nullptr, *j2d = nullptr, *tp = nullptr;
};
// Placed layer: d_rotvec [P,53,3], d_shape [P,num_betas], d_expr [P,10] (nullable), d_loc [P,2], d_dist [P];
// d_rotmat [P,53,9] (nullable): the gradient with respect to each joint's rotation matrix R = exp(rotvec).
int smplx_backward(const SmplxDeviceModel& bm, SmplxGradScratch& gs, int P, const float* rotvec, const float* shape,
                   const float* expr, const float* loc, const float* dist, const float* K_det, const BodyGrads& g,
                   const float* g_transl, float* d_rotvec, float* d_shape, float* d_expr, float* d_loc, float* d_dist,
                   cudaStream_t st, float* d_rotmat = nullptr);
// Raw body model: d_full_pose [P,NJ,3], d_betas [P,num_betas], d_expr [P,10] (nullable), d_transl [P,3].
int body_backward_raw(const SmplxDeviceModel& bm, SmplxGradScratch& gs, int P, const float* full_pose,
                      const float* betas, const float* expr, const float* transl, const float* K, const BodyGrads& g,
                      float* d_full_pose, float* d_betas, float* d_expr, float* d_transl, cudaStream_t st);

// ---- train_loss.cu: the SMPL-X head's training loss and its gradient (DESIGN.md §10) ------------------------
// Targets and weights of mhmr_train_loss (include/mhmr.h), in that entry's order.
struct TrainTargets {
  const float *scores, *offset, *rotmat, *shape, *dist_pp, *transl, *transl_pelvis, *j3d, *v3d, *j2d, *v2d;
  int shape_dim;
};
struct LossWeights {
  float bce, offset, rotmat, shape, dist, transl, j3d, v3d, j2d, v2d;
};
struct TrainLossArgs {
  int B = 0, res = 0, P = 0, img_size = 0, use_2d = 0;
  const float* K = nullptr;  // [B, 3, 3]
  const mhmr_outputs* y_hat = nullptr;
  TrainTargets y;
  LossWeights w;
  float *loss = nullptr, *d_logits = nullptr, *d_offset = nullptr, *d_dec = nullptr;
};
// Arguments checked by the caller; enqueues everything on `st`.
int train_loss_smplx(const SmplxDeviceModel& bm, SmplxGradScratch& gs, const TrainLossArgs& a, cudaStream_t st);

// ---- body.cu: a body model on the device ----------------------------------------------------------
// The folded tables, the forward and backward scratch and the person count of one SMPL / SMPL-X layer, in zero-filled
// device allocations it owns and frees.
struct DeviceBody {
  SmplxDeviceModel bm;
  SmplxScratch ws;
  SmplxGradScratch gs;
  int* count = nullptr;  // device person count of a forward
  std::vector<void*> allocs;
  DeviceBody() = default;
  DeviceBody(const DeviceBody&) = delete;
  DeviceBody& operator=(const DeviceBody&) = delete;
  ~DeviceBody() {
    for (void* p : allocs) cudaFree(p);
  }
  template <typename T>
  int alloc(T** out, size_t n, cudaStream_t st) {
    void* p = nullptr;
    MHMR_CUDA_CHECK(cudaMalloc(&p, n * sizeof(T)));
    allocs.push_back(p);
    MHMR_CUDA_CHECK(cudaMemsetAsync(p, 0, n * sizeof(T), st));
    *out = static_cast<T*>(p);
    return MHMR_OK;
  }
};
// Loads a body model of `joints` kinematic joints (24: SMPL; 55: SMPL-X with 51 face landmarks) and V vertices into
// `b`, with scratch for max_persons.  The float arrays are device memory the folding kernels read; the integer tables
// (parents, extra_idx [21], lmk_tri [51, 3]) are read with cudaMemcpyDefault and checked on the host before `b` keeps
// device copies of them.  Synchronises `st`.
int body_build(DeviceBody* b, int joints, int V, int num_betas, int num_expr, int center_idx, int max_persons,
               const float* v_template, const float* shapedirs, const float* expr_dirs, const float* posedirs,
               const float* J_regressor, const float* lbs_weights, const int32_t* parents, const int32_t* extra_idx,
               const int32_t* lmk_tri, const float* lmk_bary, cudaStream_t st);
// (smplx_lbs.cu) Allocates b->gs through b and uploads the vertex -> joint table built from b->bm's extra_idx / lmk
// tables; synchronises `st`.
int smplx_grad_init(DeviceBody* b, int max_persons, cudaStream_t st);

}  // namespace mhmr
