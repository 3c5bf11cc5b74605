/*
 * libmhmr_sm90.so — C-ABI of the H100-native Multi-HMR inference path.
 *
 * Drop-in boundary for the ONE hot path of naver/multi-hmr: `Model.forward(x, K)` as called by
 * `demo.py:forward_model` (reference demo.py:108-126, model.py:205-349).  The reference has no native
 * layer (pure PyTorch); what this library replaces are the ATen/cuBLAS/cuDNN dispatches listed in
 * SURVEY.md §2.4 (k1..k19).  Signatures use plain pointers and sizes only (no torch types): device
 * buffers are borrowed for the duration of a call, `stream` is a `cudaStream_t` passed as void*.
 *
 * Every function returns 0 on success and a negative code on failure; `mhmr_last_error()` returns a
 * thread-local message.  Nothing here falls back to a CPU path: without a CUDA device the compute
 * entry points fail loudly.
 */
#ifndef MHMR_H_
#define MHMR_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MHMR_OK 0
#define MHMR_ERR_CUDA (-1)
#define MHMR_ERR_ARG (-2)
#define MHMR_ERR_STATE (-3)
#define MHMR_ERR_CAPACITY (-4)
#define MHMR_ERR_UNSUPPORTED (-5)

const char* mhmr_last_error(void);

/* ------------------------------------------------------------------------------------------------
 * Stage-level operators (unit parity + ncu targets)
 * ---------------------------------------------------------------------------------------------- */

/* Epilogue kinds of mhmr_op_gemm_f16 */
#define MHMR_EPI_BIAS_F16 0      /* out16 = acc + bias                — dinov2 Attention.qkv              */
#define MHMR_EPI_BIAS_GELU_F16 1 /* out16 = gelu_erf(acc + bias)      — dinov2 Mlp.fc1 + nn.GELU          */
#define MHMR_EPI_BIAS_RELU_F16 2 /* out16 = relu(acc + bias)          — regression_mlp, model.py:596-609  */
#define MHMR_EPI_LS_RESID_F32 3  /* out32 += gamma*(acc + bias)       — attn.proj / mlp.fc2 + LayerScale  */
#define MHMR_EPI_ROWADD_F32 4    /* out32[remap(m)] = acc + rowadd[m % rows_in] — patch-embed + pos-embed */
#define MHMR_EPI_BIAS_F32 5      /* out32 = acc (+ bias)              — HPH to_kv, cross_attn_transformer.py:187 */

/* C = epilogue(A[M,K] x W[N,K]^T): fp16 operands (K contiguous, torch nn.Linear weight layout), fp32
 * accumulation on the wgmma tensor cores.  Replaces torch.nn.functional.linear on the hot path
 * (reference blocks/dinov2.py:25 -> dinov2 Attention/Mlp; model.py:135; cross_attn_transformer.py:187).
 * Row remap for MHMR_EPI_ROWADD_F32: out_row = (m / rows_in) * rows_out + row_off + m % rows_in.
 * block_n: 128 or 256 = single-CTA 128 x block_n tiles; 512 = CTA pairs (2-CTA cluster sharing the weight tile), 256 x 256 tiles. */
int mhmr_op_gemm_f16(const void* A, int64_t lda, const void* W, int64_t ldw, int M, int N, int K,
                     int epilogue, const float* bias, const float* gamma, const float* rowadd,
                     void* out, int64_t ldo, int rows_in, int rows_out, int row_off, int block_n,
                     void* stream);

/* One seam of a dinov2 Block with the LayerNorm folded into the GEMMs on both sides of it -- what the engine runs
 * between attention and the MLP (and between one block's MLP and the next block's attention):
 *     X += ls * (A @ Wp^T + bp)                       attn.proj / mlp.fc2 + LayerScale + residual (layers/block.py)
 *     out16 = act(LayerNorm(X; ln_g, ln_b, eps 1e-6) @ W^T + b)      norm2 -> mlp.fc1 (+ GELU) / norm1 -> attn.qkv
 * Between the two the residual stream is a two-term fp16 split X = hi + lo (22 significant bits, 4 bytes per element
 * like fp32): the first GEMM's epilogue updates (hi, lo) in place and leaves per-row partial (sum, sum of squares); the
 * second GEMM runs on the hi plane with the row-centred W * diag(ln_g) and applies 1/sigma in its epilogue.  A, Wp fp16
 * (K contiguous); X fp32 [M, D] in place (split on entry, merged on exit); W fp32 [N, D] (folded and rounded inside);
 * D multiple of 128 (<= 1024), N multiple of 32.
 * Unit-test entry: allocates its temporaries and synchronises the stream. */
int mhmr_op_resid_ln_linear_f16(const void* A, int64_t lda, const void* Wp, int64_t ldwp, const float* bp,
                                const float* ls, float* X, int M, int D, int Ka, const float* ln_g,
                                const float* ln_b, const float* W, const float* b, int N, int gelu, void* out16,
                                int64_t ldo, void* stream);

/* Multi-head self-attention of the ViT backbone, head dim 64: out[:, h*64:(h+1)*64] =
 * softmax(q_h k_h^T / 8) v_h per image.  qkv is [B*T, 3*D] fp16 (q | k | v column blocks, the layout the
 * qkv Linear produces), out is [B*T, D] fp16.  Replaces dinov2 Attention.forward's
 * `q*scale @ k^T -> softmax -> @ v` (reached from reference blocks/dinov2.py:25). */
int mhmr_op_attention(const void* qkv, int64_t ld_qkv, void* out, int64_t ldo, int B, int T, int D,
                      void* stream);

/* Image preprocessing on the device: uint8 [B,H,W,3] (RGB, HWC) -> fp32 [B,3,H,W] through a [3][256] fp32 table.
 * Replaces reference utils/image.py:12-24 `normalize_rgb` (called from demo.py:48 `open_image`); with the table the
 * host derives from that function the output is bit-identical, and the upload is 4x smaller.  W % 4 == 0. */
int mhmr_op_normalize_u8(const void* img_u8, const float* lut, float* out, int B, int H, int W, void* stream);

/* Person-decoder kernels (the per-person path after the backbone), each the engine's own launcher behind a thin
 * validating entry.  All pointers are device pointers; `count` is a device int32 holding the person count
 * (<= max_persons), read on the device as in the engine: grids are sized for max_persons and exit early, and rows
 * >= count are not written.  fp32 throughout. */

/* out[p, n] = resid[p, n] + act(LN(x[p, :K]) . W[n, :K] + bias[n]) for p < count; the skinny Linear of the HPH and
 * the regressors.  LN (ln_g, ln_b, eps; both or neither, K % 4 == 0) is applied to the input row, act 0 none,
 * 1 ReLU, 2 erf GELU; bias, LN and resid are nullable, out may equal resid (in-place residual update).
 * W pitch ldw >= K rounded up to 4, multiple of 4; its padding columns are multiplied by zero, so must be finite.
 * ldx % 4 == 0: 128-bit loads (ldx >= K rounded to 4); otherwise scalar loads.  cols: 16 or 32 output columns per
 * CTA (2 or 4 per warp), 0 lets the device's SM count decide as the engine does. */
int mhmr_op_skinny_linear(const float* x, int ldx, const int* count, int max_persons, int K, const float* W, int ldw,
                          const float* bias, int Nout, const float* ln_g, const float* ln_b, float ln_eps, int act,
                          const float* resid, int ldr, float* out, int ldo, int cols, void* stream);

/* HPH self-attention among the persons of each image (cross_attn_transformer.py:129-159, heads of 32,
 * softmax(q k^T / sqrt(32)) v): qkv [P, ld] = q | k | v column blocks of heads * 32; persons sorted by image,
 * det_b[p] their image, img_off[b] .. img_off[b + 1] the persons of image b. */
int mhmr_op_hph_self_attn(const float* qkv, int ld, const int* det_b, const int* img_off, const int* count,
                          int max_persons, int heads, float* out, int ldo, void* stream);

/* HPH cross-attention (cross_attn_transformer.py:185-205): person p attends to the N rows of image det_b[p] of
 * KV [B * N, ldkv], keys at columns k_col + h * 32, values at v_col + h * 32 (multiples of 4). */
int mhmr_op_hph_cross_attn(const float* q, int ldq, const float* KV, int64_t ldkv, int k_col, int v_col,
                           const int* det_b, const int* count, int max_persons, int heads, int N, float* out, int ldo,
                           void* stream);

/* Detection (model.py:145-149, :612-638): scores_out = scores * (maxpool_k(scores) == scores) (k in [1, 15]; padding
 * (k - 1) / 2, 1 for k = 2, 2 for k = 4), then the cells with scores_out >= thresh in (b, y, x) order: the first
 * max_persons of them in det_b / det_y / det_x / det_score, their true number in count, min(count, max_persons) in
 * count_clamped, and img_off[b] (B + 1 entries) = first kept person of image b. */
int mhmr_op_detect(const float* scores, int B, int res, int nms_k, float thresh, int max_persons, float* scores_out,
                   int* det_b, int* det_y, int* det_x, float* det_score, int* count, int* count_clamped, int* img_off,
                   void* stream);

/* SMPL-X per-person outputs (utils/humans.py:12-22, model.py:189-203, :272-275, :291, blocks/smpl_layer.py:123):
 * dec [P, ld_dec] = pose6 (318) | betas (num_betas) | cam (3) | expression (10); K [B, 3, 3] (inverted inside);
 * focal_norm = img_size / (2 tan 30 deg).  Writes rotmat [P, 53, 3, 3], rotvec [P, 53, 3], shape, expr, dist_pp,
 * dist, loc [P, 2], transl [P, 3], K_det [P, 3, 3].  Allocates a temporary and synchronises the stream. */
int mhmr_op_person_post(const float* dec, int ld_dec, int num_betas, const float* offset, const float* K, int B,
                        const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons,
                        float focal_norm, float* rotmat, float* rotvec, float* shape, float* expr, float* dist_pp,
                        float* dist, float* loc, float* transl, float* K_det, void* stream);

/* Anny camera and per-person outputs (encoder.py:50-56, multi_hmr.py:133-175): from hid [B, D] (the hidden layer of
 * mlp_fov_unique) fov [B], K_regressed and K_use [B, 3, 3] (K if given, else K_regressed); then per person the 6D
 * rows rot6d [P, ld6] (J joints) -> rotmat [P, J, 3, 3] blended with the identity by useful [J], rotmat_homo
 * [P, J, 4, 4], rotvec, dist = K_use[0,0] / max(exp(dist_pp), 1e-5), loc, transl, K_det, and shape [P, num_betas]
 * replaced by its sigmoid in place.  Allocates a temporary and synchronises the stream. */
int mhmr_op_anny_person_post(const float* hid, int D, const float* w2, const float* b2, const float* fov_max,
                             const float* K, int B, int img_size, float* fov, float* K_regressed, float* K_use,
                             const float* rot6d, int ld6, int J, const float* useful, float* shape, int num_betas,
                             const float* offset, const float* dist_pp, const int* det_b, const int* det_y,
                             const int* det_x, const int* count, int max_persons, float* rotmat, float* rotmat_homo,
                             float* rotvec, float* dist, float* loc, float* transl, float* K_det, void* stream);

/* Central-stream refinement (DESIGN.md §3) of `count` rows x [max_persons, D] in place, through `depth` dinov2
 * blocks: x += ls1 * (Wproj . O16[l][rowidx[p]] + bproj);  x += ls2 * (Wfc2 . gelu(Wfc1 . LN2(x) + bfc1) + bfc2)
 * (LayerNorm eps 1e-6).  Weights stacked per layer: Wproj [depth, D, D], Wfc1 [depth, 4D, D], Wfc2 [depth, D, 4D],
 * vectors [depth, D] (bfc1 [depth, 4D]); O16 fp16 [depth, rows_o16, D].  D % 4 == 0.  Bit-reproducible.
 * Allocates its temporaries and synchronises the stream. */
int mhmr_op_refine_chain(int depth, int D, const int* count, int max_persons, const float* Wproj, const float* bproj,
                         const float* ls1, const float* ln2_g, const float* ln2_b, const float* Wfc1, const float* bfc1,
                         const float* Wfc2, const float* bfc2, const float* ls2, const void* O16, int64_t rows_o16,
                         const int* rowidx, float* x, void* stream);

/* Backbone entry, folded LayerNorm and the gathers of the heads: the engine's own launchers behind thin validating
 * entries, arguments checked before any launch.  Device pointers; fp16 buffers are passed as void*.  Entries with a
 * person capacity read the count from the device int32 `count` like the person-decoder entries above, and return
 * without a launch for a capacity of 0. */

/* Patch rows of the 14x14/14 patch-embed conv: A[b*N + gy*(S/14) + gx, c*196 + ky*14 + kx] = fp16 of pixel
 * (c, gy*14 + ky, gx*14 + kx) of image b, from img fp32 [B,3,S,S] or img_u8 [B,S,S,3] through lut [3][256] (exactly
 * one source).  Columns 588 .. ldA-1 are not written. */
int mhmr_op_im2col_patch14(const float* img, const void* img_u8, const float* lut, int B, int S, void* A, int ldA,
                           void* stream);
/* LayerNorm of M rows of width D (multiple of 128, <= 1024): X fp32 [M, D], or the two-term fp16 stream X = hi plane,
 * Xlo = lo plane.  out16 (fp16, pitch ld16) and out32 (fp32, pitch ld32) are each nullable, not both.  rows_in > 0:
 * row g*rows_in + t is dropped when t < skip, else written to row g*(rows_in - skip) + t - skip (the final norm drops
 * the cls row). */
int mhmr_op_layernorm(const void* X, const void* Xlo, const float* gamma, const float* beta, void* out16, int64_t ld16,
                      float* out32, int64_t ld32, int M, int D, float eps, int rows_in, int skip, void* stream);
/* Entry of the folded-LayerNorm chain: X fp32 [M, D] -> xhi = fp16(X), xlo = fp16(X - xhi) (pitch ld16), and
 * stats [M, slots] (sum, sum of squares) pairs: slot 0 the whole row, slots >= 1 zero. */
int mhmr_op_split_rowstats(const float* X, void* xhi, void* xlo, int64_t ld16, float* stats, int slots, int M, int D,
                           void* stream);
/* Load-time folding of a LayerNorm into the Linear after it: W16[n,k] = fp16(W[n,k] ln_g[k] - mean_k(W[n,:] ln_g)),
 * bias2[n] = bias[n] + sum_k ln_b[k] W[n,k]; W fp32 [N, K], W16 fp16 [N, K]. */
int mhmr_op_fold_ln_linear(const float* W, const float* bias, const float* ln_g, const float* ln_b, void* W16,
                           float* bias2, int N, int K, void* stream);
/* The GEMM of mhmr_op_gemm_f16 as the engine runs it: every epilogue kind (0-5 as above, with rows_out / row_off
 * for kind 4, and the internal kinds 6-9), and a plan built for M rows but run on the first M_run <= M of them
 * (M_run 0 runs all M), which is how the engine runs its maximum-batch plans at a smaller batch: rows
 * M_run .. M-1 of A are loaded and nothing is written for them.
 *   6  LS_RESID_SPLIT  x = (x16 + xlo) + gamma * (acc + bias) written back as two fp16 planes (pitch ldx16), and per
 *                      row the (sum, sum of squares) of the new x over the N/stat_slots columns of each slot into
 *                      stats [M, stat_slots]; stat_slots = 2 * ceil(N / tile), tile 128 (block_n 128) or 256
 *   7  LN_BIAS_F16     out16 = rstd * acc + bias, rstd = 1/sqrt(max(q/K - (s/K)^2, 0) + 1e-6) from the slot sums of
 *                      stats
 *                      [M, stat_slots] (stat_slots even, <= 8)
 *   8  LN_GELU_F16     out16 = gelu_erf(rstd * acc + bias)
 *   9  ROWADD_F16      out16 = acc + rowadd[m % rows_in] */
int mhmr_op_gemm_internal(const void* A, int64_t lda, const void* W, int64_t ldw, int M, int N, int K, int epilogue,
                          const float* bias, const float* gamma, void* x16, void* xlo, int64_t ldx16, float* stats,
                          int stat_slots, const float* rowadd, int rows_in, int rows_out, int row_off, void* out,
                          int64_t ldo, int block_n, int M_run, void* stream);
/* Camera rays of every token (model.py:160-187): Kinv [B, 3, 3] = K^-1, then ctx[b*res*res + n, col0 + j] = fp16 of
 * feature j < 99 of cell n (the (row, col) grid passed as (x, y)), zero for 99 <= j < pad_cols (<= 128). */
int mhmr_op_camera_ctx(const float* K, int B, const float* freqs, float* Kinv, void* ctx, int64_t ld, int res, int col0,
                       int pad_cols, void* stream);
/* scores[r] = sigmoid(hid[r, :D] . w + b[0]) for r < M, hid fp16 (pitch ld); clamped to [1e-4, 1 - 1e-4] when clamp
 * is set; logits (nullable) receives the dot product plus bias. */
int mhmr_op_rowdot_sigmoid(const void* hid, int64_t ld, const float* w, const float* b, float* scores, float* logits,
                           int clamp, int M, int D, void* stream);
/* Per person: zc [P, D] = feature row of the cell (z32 [B*res*res, D]), or LayerNorm(xr[p]; norm_g, norm_b, 1e-6) when
 * xr is given; query [P, ldq] = cat(zc, camera feature) + cq_x[y] + cq_y[x]; vals [P, ldq] = cv_x[y] + cv_y[x]
 * (tables [res, D + 99]); columns D + 99 .. ldq-1 of query and vals are zero. */
int mhmr_op_person_gather(const float* z32, const float* xr, const float* norm_g, const float* norm_b, const float* Kinv,
                          const float* freqs, const float* cq_x, const float* cq_y, const float* cv_x, const float* cv_y,
                          const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons,
                          int res, int D, float* zc, float* query, float* vals, int ldq, void* stream);
/* Inputs of the central-stream refinement: rows [0, n_cls) are the cls rows of images 0..n_cls-1 (rowidx b*(N+1),
 * zero patch, xr = cls_pos), row n_cls + p is person p (rowidx b*(N+1) + 1 + cell, its 588 pixels in (c, ky, kx)
 * order from img fp32 or img_u8 + lut, xr = rowadd[cell]); patch pitch ldp; rows_out (nullable) = n_cls + count. */
int mhmr_op_refine_prepare(const float* img, const void* img_u8, const float* lut, int S, const float* rowadd, int D,
                           const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons,
                           int n_cls, const float* cls_pos, int* rows_out, int* rowidx, float* patch, int ldp, float* xr,
                           void* stream);
/* KV[b*res*res + y*res + x, :ncols] += dKV[p, :ncols] once per distinct cell of the persons p < count (model.py:517). */
int mhmr_op_kv_add_rows(float* KV, int64_t ldkv, const float* dKV, int ncols, const int* det_b, const int* det_y,
                        const int* det_x, const int* count, int max_persons, int res, void* stream);
/* out[b, :D] = row b*T of the residual stream: X fp32, or the two-term split X = hi, Xlo = lo (fp16); pitch ld. */
int mhmr_op_cls_gather(const void* X, const void* Xlo, int64_t ld, int T, int B, int D, float* out, void* stream);
/* Anny decoder inputs per person: zc [P, D] as in mhmr_op_person_gather, xa [P, dim] = pos[cell]. */
int mhmr_op_anny_gather(const float* z32, const float* xr, const float* norm_g, const float* norm_b, const float* pos,
                        const int* det_b, const int* det_y, const int* det_x, const int* count, int max_persons, int res,
                        int D, int dim, float* zc, float* xa, void* stream);
/* Placement of P bodies (mhmr_anny_place with the centre bone given): v3d in place and j3d from bone_poses, both
 * shifted by transl - bone(center); v2d (nullable), j2d projected with K_det; transl_pelvis = j3d[:, 0]. */
int mhmr_op_anny_place(const float* bone_poses, const float* transl, const float* K_det, int center, int P, int V, int J,
                       float* v3d, float* j3d, float* v2d, float* j2d, float* transl_pelvis, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Engine: the whole `Model.forward(x, K)` path (reference model.py:205-349) behind one handle
 * ---------------------------------------------------------------------------------------------- */
typedef struct mhmr_engine mhmr_engine;

typedef struct mhmr_config {
  int arch;              /* 0 = dinov2_vits14, 1 = dinov2_vitb14, 2 = dinov2_vitl14 (Model(backbone=...), model.py:35) */
  int img_size;          /* Model(img_size=...), multiple of 14 (model.py:37,65) */
  int max_batch;         /* capacity of the activation workspaces */
  int max_persons;       /* capacity of the per-person buffers; more detections => MHMR_ERR_CAPACITY */
  int xat_depth;         /* Model(xat_depth=...)     model.py:42 */
  int xat_num_heads;     /* Model(xat_num_heads=...) model.py:43 */
  int num_betas;         /* Model(num_betas=...)     model.py:47 (10 or 11) */
  int person_center_idx; /* index of Model(person_center=...) in smplx JOINT_NAMES ('head' = 15) */
  int num_verts;         /* body-model vertices (SMPL-X: 10475) */
  int refine_central;    /* 1: fp32 refinement of the detected tokens' residual streams (DESIGN.md §3); 0: bulk fp16 pass only */
  /* Appended fields; all zero = the SMPL-X head above.  With head == MHMR_HEAD_ANNY, xat_depth / xat_num_heads are
   * the Anny HPH's (multi_hmr_anny/multi_hmr.py:28-33, dim_head 32), person_center_idx is the index of the centre
   * bone in the body model's bone_labels, num_betas is the shape-head width (11), and num_verts is unused. */
  int head;              /* MHMR_HEAD_SMPLX (0) or MHMR_HEAD_ANNY (1) */
  int xat_dim;           /* Anny: HPH width (512), multiple of 32 */
  int xat_mlp_dim;       /* Anny: HPH FeedForward hidden width (2048), multiple of 32 */
  int num_joints;        /* Anny: body-model bones / rotations per person (163) */
} mhmr_config;

#define MHMR_HEAD_SMPLX 0
#define MHMR_HEAD_ANNY 1

/* Per-call outputs: device buffers owned by the caller (torch tensors), sized for max_persons.
 * Person order = torch.where order (b, y, x) (model.py:149,616).  Nullable: v2d, z. */
typedef struct mhmr_outputs {
  float* scores_map;   /* [B, res, res]    'scores' (after NMS in inference mode, model.py:145-157)      */
  int32_t* count;      /* [1]              number of detected persons P                                   */
  int32_t* det_idx;    /* [3, max_persons] image index b, row y, col x of each person                     */
  float* det_score;    /* [max_persons]    person 'scores'                                                */
  float* offset;       /* [max_persons, 2] mlp_offset output (model.py:258)                               */
  float* loc;          /* [max_persons, 2] 'loc' (model.py:272-275)                                       */
  float* dist_pp;      /* [max_persons]    'dist_postprocessed' (raw pred_cam[:,0])                       */
  float* dist;         /* [max_persons]    'dist' (model.py:189-203)                                      */
  float* rotmat;       /* [max_persons, 53, 3, 3]                                                         */
  float* rotvec;       /* [max_persons, 53, 3]                                                            */
  float* shape;        /* [max_persons, num_betas]                                                        */
  float* expression;   /* [max_persons, 10]                                                               */
  float* transl;       /* [max_persons, 3]                                                                */
  float* transl_pelvis;/* [max_persons, 3]                                                                */
  float* v3d;          /* [max_persons, V, 3]                                                             */
  float* v2d;          /* [max_persons, V, 2]   nullable (not part of the inference person dict)          */
  float* j3d;          /* [max_persons, 127, 3]                                                           */
  float* j2d;          /* [max_persons, 127, 2]                                                           */
  float* z;            /* [B, N, D] backbone features (blocks/dinov2.py:25), nullable (stage parity)      */
} mhmr_outputs;

/* Replaces `Model(**ckpt_args)` (reference demo.py:98-100, model.py:33-131). */
int mhmr_create(const mhmr_config* cfg, mhmr_engine** out);
int mhmr_destroy(mhmr_engine* h);

/* Replaces `model.load_state_dict(ckpt['model_state_dict'], strict=False)` (demo.py:103): one call per
 * fp32 tensor, `key` = the reference's state_dict key (SURVEY.md Appendix B).  `data` may be a host or a
 * device pointer; the engine keeps its own device copy.  Extra keys the C-ABI expects:
 *   backbone.encoder.pos_embed  must already be interpolated to the working grid: [1, 1+N, D]
 *   camera.freq_bands           [16] = torch.linspace(1, 32, 16)   (blocks/camera_embed.py:46)
 *   smplx.{v_template,shapedirs,expr_dirs,posedirs,J_regressor,lbs_weights,lmk_bary_coords}
 *                               the buffers smplx.create() registers (blocks/smpl_layer.py:38). */
int mhmr_set_weight(mhmr_engine* h, const char* key, const float* data, int64_t numel);
/* Integer body-model tables: smplx.parents [55], smplx.extra_joints_idxs [21],
 * smplx.lmk_tri [51*3] (= faces[lmk_faces_idx]). */
int mhmr_set_table_i32(mhmr_engine* h, const char* key, const int32_t* data, int64_t numel);
/* Repack (fp16 K-major weight tiles, fused tables, folded joint regressor), allocate workspaces, build
 * TMA descriptors.  Fails if a required key is missing. */
int mhmr_finalize(mhmr_engine* h);

/* One forward of `Model.forward(x, idx, det_thresh, nms_kernel_size, K, is_training)` (model.py:205-349):
 * x [B,3,S,S] fp32 NCHW and K [B,3,3] fp32 are DEVICE pointers.  forced_idx (nullable) is a device
 * int64 [4, forced_P] tensor (b, y, x, c) = the reference's `idx=` argument (training-style path,
 * model.py:150-151: no NMS/threshold).  Asynchronous on `stream`; no host synchronisation. */
int mhmr_forward(mhmr_engine* h, const float* x, const float* K, int B, float det_thresh,
                 int nms_kernel_size, const int64_t* forced_idx, int forced_P, const mhmr_outputs* out,
                 void* stream);
/* The same forward fed by the fused image loader (SURVEY.md §8f row 1; replaces `normalize_rgb` of
 * utils/image.py:12-24 + the fp32 upload of demo.py:48-50): img_u8 [B,S,S,3] uint8 RGB (HWC, what PIL yields after
 * ImageOps.pad) and the [3][256] fp32 table of normalize_rgb; uint8 -> normalised fp16 patch rows in one kernel. */
int mhmr_forward_u8(mhmr_engine* h, const uint8_t* img_u8, const float* lut, const float* K, int B, float det_thresh,
                    int nms_kernel_size, const int64_t* forced_idx, int forced_P, const mhmr_outputs* out,
                    void* stream);
/* Waits for the forward enqueued last on `stream` and returns the person count; MHMR_ERR_CAPACITY if it
 * exceeded max_persons (outputs are then incomplete — never silently truncated). */
int mhmr_sync_count(mhmr_engine* h, void* stream, int* num_persons);

/* ------------------------------------------------------------------------------------------------
 * Anny variant: `Multi_HMR.forward` of multi_hmr_anny/multi_hmr.py:98-246 on an engine created with
 * head == MHMR_HEAD_ANNY.  The body model (the `anny` package) is NOT part of the library: mhmr_forward_anny computes
 * everything up to its inputs (rotmat_homo, shape), the caller runs the body model, and mhmr_anny_place finishes
 * (centre bone, translation, projection).  Weights are set under the checkpoint's own keys (encoder.backbone.*,
 * encoder.mlp_det.*, encoder.mlp_fov_unique.*, dec_to_token.*, decoder.transformer.layers.*, mlp_{offset,pose,
 * shape,dist}.*, useful_rotmat, init_body_pose, dec_pos_emb); encoder.backbone.pos_embed interpolated as above.
 * Person order = (b, y, x); the depth sort of the reference is left to the caller.
 * ---------------------------------------------------------------------------------------------- */
typedef struct mhmr_anny_outputs {
  float* scores_map;   /* [B, res, res]   sigmoid of the detection logits, NMS applied in inference mode       */
  float* logits;       /* [B, res, res]   'scores_logits' (before NMS)                                          */
  int32_t* count;      /* [1]             number of persons P                                                   */
  int32_t* det_idx;    /* [3, max_persons] b, y, x                                                              */
  float* K_regressed;  /* [B, 3, 3]       intrinsics from the regressed field of view (encoder.py:50-56)        */
  float* fov;          /* [B]             regressed field of view, radians                                      */
  float* K_det;        /* [max_persons, 3, 3] intrinsics used for each person (K, or K_regressed when K is NULL) */
  float* offset;       /* [max_persons, 2]                                                                      */
  float* loc;          /* [max_persons, 2]                                                                      */
  float* dist;         /* [max_persons]   focal / clamp(exp(dist_pp), 1e-5)                                     */
  float* dist_pp;      /* [max_persons]   raw mlp_dist output ('dist_postprocessed')                            */
  float* shape;        /* [max_persons, num_betas] sigmoid(mlp_shape)                                           */
  float* rotmat;       /* [max_persons, J, 3, 3]  after the useful_rotmat blend                                 */
  float* rotmat_homo;  /* [max_persons, J, 4, 4]  homogeneous form (the body model's pose_parameters)           */
  float* rotvec;       /* [max_persons, J, 3]                                                                   */
  float* transl;       /* [max_persons, 3]  K^-1 [loc, 1] dist                                                  */
  float* z;            /* [B, N, D] backbone features, nullable                                                 */
} mhmr_anny_outputs;

/* x [B,3,S,S] fp32 (mhmr_forward_anny) or img_u8 [B,S,S,3] + table (mhmr_forward_anny_u8); K [B,3,3] or NULL (the
 * regressed intrinsics are used); forced_idx as in mhmr_forward.  nms_kernel_size must be odd.  Asynchronous. */
int mhmr_forward_anny(mhmr_engine* h, const float* x, const float* K, int B, float det_thresh, int nms_kernel_size,
                      const int64_t* forced_idx, int forced_P, const mhmr_anny_outputs* out, void* stream);
int mhmr_forward_anny_u8(mhmr_engine* h, const uint8_t* img_u8, const float* lut, const float* K, int B,
                         float det_thresh, int nms_kernel_size, const int64_t* forced_idx, int forced_P,
                         const mhmr_anny_outputs* out, void* stream);
/* After the body model, for P persons (device pointers): v3d [P,V,3] (vertices in, camera-space vertices out, in
 * place), j3d [P,J,3] out from bone_poses [P,J,4,4] (translation column), both shifted by -bone(center) + transl;
 * j2d [P,J,2] and (nullable) v2d [P,V,2] projected with K_det; transl_pelvis [P,3] = j3d[:, 0]. */
int mhmr_anny_place(mhmr_engine* h, int P, int V, const float* bone_poses, const float* transl, const float* K_det,
                    float* v3d, float* j3d, float* v2d, float* j2d, float* transl_pelvis, void* stream);

/* Stage-level entry: backbone only (blocks/dinov2.py:16-26): x [B,3,S,S] -> z [B,N,D] fp32. */
int mhmr_vit_forward(mhmr_engine* h, const float* x, int B, float* z, void* stream);
/* Stage-level entry: the bulk pass of mhmr_vit_forward stopped after its patch embedding and first `layers` blocks
 * (0 <= layers <= depth): out [B,T,D] fp32 residual stream, cls row first.  Folded LayerNorm: hi + lo of the
 * two-term fp16 stream; MHMR_LN_FOLD=0: the fp32 stream. */
int mhmr_op_vit_stream(mhmr_engine* h, const float* x, int B, int layers, float* out, void* stream);
/* Stage-level entry: SMPL-X layer only (blocks/smpl_layer.py:47-155) for P persons (device pointers):
 * rotvec [P,53,3], shape [P,nb], expression [P,10], loc [P,2], dist [P], K_det [P,3,3]. */
int mhmr_smplx_forward(mhmr_engine* h, int P, const float* rotvec, const float* shape,
                       const float* expression, const float* loc, const float* dist, const float* K_det,
                       float* v3d, float* v2d, float* j3d, float* j2d, float* transl, float* transl_pelvis,
                       void* stream);
/* Backward of mhmr_smplx_forward for the same inputs: upstream gradients g_v3d [P,V,3], g_v2d [P,V,2], g_j3d /
 * g_j2d [P,127,3 / 2], g_transl [P,3], g_transl_pelvis [P,3], each nullable (NULL = zero); input gradients
 * d_rotvec [P,53,3], d_shape [P,nb], d_expression [P,10] (nullable: not computed), d_loc [P,2], d_dist [P] are
 * written, not accumulated.  Stateless (recomputes the forward quantities it needs), no float atomics: repeated
 * calls are bitwise identical and each person's gradients do not depend on the other persons.  Asynchronous. */
int mhmr_smplx_backward(mhmr_engine* h, int P, const float* rotvec, const float* shape, const float* expression,
                        const float* loc, const float* dist, const float* K_det, const float* g_v3d, const float* g_v2d,
                        const float* g_j3d, const float* g_j2d, const float* g_transl, const float* g_transl_pelvis,
                        float* d_rotvec, float* d_shape, float* d_expression, float* d_loc, float* d_dist,
                        void* stream);
/* ------------------------------------------------------------------------------------------------
 * Sharded batches (one process per GPU, image shards per rank; SURVEY.md §8e).  The reference is single-GPU
 * (README.md:107); these entry points are what a multi-GPU caller of `forward_model` binds.
 *   block  = header (8 x int32: persons detected, persons packed, capacity, floats per record, first global
 *            image index of the rank, 0, 0, 0) | capacity x record (fp32)
 *   record = [global image index, score, loc 2, transl 3, transl_pelvis 3, rotvec 159, expression 10,
 *             shape nb, v3d 3V, j3d 381, j2d 254]  — the person dict of model.py:329-347
 * ---------------------------------------------------------------------------------------------- */
int mhmr_record_floats(int num_betas, int num_verts);
int64_t mhmr_record_block_bytes(int num_betas, int num_verts, int capacity);
/* ONE kernel: packs the (device-resident) outputs of a forward into `block`; the person count is read on the
 * device and travels in the header, unused record slots are zero-filled. */
int mhmr_pack_records(const mhmr_outputs* out, int max_persons, int num_betas, int num_verts, int image_offset,
                      int capacity, float* block, void* stream);
/* NCCL communicator of the record exchange (libnccl.so.2 is resolved at run time from the process). */
typedef struct mhmr_comm mhmr_comm;
int mhmr_nccl_unique_id(void* id128);                                   /* ncclGetUniqueId (rank 0) */
int mhmr_comm_create(const void* id128, int world, int rank, mhmr_comm** out);  /* ncclCommInitRank  */
int mhmr_comm_destroy(mhmr_comm* c);
/* ONE ncclAllGather of the per-rank blocks (all_blocks = world x block_bytes, rank order) on `stream`. */
int mhmr_allgather_records(mhmr_comm* c, const void* block, void* all_blocks, int64_t block_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Evaluation metrics (SURVEY.md §8f row 3): what the reference's `Trainer.evaluate` (train.py:336-482) computes
 * from the outputs of Model.forward.  All pointers are DEVICE pointers; nothing synchronises with the host.
 * ---------------------------------------------------------------------------------------------- */
/* Replaces utils/training.py:25-147 `match_2d_greedy(pred_kps, gtkp, valid_mask)` (valid=None, as train.py:364
 * calls it) including the IoU gate of :149-193: pred_j2d [P,J,2], gt_j2d [G,J,2] pixels, valid_mask [G,J] bytes or
 * NULL (all valid).  Outputs: pairs [min(P,G),2] = (pred, gt) in the order the greedy loop finds them, n_pairs [1],
 * pred_to_gt [P] (-1 = false positive), gt_to_pred [G] (-1 = miss).  P, G <= 48. */
int mhmr_eval_match_2d(const float* pred_j2d, const float* gt_j2d, const uint8_t* valid_mask, int P, int G, int J,
                       float iou_thresh, int32_t* pairs, int32_t* n_pairs, int32_t* pred_to_gt, int32_t* gt_to_pred,
                       void* stream);
/* Replaces train.py:373-394 (PVE / PA-PVE) and :411-427 (MPJPE / PA-MPJPE) for the matched pairs: point sets
 * pred [*,n,3], gt [*,n,3] (metres), optional per-person centres [*,3] subtracted first (the pelvis, train.py:376-382);
 * err_mm[m] = mean |gt - pred| * 1000, pa_err_mm[m] = the same after the similarity alignment of pred onto gt
 * (roma.rigid_points_registration(compute_scaling=True)).  One CTA per pair m < *n_pairs (m < max_pairs). */
int mhmr_eval_points_error(const float* pred, const float* pred_center, const float* gt, const float* gt_center,
                           const int32_t* pairs, const int32_t* n_pairs, int max_pairs, int n_points, float* err_mm,
                           float* pa_err_mm, void* stream);
/* Sparse regression of matched pairs, centre first (train.py:375-384, :406-415):
 *     out[m, i] = A[r] . (X[s] - center[s]) - (root >= 0 ? A[root] . (X[s] - center[s]) : 0)
 * with s = pairs[2m + side], r = rows[i] (rows NULL: r = i and R_out = R), for m < *n_pairs (m < max_pairs <= 48).
 * Device data is not range-checked here: rows[i] and root must lie in [0, R), pairs / n_pairs must come from
 * mhmr_eval_match_2d (or index X and center), CSR columns must lie in [0, N).
 * A [R, N] in CSR form (rowptr [R+1], col, val; rows need not sum to 1), X [*, N, 3], center [*, 3] nullable,
 * out [max_pairs, R_out, 3].  K [*, 3, 3] and out2d [max_pairs, R_out, 2] (both or neither) add the perspective
 * projection of the outputs (utils/camera.py:14-27).  Serves the SMPL-X -> SMPL transfer (smplx2smpl.pkl), the H36M
 * joints of 3DPW (J_regressor_h36m, rows H36M_TO_J14, root 0) and the EHF joints (J_regressor @ vertices). */
int mhmr_eval_regress(const int32_t* rowptr, const int32_t* col, const float* val, int R, int N, const int32_t* rows,
                      int R_out, int root, const float* X, const float* center, const int32_t* pairs, int side,
                      const int32_t* n_pairs, int max_pairs, const float* K, float* out, float* out2d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Ground-truth body models (Trainer.prepare_gt, train.py:58-134): the raw `smplx` forward with `transl`, as
 * smplx.create(SMPLX_DIR, 'smpl', gender=...) and smplx.create(..., 'smplx', gender='neutral', use_pca=False,
 * flat_hand_mean=True, num_betas=11) compute it (train.py:41-43).  Independent of the engine handle.
 *   MHMR_BODY_SMPL   24 joints, 207 pose features; joints = 24 LBS + 21 vertex-picked = 45; no expression
 *   MHMR_BODY_SMPLX  55 joints, 486 pose features, 10 expression coefficients; 55 + 21 + 51 landmarks = 127
 * ---------------------------------------------------------------------------------------------- */
#define MHMR_BODY_SMPL 0
#define MHMR_BODY_SMPLX 1
typedef struct mhmr_body mhmr_body;
/* Arrays (host or device, fp32 / int32; the handle keeps its own folded copies): v_template [V,3], shapedirs
 * [V,3,num_betas], expr_dirs [V,3,10] (SMPL-X), posedirs [9(NJ-1), 3V], J_regressor [NJ,V], lbs_weights [V,NJ],
 * parents [NJ] (parents[0] = -1, parents[j] < j), extra_joints_idxs [21] (smplx.vertex_ids order), lmk_tri [51*3] and
 * lmk_bary [51*3] (SMPL-X).  Every array is first copied into device memory (cudaMemcpyDefault), so host and device
 * pointers are both accepted.  Sizes (9 (NJ-1) + num_betas + expression <= 512) and table ranges are checked before
 * any kernel is launched; synchronises `stream`. */
int mhmr_body_create(int kind, int num_verts, int num_betas, int max_persons, const float* v_template,
                     const float* shapedirs, const float* expr_dirs, const float* posedirs, const float* J_regressor,
                     const float* lbs_weights, const int32_t* parents, const int32_t* extra_joints_idxs,
                     const int32_t* lmk_tri, const float* lmk_bary, void* stream, mhmr_body** out);
int mhmr_body_destroy(mhmr_body* h);
/* Any output pointer may be NULL.  num_joints_out = joints per person of mhmr_body_forward (45 or 127). */
int mhmr_body_info(const mhmr_body* h, int* num_verts, int* num_joints_out, int* num_pose_joints, int* num_betas,
                   int* num_expression);
/* P <= max_persons persons, device pointers: full_pose [P,NJ,3] in smplx order (SMPL: global, body 23; SMPL-X:
 * global, body 21, jaw, leye, reye, lhand 15, rhand 15), betas [P,num_betas], expression [P,10] (SMPL-X; NULL for
 * SMPL), transl [P,3], K [P,3,3].  Outputs v3d [P,V,3], v2d [P,V,2] (nullable), j3d / j2d [P,num_joints_out,3 / 2],
 * transl_pelvis [P,3] = j3d[:, 0]; vertices and joints include transl, j2d = perspective_projection(j3d, K). */
int mhmr_body_forward(mhmr_body* h, int P, const float* full_pose, const float* betas, const float* expression,
                      const float* transl, const float* K, float* v3d, float* v2d, float* j3d, float* j2d,
                      float* transl_pelvis, void* stream);
/* Backward of mhmr_body_forward for the same inputs: upstream gradients g_v3d [P,V,3], g_v2d [P,V,2], g_j3d / g_j2d
 * [P,num_joints_out,3 / 2], g_transl_pelvis [P,3], each nullable (NULL = zero); input gradients d_full_pose [P,NJ,3],
 * d_betas [P,num_betas], d_expression [P,10] (SMPL-X; nullable: not computed), d_transl [P,3] are written, not
 * accumulated.  Stateless, no float atomics, batch-independent bits; asynchronous. */
int mhmr_body_backward(mhmr_body* h, int P, const float* full_pose, const float* betas, const float* expression,
                       const float* transl, const float* K, const float* g_v3d, const float* g_v2d, const float* g_j3d,
                       const float* g_j2d, const float* g_transl_pelvis, float* d_full_pose, float* d_betas,
                       float* d_expression, float* d_transl, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Mesh renderer: the overlay of reference utils/render.py:175 `render_meshes` (pyrender / OpenGL there), reached from
 * demo.py:340-346 `overlay_human_meshes`, the rotating video (demo.py:159-195), app.py and train.py:440-469.  A
 * z-buffer rasterizer over meshes already on the device, for any body model (SMPL-X, Anny): one sample per pixel
 * centre, top-left fill rule, back faces culled, near plane 0.05 / far plane 100, pyrender's metallic-roughness
 * shading under a white directional light at the camera plus ambient 0.3, then the reference's 3x3 foreground
 * smoothing and alpha blend.  Four launches per call, no host synchronisation.
 * ---------------------------------------------------------------------------------------------- */
typedef struct mhmr_render mhmr_render;
typedef struct mhmr_render_args {
  int views, H, W;              /* B views of H x W pixels                                                        */
  const uint8_t* images;        /* backgrounds [*, H, W, 3] RGB                                                   */
  const int32_t* view_image;    /* [views]: background image of each view; person p is drawn into view b when
                                   person_image[p] == view_image[b]                                               */
  const float* K;               /* [views, 3, 3] intrinsics, fx > 0 and fy > 0 (a view without is left empty)     */
  const float* pose;            /* [views, 3, 4] world -> camera [R | t] (OpenCV convention, R a rotation), NULL = I */
  const float* verts;           /* [max_persons, num_verts, 3] in world (camera) coordinates, metres              */
  int max_persons;
  const int32_t* person_image;  /* [max_persons] image of each person (the engine's det_idx[0])                   */
  const int32_t* count;         /* [1] persons, read on the device (clamped to [0, max_persons])                  */
  const float* colors;          /* [max_persons, 3] base colours in [0, 1]                                        */
  float alpha, intensity, metallic, roughness;
  int smooth;                   /* 1: trimesh's angle-weighted vertex normals; 0: face normals                    */
  uint8_t* overlay;             /* out [views, H, W, 3]                                                           */
  float* depth;                 /* out [views, H, W] camera z, 0 = background (nullable)                          */
  int32_t* person;              /* out [views, H, W] person index, -1 = background (nullable)                     */
} mhmr_render_args;
/* faces int32 [F, 3] (host or device); every index must lie in [0, num_verts).  Builds the vertex -> face CSR of the
 * normal pass; synchronises `stream`. */
int mhmr_render_create(const int32_t* faces, int num_faces, int num_verts, void* stream, mhmr_render** out);
int mhmr_render_destroy(mhmr_render* h);
/* face_bits: bits of the depth key's low word that hold the face index; max_persons may be up to 2^(32 - face_bits). */
int mhmr_render_info(const mhmr_render* h, int* num_faces, int* num_verts, int* face_bits);
/* Every pointer of `a` is a device pointer.  The handle owns a key buffer of 8 B per pixel per view, grown on demand
 * (growing frees the old buffer, which waits for the device).  One call at a time per handle. */
int mhmr_render_forward(mhmr_render* h, const mhmr_render_args* a, void* stream);

/* Several topologies in one z-buffer.  A handle made by mhmr_render_create_topologies holds, besides the body mesh,
 * `num_topologies` extra face arrays (topology t: topo_num_faces[t] faces over topo_num_verts[t] vertices, its faces
 * in `topo_faces` after those of topologies 0..t-1, indices local to the topology), each with its own normal CSR.
 * The depth key's low word holds (mesh, face); face_bits is sized for the largest topology.  With num_topologies 0
 * this is mhmr_render_create. */
int mhmr_render_create_topologies(const int32_t* faces, int num_faces, int num_verts, int num_topologies,
                                  const int32_t* topo_faces, const int32_t* topo_num_faces,
                                  const int32_t* topo_num_verts, void* stream, mhmr_render** out);
#define MHMR_RENDER_MAX_PROPS 16
typedef struct mhmr_render_extra {
  int num_props;                /* extra meshes ("props") drawn next to the persons, <= MHMR_RENDER_MAX_PROPS     */
  const int32_t* prop_topology; /* HOST [num_props]: topology of each prop                                        */
  const float* prop_verts;      /* [sum of the props' vertex counts, 3] back to back, world coordinates            */
  const float* prop_colors;     /* [num_props, 3] base colours in [0, 1]                                          */
  const uint8_t* prop_visible;  /* [views, num_props]: nonzero draws prop j into view b; NULL = everywhere         */
  const float* view_alpha;      /* [views] blend alpha of each view; NULL = args->alpha                           */
  const int32_t* view_background; /* [views] background image of each view; NULL = args->view_image             */
} mhmr_render_extra;
/* mhmr_render_forward plus props, per-view alpha and backgrounds.  Mesh m of the key is person m for m <
 * max_persons and prop m - max_persons after; max_persons + num_props must fit the key next to the face index.  The
 * person map (args->person) holds that mesh index. */
int mhmr_render_forward_extra(mhmr_render* h, const mhmr_render_args* a, const mhmr_render_extra* e, void* stream);

/* Camera poses of the demo's views, on the device (demo.py:160-241 create_rotating_video, utils/render.py:407
 * render_side_views), one CTA per image.  Per image, the views are: the photo's own camera (identity); if n_frames
 * >= 2, the orbit frames i = 0..n_frames-1 of the sweeps y by +angle_range, y by -angle_range and x by
 * +angle_range degrees about the centroid of the image's first person ([R | c - R c]); if side, lookAt poses of the
 * displaced, side and bird's-eye views.  The first person is the first listed (person_image order) or, with `transl`,
 * the smallest transl z (ties to the first).  Arithmetic in fp64, rounded once to fp32. */
typedef struct mhmr_render_pose_args {
  int images, max_persons, num_verts;
  const int32_t* count;         /* [1] persons, read on the device                                                */
  const int32_t* person_image;  /* [max_persons]                                                                  */
  const float* verts;           /* [max_persons, num_verts, 3]                                                    */
  const float* transl_pelvis;   /* [max_persons, 3]: the side views look at the median pelvis z                   */
  const float* transl;          /* [max_persons, 3] or NULL: closest first by transl z (Anny's order)             */
  int n_frames;                 /* 0 (no orbit) or >= 2                                                           */
  double angle_range;           /* degrees                                                                        */
  int side;
  float* pose;                  /* out [images, views per image, 3, 4]                                            */
  uint8_t* nonempty;            /* out [images]: 1 when the image has a person                                    */
  int32_t* rank;                /* out [max_persons]: position of the person in its image's list, -1 past count   */
} mhmr_render_pose_args;
int mhmr_render_view_poses(const mhmr_render_pose_args* a, void* stream);

/* Kernel launches enqueued by the last mhmr_forward (bench.py's `gpu_launches`). */
int mhmr_last_launch_count(mhmr_engine* h);

/* Live per-kernel-family timing with CUDA events on the launching stream (bench.py's `roofline`):
 * while enabled, every launch of mhmr_forward is bracketed by an event pair; mhmr_get_profile waits for
 * them, returns the summed device milliseconds and launch counts per category and resets the record. */
#define MHMR_CAT_MISC 0        /* im2col, cls rows                          */
#define MHMR_CAT_LAYERNORM 1
#define MHMR_CAT_GEMM_QKV 2
#define MHMR_CAT_ATTENTION 3
#define MHMR_CAT_GEMM_PROJ 4
#define MHMR_CAT_GEMM_FC1 5
#define MHMR_CAT_GEMM_FC2 6
#define MHMR_CAT_GEMM_OTHER 7  /* patch-embed, detection hidden, HPH to_kv */
#define MHMR_CAT_HEAD 8        /* detection / HPH / post-processing kernels */
#define MHMR_CAT_SMPLX 9       /* prep + vertex + joints kernels            */
#define MHMR_CAT_REFINE 10     /* fp32 refinement of the detected tokens' residual streams */
#define MHMR_NUM_CATEGORIES 11
int mhmr_set_profiling(mhmr_engine* h, int enable);
int mhmr_get_profile(mhmr_engine* h, float* ms_by_category, int* launches_by_category);

#ifdef __cplusplus
}
#endif
#endif /* MHMR_H_ */
