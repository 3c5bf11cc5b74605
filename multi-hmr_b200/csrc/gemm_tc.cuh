// wgmma / TMA GEMM family for the Multi-HMR hot path (sm_90a).
//
//   C[M,N] = epilogue( A[M,K] (fp16, K-major) x W[N,K]^T (fp16, K-major, i.e. torch Linear.weight) )
//
// fp32 accumulation in registers.  The epilogues cover every Linear of the reference's ViT backbone and
// of the dense part of the head (SURVEY.md §2.4 k1,k3,k5,k6,k7,k9,k15):
//   EPI_BIAS_F16       out16 = acc + bias                       (qkv: dinov2 Attention.qkv)
//   EPI_BIAS_GELU_F16  out16 = gelu_erf(acc + bias)             (mlp.fc1 + nn.GELU)
//   EPI_BIAS_RELU_F16  out16 = relu(acc + bias)                 (regression_mlp hidden, model.py:596-609)
//   EPI_LS_RESID_F32   out32 += gamma * (acc + bias)  in place  (attn.proj / mlp.fc2 + LayerScale + residual)
//   EPI_ROWADD_F32     out32[remap(m)] = acc + rowadd[m % rows_in]  (patch-embed + bias + pos-embed scatter)
//   EPI_BIAS_F32       out32 = acc + bias (bias may be null)    (HPH to_kv, cross_attn_transformer.py:187)
//   EPI_ROWADD_F16     out16 = acc + rowadd[m % rows_in]         (Anny dec_to_token + bias + dec_pos_emb)
//
// LayerNorm folded into the two Linears that follow it (dinov2 Block: norm1 -> attn.qkv, norm2 -> mlp.fc1).
// With W'[n,k] = W[n,k] ln_gamma[k] - mean_k(W[n,:] ln_gamma) (rows centred, rounded to fp16) and
// b'[n] = b[n] + sum_k ln_beta[k] W[n,k]:
//     Linear(LN(x))[n] = rstd * sum_k x[k] W'[n,k] + b'[n]        (sum_k (x[k] - mean) W'[n,k] = sum_k x[k] W'[n,k])
// so the GEMM runs on the RAW residual stream and only 1/sigma enters, in the epilogue.  The raw fp16 operand costs
// nothing extra because the residual stream itself is kept as a two-term fp16 split x = hi + lo (22 significant
// bits; hi = fp16(x) IS the tensor-core operand, lo = fp16(x - hi)), the same 4 bytes per element as fp32:
//   EPI_LS_RESID_SPLIT   x = (hi + lo) + gamma * (acc + bias), written back as (hi, lo) in place, + per-row partial
//                        (sum, sum of squares) of the new x over the columns one epilogue warp owns:
//                        stats[m][slot], slot = 2 n_blk + par                  (attn.proj / mlp.fc2 + LayerScale)
//   EPI_LN_BIAS_F16      out16 = rstd acc + b'                       statistics reduced from stats[m][0..slots)
//   EPI_LN_GELU_F16      out16 = gelu_erf(rstd acc + b')
#pragma once
#include "common.cuh"

namespace mhmr {

enum GemmEpiKind : int {
  EPI_BIAS_F16 = 0,
  EPI_BIAS_GELU_F16 = 1,
  EPI_BIAS_RELU_F16 = 2,
  EPI_LS_RESID_F32 = 3,
  EPI_ROWADD_F32 = 4,
  EPI_BIAS_F32 = 5,
  EPI_NUM_PUBLIC_KINDS = 6,   // what mhmr_op_gemm_f16 accepts
  EPI_LS_RESID_SPLIT = 6,
  EPI_LN_BIAS_F16 = 7,
  EPI_LN_GELU_F16 = 8,
  EPI_ROWADD_F16 = 9,
  EPI_NUM_KINDS = 10,
};

struct GemmEpi {
  const float* bias = nullptr;    // [N]
  const float* gamma = nullptr;   // [N]            (EPI_LS_RESID_F32)
  const float* rowadd = nullptr;  // [rows_in, N]   (EPI_ROWADD_F32 / EPI_ROWADD_F16)
  void* out = nullptr;            // fp16 or fp32, row pitch ldo elements
  int64_t ldo = 0;
  // Row remap: out_row = (m / rows_in) * rows_out + row_off + (m % rows_in); rows_in == 0 => identity.
  int rows_in = 0, rows_out = 0, row_off = 0;
  // folded LayerNorm (see above)
  __half* x16 = nullptr;          // [M, ldx16] hi plane of the residual stream  (EPI_LS_RESID_SPLIT, in place)
  __half* xlo = nullptr;          // [M, ldx16] lo plane
  int64_t ldx16 = 0;
  float2* stats = nullptr;        // [M, stat_slots] partial (sum, sumsq)   (written by RESID_SPLIT, read by LN_*)
  int stat_slots = 0;
  float ln_eps = 1e-6f;
};

struct GemmPlan {
  CUtensorMap tmA, tmB;
  int M = 0, N = 0, K = 0;
  int bn = 256;          // 128 / 256: single-CTA tile width; 512: CTA pair (2-CTA cluster), 256 x 256 tile
  int epi = EPI_BIAS_F16;
  GemmEpi ep;
  int grid = 0;
};

// Build the TMA descriptors + launch geometry once (weights and workspaces are persistent).
int gemm_plan_init(GemmPlan* plan, const __half* A, int64_t lda, const __half* W, int64_t ldw, int M,
                   int N, int K, int epi_kind, const GemmEpi& ep, int bn);
int gemm_plan_run(const GemmPlan* plan, cudaStream_t stream);
// Runs the plan on its first M (<= plan->M) rows: re-gridded for M, rows M .. plan->M - 1 are loaded (the tensor
// map covers them) but neither stored nor counted in the statistics.  The engine runs its maximum-batch plans so.
int gemm_plan_run_rows(const GemmPlan* plan, int M, cudaStream_t stream);
// launch geometry for `M` rows with this plan's tile shape
int gemm_plan_grid(const GemmPlan* plan, int M);
// partial-statistics slots per row that an EPI_LS_RESID_SPLIT GEMM with N columns and tile selector `bn` writes
int gemm_stat_slots(int N, int bn);

}  // namespace mhmr
