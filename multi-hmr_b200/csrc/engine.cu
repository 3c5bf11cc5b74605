// Engine: weights, workspaces, TMA plans and the launch sequence of the whole Multi-HMR forward
// (reference model.py:205-349) behind the C-ABI of include/mhmr.h.
#include <cmath>
#include <map>
#include <memory>
#include <cstdlib>
#include <string>
#include <vector>

#include "gemm_tc.cuh"
#include "kernels.cuh"

using namespace mhmr;

namespace {

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
};

struct ArchSpec { int D, depth; };
const ArchSpec kArch[3] = {{384, 12}, {768, 12}, {1024, 24}};
constexpr int kHphDim = 1024;
constexpr int kCamDim = 99;

struct VitLayer {
  const float *ln1_g, *ln1_b, *ln2_g, *ln2_b, *bqkv, *bproj, *ls1, *bfc1, *bfc2, *ls2;
  __half *Wqkv, *Wproj, *Wfc1, *Wfc2;
  const float *Wproj32, *Wfc1_32, *Wfc2_32;  // fp32 masters (central-stream refinement)
  __half* O16;                               // this layer's attention output [max_batch*T, D]
  // norm1 / norm2 folded into qkv / fc1 (gemm_tc.cuh): biases with the LayerNorm beta folded in
  float *bqkv_f = nullptr, *bfc1_f = nullptr;
  GemmPlan qkv, proj, fc1, fc2;
};
struct HphLayer {
  const float *ln0_g, *ln0_b, *Wqkv, *Wsa_out, *bsa_out;
  const float *ln1_g, *ln1_b, *Wq, *Wca_out, *bca_out;
  const float *ln2_g, *ln2_b, *Wff0, *bff0, *Wff3, *bff3;
};
// fp32 weights the SMPL-X head reads as they are: camera.freq_bands, x_attention_head.cross_{queries,values}_{x,y},
// mlp_offset
struct SmplxHeadWeights {
  const float *freq_bands, *cq_x, *cq_y, *cv_x, *cv_y;
  const float *off0_w, *off0_b, *off2_w, *off2_b;
};
// the Anny head's: mlp_fov_unique and fov_max, dec_pos_emb, dec_to_token, the output Linears of the four regressors,
// useful_rotmat
struct AnnyHeadWeights {
  const float *fov0_w, *fov0_b, *fov2_w, *fov2_b, *fov_max, *dec_pos_emb, *dt_w, *dt_b;
  const float *off2_w, *off2_b, *dist2_w, *dist2_b, *shape2_w, *shape2_b, *pose2_w, *useful_rotmat;
};

}  // namespace

struct mhmr_engine {
  mhmr_config cfg{};
  std::string enc = "backbone.encoder.";   // state-dict prefix of the DINOv2 backbone
  int D = 0, depth = 0, res = 0, N = 0, T = 0, C = 0, Cp = 0, Cq = 0, nkv = 0, ndec = 0;
  int dec_dim = 0, dec_mlp = 0;            // HPH decoder width and feed-forward width
  bool finalized = false;
  std::map<std::string, DevBuf> weights;   // raw fp32 device copies, keyed like the state_dict
  std::map<std::string, DevBuf> tables;    // int32 tables
  std::vector<void*> owned;                // everything cudaMalloc'ed (freed in destroy)
  int launches = 0;
  bool profiling = false;
  struct ProfEntry { int cat; cudaEvent_t a, b; };
  std::vector<ProfEntry> prof;
  std::vector<cudaEvent_t> event_pool;
  size_t events_used = 0;
  cudaEvent_t next_event() {
    if (events_used == event_pool.size()) {
      cudaEvent_t ev;
      cudaEventCreate(&ev);
      event_pool.push_back(ev);
    }
    return event_pool[events_used++];
  }

  // packed weights
  __half* Wpatch = nullptr;   // [D, 592]
  float* rowadd = nullptr;    // [N, D]  pos_embed[1:] + patch bias
  float* cls_pos = nullptr;   // [D]
  std::vector<VitLayer> vit;
  const float *norm_g = nullptr, *norm_b = nullptr;   // final LayerNorm of the backbone
  __half* Wcls0 = nullptr;    // [D, D]
  const float *cls2_w = nullptr, *cls2_b = nullptr;   // detection output row [D] and bias [1]
  SmplxHeadWeights smplx_w{};
  AnnyHeadWeights anny_w{};
  __half* Wkv16 = nullptr;    // [nkv, Cp]
  float* Wkv32 = nullptr;     // [nkv, Cq]
  float* Wte_q = nullptr;     // [1024, Cq]
  float* te_const = nullptr;  // [1024]
  float* Wdec = nullptr;      // [ndec, 1024]
  float* bdec = nullptr;      // [ndec]
  std::vector<HphLayer> hph;
  DeviceBody body;   // the SMPL-X layer

  // workspaces
  __half *A16 = nullptr, *Xn16 = nullptr, *QKV16 = nullptr, *O16 = nullptr, *H16 = nullptr, *ctx16 = nullptr;
  bool ln_fold = true;       // MHMR_LN_FOLD=0: separate LayerNorm kernels (A/B measurements)
  float2* ln_stats = nullptr;  // [max_batch*T, ln_slots] partial row statistics of the residual stream
  __half* Xlo = nullptr;       // lo plane of the two-term fp16 residual stream (hi plane = Xn16), gemm_tc.cuh
  int ln_slots = 0;
  float *X = nullptr, *z32 = nullptr, *scores_raw = nullptr, *KV32 = nullptr, *Kinv = nullptr;
  int *count = nullptr, *img_off = nullptr;
  // central-stream refinement: token rows, input patches, residual streams and MLP hidden of the detected persons
  int* r_rowidx = nullptr;
  float *r_patch = nullptr, *r_x = nullptr, *r_h = nullptr, *r_term = nullptr;
  RefineLayer* r_layers = nullptr;   // device array [depth]
  unsigned int* r_barrier = nullptr;
  const float* Wpatch32 = nullptr;
  float *zc = nullptr, *query = nullptr, *vals = nullptr, *dKV = nullptr, *offh = nullptr, *xa = nullptr,
        *qkvp = nullptr, *att = nullptr, *qca = nullptr, *ffh = nullptr, *dec = nullptr, *K_det = nullptr;
  int* one = nullptr;  // device int == 1 (count for load-time skinny launches)
  GemmPlan patch_plan, cls0_plan, kv_plan;
  int* h_count = nullptr;  // pinned host copy of the person count
  int r_rows = 0;          // capacity of the refined rows (persons, plus one cls row per image for the Anny head)

  // Anny head (multi_hmr_anny/): decoder tokens of every cell, camera from the cls token, stacked regressors
  __half *Wdt16 = nullptr, *dec16 = nullptr;     // dec_to_token [dim, D]; tokens [max_batch*N, dim]
  float* dt_rowadd = nullptr;                    // [N, dim] dec_pos_emb + dec_to_token bias
  float *cls_x = nullptr, *cls_h = nullptr;      // [max_batch, D] bulk cls rows / mlp_fov_unique hidden
  float *K_use = nullptr, *det_score = nullptr;  // [max_batch, 9] intrinsics used; [max_persons] (NMS scratch)
  float *W1 = nullptr, *b1 = nullptr;            // [4 dim, dim]: first Linears of offset | dist | shape | pose
  float* b_pose2 = nullptr;                      // [6J] mlp_pose.2 bias + init_body_pose
  int* anny_ints = nullptr;                      // device [2]: batch size, refined rows
  GemmPlan dt_plan;

  ~mhmr_engine() {
    for (void* p : owned) cudaFree(p);
    for (auto& kv : weights) cudaFree(kv.second.p);
    for (auto& kv : tables) cudaFree(kv.second.p);
    if (h_count) cudaFreeHost(h_count);
    for (cudaEvent_t ev : event_pool) cudaEventDestroy(ev);
  }

  template <typename T>
  int alloc(T** out, size_t count_elems) {
    void* p = nullptr;
    const size_t bytes = count_elems * sizeof(T);
    MHMR_CUDA_CHECK(cudaMalloc(&p, bytes > 0 ? bytes : 16));
    MHMR_CUDA_CHECK(cudaMemset(p, 0, bytes > 0 ? bytes : 16));
    owned.push_back(p);
    *out = static_cast<T*>(p);
    return MHMR_OK;
  }
  const float* w(const std::string& key, int64_t expect_numel = -1) {
    auto it = weights.find(key);
    if (it == weights.end()) {
      set_last_error("missing weight: " + key);
      return nullptr;
    }
    if (expect_numel >= 0 && static_cast<int64_t>(it->second.bytes / 4) != expect_numel) {
      set_last_error("weight " + key + " has " + std::to_string(it->second.bytes / 4) + " elements, expected " +
                     std::to_string(expect_numel));
      return nullptr;
    }
    return static_cast<const float*>(it->second.p);
  }
  const int* tab(const std::string& key, int64_t expect_numel) {
    auto it = tables.find(key);
    if (it == tables.end() || static_cast<int64_t>(it->second.bytes / 4) != expect_numel) {
      set_last_error("missing or mis-sized table: " + key);
      return nullptr;
    }
    return static_cast<const int*>(it->second.p);
  }
};

namespace {

#define GETW(dst, key, numel)                           \
  if (((dst) = e->w(key, numel)) == nullptr) return MHMR_ERR_STATE;
#define NEEDW(var, key, numel)                          \
  const float* var;                                     \
  GETW(var, key, numel)

// CTA-pair 256x256 tiles (cta_group::2) whenever N is a multiple of 256, else single-CTA 128x128 tiles
int pick_bn(int N) { return (N % 256 == 0) ? 512 : 128; }

int to_f16(mhmr_engine* e, const float* src, int64_t lds, int rows, int cols, int64_t ldd, __half** out,
           cudaStream_t st) {
  TRY(e->alloc(out, static_cast<size_t>(rows) * ldd));
  return f32_to_f16_2d(src, lds, *out, ldd, rows, cols, st);
}

int finalize_vit(mhmr_engine* e, cudaStream_t st) {
  const int D = e->D, N = e->N, T = e->T, Bm = e->cfg.max_batch;
  const std::string enc = e->enc;
  NEEDW(pw, enc + "patch_embed.proj.weight", static_cast<int64_t>(D) * 588);
  NEEDW(pb, enc + "patch_embed.proj.bias", D);
  NEEDW(cls, enc + "cls_token", D);
  const float* pos = e->w(enc + "pos_embed", static_cast<int64_t>(1 + N) * D);
  if (pos == nullptr) {
    set_last_error(std::string(get_last_error()) + " (pos_embed must be interpolated to the working grid [1,1+N,D])");
    return MHMR_ERR_STATE;
  }
  TRY(to_f16(e, pw, 588, D, 588, 592, &e->Wpatch, st));
  e->Wpatch32 = pw;
  TRY(e->alloc(&e->rowadd, static_cast<size_t>(N) * D));
  TRY(add_vec(pos + D, pb, e->rowadd, static_cast<int64_t>(N) * D, D, st));
  TRY(e->alloc(&e->cls_pos, D));
  TRY(add_vec(cls, pos, e->cls_pos, D, D, st));

  const size_t M = static_cast<size_t>(Bm) * T;
  TRY(e->alloc(&e->A16, static_cast<size_t>(Bm) * N * 592));
  TRY(e->alloc(&e->X, M * D));
  TRY(e->alloc(&e->Xn16, M * D));
  TRY(e->alloc(&e->QKV16, M * 3 * D));
  // one attention-output buffer per layer when the refinement pass needs the rows of every layer afterwards
  const size_t o_layers = e->cfg.refine_central ? static_cast<size_t>(e->depth) : 1;
  TRY(e->alloc(&e->O16, o_layers * M * D));
  TRY(e->alloc(&e->H16, M * 4 * D));
  {
    const char* lf = std::getenv("MHMR_LN_FOLD");
    e->ln_fold = !(lf != nullptr && lf[0] == '0');
  }
  e->ln_slots = gemm_stat_slots(D, pick_bn(D));
  if (e->ln_fold) {
    TRY(e->alloc(&e->ln_stats, M * e->ln_slots));
    TRY(e->alloc(&e->Xlo, M * D));
  }

  GemmEpi ep;
  ep.rowadd = e->rowadd; ep.out = e->X; ep.ldo = D; ep.rows_in = N; ep.rows_out = T; ep.row_off = 1;
  TRY(gemm_plan_init(&e->patch_plan, e->A16, 592, e->Wpatch, 592, Bm * N, D, 588, EPI_ROWADD_F32, ep, pick_bn(D)));

  e->vit.resize(e->depth);
  for (int l = 0; l < e->depth; ++l) {
    VitLayer& L = e->vit[l];
    const std::string b = enc + "blocks." + std::to_string(l) + ".";
    NEEDW(n1g, b + "norm1.weight", D) NEEDW(n1b, b + "norm1.bias", D)
    NEEDW(n2g, b + "norm2.weight", D) NEEDW(n2b, b + "norm2.bias", D)
    NEEDW(wqkv, b + "attn.qkv.weight", 3ll * D * D) NEEDW(bqkv, b + "attn.qkv.bias", 3 * D)
    NEEDW(wproj, b + "attn.proj.weight", static_cast<int64_t>(D) * D) NEEDW(bproj, b + "attn.proj.bias", D)
    NEEDW(ls1, b + "ls1.gamma", D) NEEDW(ls2, b + "ls2.gamma", D)
    NEEDW(wfc1, b + "mlp.fc1.weight", 4ll * D * D) NEEDW(bfc1, b + "mlp.fc1.bias", 4 * D)
    NEEDW(wfc2, b + "mlp.fc2.weight", 4ll * D * D) NEEDW(bfc2, b + "mlp.fc2.bias", D)
    L.ln1_g = n1g; L.ln1_b = n1b; L.ln2_g = n2g; L.ln2_b = n2b;
    L.Wproj32 = wproj; L.Wfc1_32 = wfc1; L.Wfc2_32 = wfc2;
    L.O16 = e->O16 + (e->cfg.refine_central ? static_cast<size_t>(l) * M * D : 0);
    L.bqkv = bqkv; L.bproj = bproj; L.ls1 = ls1; L.bfc1 = bfc1; L.bfc2 = bfc2; L.ls2 = ls2;
    TRY(to_f16(e, wproj, D, D, D, D, &L.Wproj, st));
    TRY(to_f16(e, wfc2, 4 * D, D, 4 * D, 4 * D, &L.Wfc2, st));
    GemmEpi a; a.out = e->QKV16; a.ldo = 3 * D;
    GemmEpi p; p.bias = bproj; p.gamma = ls1; p.out = e->X; p.ldo = D;
    GemmEpi f1; f1.out = e->H16; f1.ldo = 4 * D;
    GemmEpi f2; f2.bias = bfc2; f2.gamma = ls2; f2.out = e->X; f2.ldo = D;
    int epi_qkv = EPI_BIAS_F16, epi_fc1 = EPI_BIAS_GELU_F16, epi_proj = EPI_LS_RESID_F32, epi_fc2 = EPI_LS_RESID_F32;
    if (e->ln_fold) {
      // qkv / fc1 read the hi plane of the residual stream that the previous proj / fc2 epilogue (layer 0:
      // split_rowstats) left in Xn16, and normalise in their epilogue from the row statistics
      TRY(e->alloc(&L.Wqkv, static_cast<size_t>(3) * D * D));
      TRY(e->alloc(&L.bqkv_f, 3 * D));
      TRY(fold_ln_linear(wqkv, bqkv, n1g, n1b, L.Wqkv, L.bqkv_f, 3 * D, D, st));
      TRY(e->alloc(&L.Wfc1, static_cast<size_t>(4) * D * D));
      TRY(e->alloc(&L.bfc1_f, 4 * D));
      TRY(fold_ln_linear(wfc1, bfc1, n2g, n2b, L.Wfc1, L.bfc1_f, 4 * D, D, st));
      a.bias = L.bqkv_f; a.stats = e->ln_stats; a.stat_slots = e->ln_slots;
      f1.bias = L.bfc1_f; f1.stats = e->ln_stats; f1.stat_slots = e->ln_slots;
      epi_qkv = EPI_LN_BIAS_F16;
      epi_fc1 = EPI_LN_GELU_F16;
      // the residual stream lives in (Xn16, Xlo) = (hi, lo); hi is the A operand of qkv / fc1
      p.out = nullptr; p.x16 = e->Xn16; p.xlo = e->Xlo; p.ldx16 = D; p.stats = e->ln_stats; p.stat_slots = e->ln_slots;
      f2.out = nullptr; f2.x16 = e->Xn16; f2.xlo = e->Xlo; f2.ldx16 = D; f2.stats = e->ln_stats; f2.stat_slots = e->ln_slots;
      epi_proj = epi_fc2 = EPI_LS_RESID_SPLIT;
    } else {
      TRY(to_f16(e, wqkv, D, 3 * D, D, D, &L.Wqkv, st));
      TRY(to_f16(e, wfc1, D, 4 * D, D, D, &L.Wfc1, st));
      a.bias = bqkv;
      f1.bias = bfc1;
    }
    TRY(gemm_plan_init(&L.qkv, e->Xn16, D, L.Wqkv, D, static_cast<int>(M), 3 * D, D, epi_qkv, a, pick_bn(3 * D)));
    TRY(gemm_plan_init(&L.proj, L.O16, D, L.Wproj, D, static_cast<int>(M), D, D, epi_proj, p, pick_bn(D)));
    TRY(gemm_plan_init(&L.fc1, e->Xn16, D, L.Wfc1, D, static_cast<int>(M), 4 * D, D, epi_fc1, f1, pick_bn(4 * D)));
    TRY(gemm_plan_init(&L.fc2, e->H16, 4 * D, L.Wfc2, 4 * D, static_cast<int>(M), D, 4 * D, epi_fc2, f2, pick_bn(D)));
  }
  GETW(e->norm_g, enc + "norm.weight", D)
  GETW(e->norm_b, enc + "norm.bias", D)
  return MHMR_OK;
}

// workspaces of the central-stream refinement for `rows` token rows
int alloc_refine(mhmr_engine* e, int rows, cudaStream_t st) {
  const int D = e->D;
  e->r_rows = rows;
  TRY(e->alloc(&e->r_rowidx, rows));
  TRY(e->alloc(&e->r_patch, static_cast<size_t>(rows) * 592));
  TRY(e->alloc(&e->r_x, static_cast<size_t>(rows) * D));
  TRY(e->alloc(&e->r_h, static_cast<size_t>(rows) * 4 * D));
  TRY(e->alloc(&e->r_term, static_cast<size_t>(e->depth) * rows * D));
  TRY(e->alloc(&e->r_barrier, 4));
  std::vector<RefineLayer> rl(e->depth);
  for (int l = 0; l < e->depth; ++l) {
    const VitLayer& L = e->vit[l];
    rl[l] = RefineLayer{L.O16, L.Wproj32, L.bproj, L.ls1, L.ln2_g, L.ln2_b, L.Wfc1_32, L.bfc1, L.Wfc2_32, L.bfc2, L.ls2};
  }
  TRY(e->alloc(&e->r_layers, rl.size()));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->r_layers, rl.data(), rl.size() * sizeof(RefineLayer), cudaMemcpyHostToDevice, st));
  MHMR_CUDA_CHECK(cudaStreamSynchronize(st));  // rl lives on this stack frame
  return MHMR_OK;
}

// detection and decoder workspaces of both heads; the per-person ones are sized by the decoder and MLP widths
int alloc_head_workspaces(mhmr_engine* e, cudaStream_t st) {
  const int D = e->D, Bm = e->cfg.max_batch, Pm = e->cfg.max_persons, inner = e->cfg.xat_num_heads * 32;
  const size_t BN = static_cast<size_t>(Bm) * e->N;
  TRY(e->alloc(&e->z32, BN * D));
  TRY(e->alloc(&e->ctx16, BN * e->Cp));
  TRY(e->alloc(&e->scores_raw, BN));
  TRY(e->alloc(&e->KV32, BN * e->nkv));
  TRY(e->alloc(&e->Kinv, static_cast<size_t>(Bm) * 9));
  TRY(e->alloc(&e->count, 4));
  TRY(e->alloc(&e->img_off, static_cast<size_t>(Bm) + 1));
  TRY(e->alloc(&e->one, 4));
  const int one_h = 1;
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->one, &one_h, sizeof(int), cudaMemcpyHostToDevice, st));
  MHMR_CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&e->h_count), sizeof(int)));
  TRY(e->alloc(&e->zc, static_cast<size_t>(Pm) * D));
  TRY(e->alloc(&e->xa, static_cast<size_t>(Pm) * e->dec_dim));
  TRY(e->alloc(&e->qkvp, static_cast<size_t>(Pm) * 3 * inner));
  TRY(e->alloc(&e->att, static_cast<size_t>(Pm) * inner));
  TRY(e->alloc(&e->qca, static_cast<size_t>(Pm) * inner));
  TRY(e->alloc(&e->ffh, static_cast<size_t>(Pm) * e->dec_mlp));
  return MHMR_OK;
}

// detection MLP under `p`: its hidden Linear runs as a GEMM on the fp16 context, its output row in rowdot_sigmoid
int load_detector(mhmr_engine* e, const std::string& p, cudaStream_t st) {
  const int D = e->D, BN = e->cfg.max_batch * e->N;
  NEEDW(c0w, p + "0.weight", static_cast<int64_t>(D) * D) NEEDW(c0b, p + "0.bias", D)
  GETW(e->cls2_w, p + "2.weight", D) GETW(e->cls2_b, p + "2.bias", 1)
  TRY(to_f16(e, c0w, D, D, D, D, &e->Wcls0, st));
  GemmEpi ce; ce.bias = c0b; ce.out = e->H16; ce.ldo = D;
  return gemm_plan_init(&e->cls0_plan, e->ctx16, e->Cp, e->Wcls0, D, BN, D, D, EPI_BIAS_RELU_F16, ce, pick_bn(D));
}

// HPH layer under `p` (PreNorm self-attention, cross-attention, feed-forward).  The cross-attention's to_kv weight
// [2 inner, kv_cols] goes to *to_kv: each head packs the keys / values of all layers into one GEMM its own way.
int load_hph_layer(mhmr_engine* e, const std::string& p, int kv_cols, HphLayer& L, const float** to_kv) {
  const int dim = e->dec_dim, mlp = e->dec_mlp, inner = e->cfg.xat_num_heads * 32;
  GETW(L.ln0_g, p + "0.norm.weight", dim) GETW(L.ln0_b, p + "0.norm.bias", dim)
  GETW(L.Wqkv, p + "0.fn.to_qkv.weight", 3ll * inner * dim)
  GETW(L.Wsa_out, p + "0.fn.to_out.0.weight", static_cast<int64_t>(dim) * inner)
  GETW(L.bsa_out, p + "0.fn.to_out.0.bias", dim)
  GETW(L.ln1_g, p + "1.norm.weight", dim) GETW(L.ln1_b, p + "1.norm.bias", dim)
  GETW(*to_kv, p + "1.fn.to_kv.weight", 2ll * inner * kv_cols)
  GETW(L.Wq, p + "1.fn.to_q.weight", static_cast<int64_t>(inner) * dim)
  GETW(L.Wca_out, p + "1.fn.to_out.0.weight", static_cast<int64_t>(dim) * inner)
  GETW(L.bca_out, p + "1.fn.to_out.0.bias", dim)
  GETW(L.ln2_g, p + "2.norm.weight", dim) GETW(L.ln2_b, p + "2.norm.bias", dim)
  GETW(L.Wff0, p + "2.fn.net.0.weight", static_cast<int64_t>(mlp) * dim) GETW(L.bff0, p + "2.fn.net.0.bias", mlp)
  GETW(L.Wff3, p + "2.fn.net.3.weight", static_cast<int64_t>(dim) * mlp) GETW(L.bff3, p + "2.fn.net.3.bias", dim)
  return MHMR_OK;
}

int finalize_head(mhmr_engine* e, cudaStream_t st) {
  const int D = e->D, N = e->N, Bm = e->cfg.max_batch, Pm = e->cfg.max_persons, C = e->C, Cp = e->Cp,
            Cq = e->Cq, nb = e->cfg.num_betas, depth = e->cfg.xat_depth, inner = e->cfg.xat_num_heads * 32;
  const int res = e->res;
  const size_t BN = static_cast<size_t>(Bm) * N;
  TRY(alloc_head_workspaces(e, st));
  TRY(load_detector(e, "mlp_classif.", st));
  SmplxHeadWeights& hw = e->smplx_w;
  GETW(hw.off0_w, "mlp_offset.0.weight", static_cast<int64_t>(D) * D) GETW(hw.off0_b, "mlp_offset.0.bias", D)
  GETW(hw.off2_w, "mlp_offset.2.weight", 2ll * D) GETW(hw.off2_b, "mlp_offset.2.bias", 2)

  // HPH
  const std::string h = "x_attention_head.";
  const int64_t rC = static_cast<int64_t>(res) * C;
  GETW(hw.cq_x, h + "cross_queries_x", rC) GETW(hw.cq_y, h + "cross_queries_y", rC)
  GETW(hw.cv_x, h + "cross_values_x", rC) GETW(hw.cv_y, h + "cross_values_y", rC)
  GETW(hw.freq_bands, "camera.freq_bands", 16)
  const int token_dim = 318 + nb + 3 + C;
  const std::string t = h + "transformer.";
  NEEDW(tew, t + "to_token_embedding.weight", static_cast<int64_t>(kHphDim) * token_dim)
  NEEDW(teb, t + "to_token_embedding.bias", kHphDim)
  NEEDW(pe, t + "pos_embedding", kHphDim)
  NEEDW(ipose, h + "init_body_pose", 318) NEEDW(ibetas, h + "init_betas", nb) NEEDW(icam, h + "init_cam", 3)
  TRY(e->alloc(&e->Wte_q, static_cast<size_t>(kHphDim) * Cq));
  TRY(repack_f32(tew, token_dim, 0, e->Wte_q, Cq, 0, kHphDim, C, true, st));
  // te_const = W_te[:, C:] . [init_pose | init_betas | init_cam] + bias + pos_embedding
  const int ni = 318 + nb + 3, nip = (ni + 3) & ~3;
  float *Wte_i = nullptr, *init_vec = nullptr, *tmpb = nullptr;
  TRY(e->alloc(&Wte_i, static_cast<size_t>(kHphDim) * nip));
  TRY(repack_f32(tew, token_dim, C, Wte_i, nip, 0, kHphDim, ni, true, st));
  TRY(e->alloc(&init_vec, nip));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(init_vec, ipose, 318 * 4, cudaMemcpyDeviceToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(init_vec + 318, ibetas, nb * 4, cudaMemcpyDeviceToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(init_vec + 318 + nb, icam, 3 * 4, cudaMemcpyDeviceToDevice, st));
  TRY(e->alloc(&tmpb, kHphDim));
  TRY(add_vec(teb, pe, tmpb, kHphDim, kHphDim, st));
  TRY(e->alloc(&e->te_const, kHphDim));
  TRY(skinny_linear(init_vec, nip, e->one, 1, ni, Wte_i, nip, tmpb, kHphDim, nullptr, nullptr, 0.f, 0, nullptr, 0,
                    e->te_const, kHphDim, st));

  e->hph.resize(depth);
  TRY(e->alloc(&e->Wkv32, static_cast<size_t>(e->nkv) * Cq));
  for (int l = 0; l < depth; ++l) {
    const float* kvw = nullptr;
    TRY(load_hph_layer(e, t + "transformer.layers." + std::to_string(l) + ".", C, e->hph[l], &kvw));
    TRY(repack_f32(kvw, C, 0, e->Wkv32 + static_cast<size_t>(l) * 2 * inner * Cq, Cq, 0, 2 * inner, C, true, st));
  }
  TRY(e->alloc(&e->Wkv16, static_cast<size_t>(e->nkv) * Cp));
  TRY(f32_to_f16_2d(e->Wkv32, Cq, e->Wkv16, Cp, e->nkv, C, st));  // cols >= C stay zero
  GemmEpi ke; ke.out = e->KV32; ke.ldo = e->nkv;
  TRY(gemm_plan_init(&e->kv_plan, e->ctx16, Cp, e->Wkv16, Cp, static_cast<int>(BN), e->nkv, Cp, EPI_BIAS_F32, ke, pick_bn(e->nkv)));

  // decoders stacked: [pose6 318 | betas nb | cam 3 | expression 10], bias + init (model.py:571-575)
  e->ndec = 318 + nb + 3 + 10;
  NEEDW(dpw, h + "decpose.weight", 318ll * kHphDim) NEEDW(dpb, h + "decpose.bias", 318)
  NEEDW(dsw, h + "decshape.weight", static_cast<int64_t>(nb) * kHphDim) NEEDW(dsb, h + "decshape.bias", nb)
  NEEDW(dcw, h + "deccam.weight", 3ll * kHphDim) NEEDW(dcb, h + "deccam.bias", 3)
  NEEDW(dew, h + "decexpression.weight", 10ll * kHphDim) NEEDW(deb, h + "decexpression.bias", 10)
  TRY(e->alloc(&e->Wdec, static_cast<size_t>(e->ndec) * kHphDim));
  TRY(e->alloc(&e->bdec, e->ndec));
  const size_t rowb = kHphDim * sizeof(float);
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->Wdec, dpw, 318 * rowb, cudaMemcpyDeviceToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->Wdec + 318 * kHphDim, dsw, nb * rowb, cudaMemcpyDeviceToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->Wdec + (318 + nb) * kHphDim, dcw, 3 * rowb, cudaMemcpyDeviceToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->Wdec + (321 + nb) * kHphDim, dew, 10 * rowb, cudaMemcpyDeviceToDevice, st));
  TRY(add_vec(dpb, ipose, e->bdec, 318, 318, st));
  TRY(add_vec(dsb, ibetas, e->bdec + 318, nb, nb, st));
  TRY(add_vec(dcb, icam, e->bdec + 318 + nb, 3, 3, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->bdec + 321 + nb, deb, 10 * 4, cudaMemcpyDeviceToDevice, st));  // init_expression = 0

  // per-person buffers
  TRY(e->alloc(&e->query, static_cast<size_t>(Pm) * Cq));
  TRY(e->alloc(&e->vals, static_cast<size_t>(Pm) * Cq));
  TRY(e->alloc(&e->dKV, static_cast<size_t>(Pm) * e->nkv));
  TRY(e->alloc(&e->offh, static_cast<size_t>(Pm) * D));
  TRY(e->alloc(&e->dec, static_cast<size_t>(Pm) * e->ndec));
  TRY(e->alloc(&e->K_det, static_cast<size_t>(Pm) * 9));
  if (e->cfg.refine_central) TRY(alloc_refine(e, Pm, st));
  return MHMR_OK;
}

int finalize_body(mhmr_engine* e, cudaStream_t st) {
  const int V = e->cfg.num_verts, nb = e->cfg.num_betas;
  NEEDW(vt, "smplx.v_template", 3ll * V)
  NEEDW(sd, "smplx.shapedirs", 3ll * V * nb)
  NEEDW(ed, "smplx.expr_dirs", 30ll * V)
  NEEDW(pd, "smplx.posedirs", 486ll * 3 * V)
  NEEDW(jr, "smplx.J_regressor", 55ll * V)
  NEEDW(lw, "smplx.lbs_weights", 55ll * V)
  NEEDW(bary, "smplx.lmk_bary_coords", 51 * 3)
  const int* parents = e->tab("smplx.parents", 55);
  const int* extra = e->tab("smplx.extra_joints_idxs", 21);
  const int* tri = e->tab("smplx.lmk_tri", 51 * 3);
  if (!parents || !extra || !tri) return MHMR_ERR_STATE;
  // with the backward scratch of mhmr_smplx_backward
  return body_build(&e->body, 55, V, nb, 10, e->cfg.person_center_idx, e->cfg.max_persons, vt, sd, ed, pd, jr, lw,
                    parents, extra, tri, bary, st);
}

// Anny head (multi_hmr_anny/multi_hmr.py:41-95, encoder.py:16-31, hph.py): weights under the checkpoint's own keys.
int finalize_anny(mhmr_engine* e, cudaStream_t st) {
  const int D = e->D, N = e->N, Bm = e->cfg.max_batch, Pm = e->cfg.max_persons, nb = e->cfg.num_betas;
  const int dim = e->dec_dim, J = e->cfg.num_joints, depth = e->cfg.xat_depth;
  const int inner = e->cfg.xat_num_heads * 32, J6 = 6 * J, J6p = (J6 + 3) & ~3;
  const size_t BN = static_cast<size_t>(Bm) * N;
  TRY(alloc_head_workspaces(e, st));
  TRY(e->alloc(&e->K_use, static_cast<size_t>(Bm) * 9));
  TRY(e->alloc(&e->det_score, Pm));
  TRY(e->alloc(&e->anny_ints, 2));

  // detection: mlp_det hidden layer as a GEMM on the normed fp16 features (encoder.py:26,59)
  TRY(load_detector(e, "encoder.mlp_det.", st));
  // field of view from the cls token (encoder.py:29-31,50)
  AnnyHeadWeights& hw = e->anny_w;
  GETW(hw.fov0_w, "encoder.mlp_fov_unique.0.weight", static_cast<int64_t>(D) * D)
  GETW(hw.fov0_b, "encoder.mlp_fov_unique.0.bias", D)
  GETW(hw.fov2_w, "encoder.mlp_fov_unique.2.weight", D) GETW(hw.fov2_b, "encoder.mlp_fov_unique.2.bias", 1)
  GETW(hw.fov_max, "encoder.fov_max", 1)
  TRY(e->alloc(&e->cls_x, static_cast<size_t>(Bm) * D));
  TRY(e->alloc(&e->cls_h, static_cast<size_t>(Bm) * D));

  // decoder tokens of every cell: dec_to_token(feat) + dec_pos_emb (multi_hmr.py:127-128), fp16 GEMM output
  GETW(hw.dt_w, "dec_to_token.weight", static_cast<int64_t>(dim) * D) GETW(hw.dt_b, "dec_to_token.bias", dim)
  GETW(hw.dec_pos_emb, "dec_pos_emb", static_cast<int64_t>(N) * dim)
  TRY(to_f16(e, hw.dt_w, D, dim, D, D, &e->Wdt16, st));
  TRY(e->alloc(&e->dt_rowadd, static_cast<size_t>(N) * dim));
  TRY(add_vec(hw.dec_pos_emb, hw.dt_b, e->dt_rowadd, static_cast<int64_t>(N) * dim, dim, st));
  TRY(e->alloc(&e->dec16, BN * dim));
  GemmEpi te; te.rowadd = e->dt_rowadd; te.rows_in = N; te.out = e->dec16; te.ldo = dim;
  TRY(gemm_plan_init(&e->dt_plan, e->ctx16, e->Cp, e->Wdt16, D, static_cast<int>(BN), dim, D, EPI_ROWADD_F16, te, pick_bn(dim)));

  // HPH layers; the keys / values of all of them come from ONE GEMM over the tokens (to_kv, hph.py:88,99)
  e->hph.resize(depth);
  TRY(e->alloc(&e->Wkv16, static_cast<size_t>(e->nkv) * dim));
  for (int l = 0; l < depth; ++l) {
    const float* kvw = nullptr;
    TRY(load_hph_layer(e, "decoder.transformer.layers." + std::to_string(l) + ".", dim, e->hph[l], &kvw));
    TRY(f32_to_f16_2d(kvw, dim, e->Wkv16 + static_cast<size_t>(l) * 2 * inner * dim, dim, 2 * inner, dim, st));
  }
  GemmEpi ke; ke.out = e->KV32; ke.ldo = e->nkv;
  TRY(gemm_plan_init(&e->kv_plan, e->dec16, dim, e->Wkv16, dim, static_cast<int>(BN), e->nkv, dim, EPI_BIAS_F32, ke, pick_bn(e->nkv)));

  // regressors (multi_hmr.py:59-66): the four first Linears stacked; mlp_pose's init_body_pose columns folded into
  // its bias, and init_body_pose added to the bias of its second Linear (:157)
  NEEDW(o0w, "mlp_offset.0.weight", static_cast<int64_t>(dim) * dim) NEEDW(o0b, "mlp_offset.0.bias", dim)
  GETW(hw.off2_w, "mlp_offset.2.weight", 2ll * dim) GETW(hw.off2_b, "mlp_offset.2.bias", 2)
  NEEDW(d0w, "mlp_dist.0.weight", static_cast<int64_t>(dim) * dim) NEEDW(d0b, "mlp_dist.0.bias", dim)
  GETW(hw.dist2_w, "mlp_dist.2.weight", dim) GETW(hw.dist2_b, "mlp_dist.2.bias", 1)
  NEEDW(s0w, "mlp_shape.0.weight", static_cast<int64_t>(dim) * dim) NEEDW(s0b, "mlp_shape.0.bias", dim)
  GETW(hw.shape2_w, "mlp_shape.2.weight", static_cast<int64_t>(nb) * dim) GETW(hw.shape2_b, "mlp_shape.2.bias", nb)
  NEEDW(p0w, "mlp_pose.0.weight", static_cast<int64_t>(dim) * (dim + J6)) NEEDW(p0b, "mlp_pose.0.bias", dim)
  GETW(hw.pose2_w, "mlp_pose.2.weight", static_cast<int64_t>(J6) * dim) NEEDW(p2b, "mlp_pose.2.bias", J6)
  GETW(hw.useful_rotmat, "useful_rotmat", J) NEEDW(init, "init_body_pose", J6)
  TRY(e->alloc(&e->W1, static_cast<size_t>(4) * dim * dim));
  TRY(e->alloc(&e->b1, static_cast<size_t>(4) * dim));
  const size_t blk = static_cast<size_t>(dim) * dim;
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->W1, o0w, blk * 4, cudaMemcpyDeviceToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->W1 + blk, d0w, blk * 4, cudaMemcpyDeviceToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->W1 + 2 * blk, s0w, blk * 4, cudaMemcpyDeviceToDevice, st));
  TRY(repack_f32(p0w, dim + J6, 0, e->W1 + 3 * blk, dim, 0, dim, dim, false, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->b1, o0b, dim * 4, cudaMemcpyDeviceToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->b1 + dim, d0b, dim * 4, cudaMemcpyDeviceToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->b1 + 2 * dim, s0b, dim * 4, cudaMemcpyDeviceToDevice, st));
  float *Wpi = nullptr, *init_pad = nullptr;
  TRY(e->alloc(&Wpi, static_cast<size_t>(dim) * J6p));
  TRY(repack_f32(p0w, dim + J6, dim, Wpi, J6p, 0, dim, J6, true, st));
  TRY(e->alloc(&init_pad, J6p));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(init_pad, init, J6 * 4, cudaMemcpyDeviceToDevice, st));
  TRY(skinny_linear(init_pad, J6p, e->one, 1, J6, Wpi, J6p, p0b, dim, nullptr, nullptr, 0.f, 0, nullptr, 0,
                    e->b1 + 3 * dim, dim, st));
  TRY(e->alloc(&e->b_pose2, J6));
  TRY(add_vec(p2b, init, e->b_pose2, J6, J6, st));

  // per-person buffers
  TRY(e->alloc(&e->offh, static_cast<size_t>(Pm) * 4 * dim));
  TRY(e->alloc(&e->dec, static_cast<size_t>(Pm) * J6p));
  if (e->cfg.refine_central) TRY(alloc_refine(e, Pm + Bm, st));
  return MHMR_OK;
}

// image of a forward: normalised fp32 NCHW (the reference's Model.forward input) or uint8 NHWC + the [3][256]
// normalize_rgb table (fused loader, SURVEY.md §8f row 1)
struct ImgSrc {
  const float* f32 = nullptr;
  const uint8_t* u8 = nullptr;
  const float* lut = nullptr;
};

struct ProfScope {
  mhmr_engine* e; int cat; cudaStream_t st; cudaEvent_t a{};
  ProfScope(mhmr_engine* e_, int cat_, cudaStream_t st_) : e(e_), cat(cat_), st(st_) {
    if (e->profiling) { a = e->next_event(); cudaEventRecord(a, st); }
  }
  ~ProfScope() {
    if (e->profiling) { cudaEvent_t b = e->next_event(); cudaEventRecord(b, st); e->prof.push_back({cat, a, b}); }
  }
};

#define LAUNCH(cat, expr)               \
  do {                                  \
    ProfScope ps_(e, cat, st);          \
    TRY(expr);                          \
    ++e->launches;                      \
  } while (0)

int run_plan(mhmr_engine* e, int cat, GemmPlan& plan, int M, cudaStream_t st) {
  ProfScope ps_(e, cat, st);
  TRY(gemm_plan_run_rows(&plan, M, st));  // plans are built for the maximum batch
  ++e->launches;
  return MHMR_OK;
}

// The bulk pass.  With stream_out (stage entry mhmr_op_vit_stream) it stops after the first `layers` blocks and writes
// the residual stream [B, T, D] fp32 instead of the final norm; the product path runs all blocks.
int vit_forward(mhmr_engine* e, const ImgSrc& x, int B, float* z_out, cudaStream_t st, int layers = -1,
                float* stream_out = nullptr) {
  const int D = e->D, N = e->N, T = e->T, M = B * T;
  if (layers < 0) layers = e->depth;
  if (x.u8 != nullptr) {
    LAUNCH(MHMR_CAT_MISC, im2col_u8_patch14(x.u8, x.lut, e->A16, B, e->cfg.img_size, 592, st));
  } else {
    LAUNCH(MHMR_CAT_MISC, im2col_patch14(x.f32, e->A16, B, e->cfg.img_size, 592, st));
  }
  LAUNCH(MHMR_CAT_MISC, cls_rows(e->X, e->cls_pos, B, T, D, st));
  TRY(run_plan(e, MHMR_CAT_GEMM_OTHER, e->patch_plan, B * N, st));
  // the folded chain enters as the two-term stream (hi, lo) + row statistics
  if (e->ln_fold)
    LAUNCH(MHMR_CAT_LAYERNORM, split_rowstats(e->X, e->Xn16, e->Xlo, D, e->ln_stats, e->ln_slots, M, D, st));
  for (int l = 0; l < layers; ++l) {
    VitLayer& L = e->vit[l];
    // norm1 / norm2: folded into qkv / fc1 (statistics + raw fp16 rows come from the previous epilogue), or kernels
    if (!e->ln_fold)
      LAUNCH(MHMR_CAT_LAYERNORM, layernorm(e->X, L.ln1_g, L.ln1_b, e->Xn16, D, nullptr, 0, M, D, 1e-6f, 0, 0, st));
    TRY(run_plan(e, MHMR_CAT_GEMM_QKV, L.qkv, M, st));
    LAUNCH(MHMR_CAT_ATTENTION, attention_forward(e->QKV16, 3 * D, L.O16, D, B, T, D, st));
    TRY(run_plan(e, MHMR_CAT_GEMM_PROJ, L.proj, M, st));
    if (!e->ln_fold)
      LAUNCH(MHMR_CAT_LAYERNORM, layernorm(e->X, L.ln2_g, L.ln2_b, e->Xn16, D, nullptr, 0, M, D, 1e-6f, 0, 0, st));
    TRY(run_plan(e, MHMR_CAT_GEMM_FC1, L.fc1, M, st));
    TRY(run_plan(e, MHMR_CAT_GEMM_FC2, L.fc2, M, st));
  }
  if (stream_out != nullptr) {
    const int64_t n = static_cast<int64_t>(M) * D;
    if (e->ln_fold) {
      LAUNCH(MHMR_CAT_MISC, merge_split(e->Xn16, e->Xlo, stream_out, n, st));
    } else {
      MHMR_CUDA_CHECK(cudaMemcpyAsync(stream_out, e->X, n * 4, cudaMemcpyDeviceToDevice, st));
    }
    return MHMR_OK;
  }
  // final norm, cls dropped: fp32 features (head query side, optional user copy) + fp16 context columns
  if (e->ln_fold) {
    LAUNCH(MHMR_CAT_LAYERNORM,
           layernorm_split(e->Xn16, e->Xlo, e->norm_g, e->norm_b, e->ctx16, e->Cp, e->z32, D, M, D, 1e-6f, T, 1, st));
  } else {
    LAUNCH(MHMR_CAT_LAYERNORM, layernorm(e->X, e->norm_g, e->norm_b, e->ctx16, e->Cp, e->z32, D, M, D, 1e-6f, T, 1, st));
  }
  if (z_out != nullptr)
    MHMR_CUDA_CHECK(cudaMemcpyAsync(z_out, e->z32, static_cast<size_t>(B) * N * D * 4, cudaMemcpyDeviceToDevice, st));
  return MHMR_OK;
}

// Central-stream refinement (DESIGN.md §3).  The bulk pass computes every token with fp16 tensor-core operands;
// what the per-person outputs are sensitive to is the residual stream of the DETECTED tokens themselves (their
// own patch embedding and their own MLP / projection branches: 92 % of the feature error variance,
// tools/precision_study.py).  Those few rows are recomputed here in fp32 with the fp32 master weights:
//   x = patch-embed(pixels) + pos;  per block: x += ls1 * (Wproj . O16[row] + b);  x += ls2 * MLP(LN2(x))
// where O16[row] is the attention output of the bulk pass for that token (kept per layer).  The final norm is
// applied by person_gather.  Same arithmetic as dinov2 Block.forward (reached from blocks/dinov2.py:25).  Four
// launches: patches / row indices, patch embedding, every projection term at once, the MLP chain of all blocks in one
// persistent cooperative kernel (refine.cu).
// With n_cls > 0 the cls rows of images 0..n_cls-1 are refined too, ahead of the persons (r_x rows [0, n_cls)), and
// `rows` receives the device-side row count.
int refine_streams(mhmr_engine* e, const ImgSrc& x, const int* det_b, const int* det_y, const int* det_x,
                   const int* count, int n_cls, int* rows, cudaStream_t st) {
  const int D = e->D, Pm = e->cfg.max_persons, Rm = e->r_rows;
  LAUNCH(MHMR_CAT_REFINE, refine_prepare(x.f32, x.u8, x.lut, e->cfg.img_size, e->rowadd, D, det_b, det_y, det_x, count, Pm, e->res,
                                         n_cls, e->cls_pos, n_cls > 0 ? rows : nullptr, e->r_rowidx, e->r_patch, 592, e->r_x, st));
  const int* rc = n_cls > 0 ? rows : count;
  LAUNCH(MHMR_CAT_REFINE, skinny_linear(e->r_patch, 592, rc, Rm, 588, e->Wpatch32, 588, nullptr, D, nullptr, nullptr, 0.f, 0,
                                        e->r_x, D, e->r_x, D, st));
  LAUNCH(MHMR_CAT_REFINE, refine_proj_terms(e->r_layers, e->depth, e->r_rowidx, rc, D, Rm, e->r_term, st));
  LAUNCH(MHMR_CAT_REFINE, refine_mlp_chain(e->r_layers, e->depth, rc, D, Rm, e->r_term, e->r_x, e->r_h, e->r_barrier, st));
  return MHMR_OK;
}

// Detection: the hidden layer as a GEMM over every cell, the score row + sigmoid (`clamp`: clamped sigmoid, SMPL-X;
// `logits`: optional copy of the pre-sigmoid scores), then the forced persons or NMS.  The true count (may exceed max_persons: reported as an error
// by mhmr_sync_count, which reads the pinned host copy) goes to count_true, the count clamped to max_persons, which the
// per-person kernels iterate over, to e->count + 2.
int detect(mhmr_engine* e, int B, float det_thresh, int nms, const int64_t* forced_idx, int forced_P, bool clamp,
           float* logits, float* scores_map, int* det_idx, float* det_score, int* count_true, cudaStream_t st) {
  const int D = e->D, res = e->res, Pm = e->cfg.max_persons, BN = B * e->N;
  int* det_b = det_idx; int* det_y = det_idx + Pm; int* det_x = det_idx + 2 * Pm;
  int* count = e->count + 2;
  TRY(run_plan(e, MHMR_CAT_GEMM_OTHER, e->cls0_plan, BN, st));
  LAUNCH(MHMR_CAT_HEAD, rowdot_sigmoid(e->H16, D, e->cls2_w, e->cls2_b, e->scores_raw, logits, clamp, BN, D, st));
  if (forced_idx != nullptr) {
    LAUNCH(MHMR_CAT_HEAD, forced_detections(e->scores_raw, scores_map, B, res, forced_idx, forced_P, det_b, det_y, det_x,
                                            det_score, count_true, count, e->img_off, st));
  } else {
    LAUNCH(MHMR_CAT_HEAD, nms_compact(e->scores_raw, scores_map, B, res, nms, det_thresh, Pm, det_b, det_y, det_x,
                                      det_score, count_true, count, e->img_off, st));
  }
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->h_count, count_true, sizeof(int), cudaMemcpyDeviceToHost, st));
  return MHMR_OK;
}

// HPH layers on the person tokens e->xa (cross_attn_transformer.py / hph.py): PreNorm self-attention among the persons
// of one image, cross-attention to the keys / values of every cell (e->KV32), feed-forward
int hph_decoder(mhmr_engine* e, const int* det_b, const int* count, cudaStream_t st) {
  const int dim = e->dec_dim, mlp = e->dec_mlp, Pm = e->cfg.max_persons, N = e->N;
  const int heads = e->cfg.xat_num_heads, inner = heads * 32;
  for (int l = 0; l < e->cfg.xat_depth; ++l) {
    HphLayer& L = e->hph[l];
    LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->xa, dim, count, Pm, dim, L.Wqkv, dim, nullptr, 3 * inner, L.ln0_g, L.ln0_b, 1e-5f, 0,
                                        nullptr, 0, e->qkvp, 3 * inner, st));
    LAUNCH(MHMR_CAT_HEAD, hph_self_attn(e->qkvp, 3 * inner, det_b, e->img_off, count, Pm, heads, e->att, inner, st));
    LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->att, inner, count, Pm, inner, L.Wsa_out, inner, L.bsa_out, dim, nullptr, nullptr,
                                        0.f, 0, e->xa, dim, e->xa, dim, st));
    LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->xa, dim, count, Pm, dim, L.Wq, dim, nullptr, inner, L.ln1_g, L.ln1_b, 1e-5f, 0,
                                        nullptr, 0, e->qca, inner, st));
    LAUNCH(MHMR_CAT_HEAD, hph_cross_attn(e->qca, inner, e->KV32, e->nkv, l * 2 * inner, l * 2 * inner + inner, det_b, count,
                                         Pm, heads, N, e->att, inner, st));
    LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->att, inner, count, Pm, inner, L.Wca_out, inner, L.bca_out, dim, nullptr, nullptr,
                                        0.f, 0, e->xa, dim, e->xa, dim, st));
    LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->xa, dim, count, Pm, dim, L.Wff0, dim, L.bff0, mlp, L.ln2_g, L.ln2_b, 1e-5f, 2,
                                        nullptr, 0, e->ffh, mlp, st));
    LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->ffh, mlp, count, Pm, mlp, L.Wff3, mlp, L.bff3, dim, nullptr, nullptr, 0.f, 0,
                                        e->xa, dim, e->xa, dim, st));
  }
  return MHMR_OK;
}

int head_forward(mhmr_engine* e, const ImgSrc& x, const float* K, int B, float det_thresh, int nms, const int64_t* forced_idx,
                 int forced_P, const mhmr_outputs* o, cudaStream_t st) {
  const int D = e->D, N = e->N, res = e->res, Pm = e->cfg.max_persons, Cq = e->Cq, nb = e->cfg.num_betas;
  const SmplxHeadWeights& hw = e->smplx_w;
  int* det_b = o->det_idx; int* det_y = o->det_idx + Pm; int* det_x = o->det_idx + 2 * Pm;
  int* count = e->count + 2;
  LAUNCH(MHMR_CAT_HEAD, invert_K(K, e->Kinv, B, st));
  LAUNCH(MHMR_CAT_HEAD, ctx_fourier(e->Kinv, hw.freq_bands, e->ctx16, e->Cp, B, res, D, e->Cp - D, st));
  // detection (model.py:133-158)
  TRY(detect(e, B, det_thresh, nms, forced_idx, forced_P, true, nullptr, o->scores_map, o->det_idx, o->det_score, o->count,
             st));
  // keys / values of both decoder layers for every token (to_kv, cross_attn_transformer.py:187)
  TRY(run_plan(e, MHMR_CAT_GEMM_OTHER, e->kv_plan, B * N, st));
  const float* xr = nullptr;
  if (e->cfg.refine_central) {
    TRY(refine_streams(e, x, det_b, det_y, det_x, count, 0, nullptr, st));
    xr = e->r_x;
  }
  LAUNCH(MHMR_CAT_HEAD, person_gather(e->z32, xr, e->norm_g, e->norm_b, e->Kinv, hw.freq_bands, hw.cq_x, hw.cq_y, hw.cv_x,
                                      hw.cv_y, det_b, det_y, det_x, count, Pm, res, D, e->zc, e->query, e->vals, Cq, st));
  // offset head (model.py:258)
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->zc, D, count, Pm, D, hw.off0_w, D, hw.off0_b, D, nullptr, nullptr, 0.f, 1, nullptr, 0,
                                      e->offh, D, st));
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->offh, D, count, Pm, D, hw.off2_w, D, hw.off2_b, 2, nullptr, nullptr, 0.f, 0, nullptr,
                                      0, o->offset, 2, st));
  // learned value embeddings injected at the detected cells (model.py:514-517)
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->vals, Cq, count, Pm, e->C, e->Wkv32, Cq, nullptr, e->nkv, nullptr, nullptr, 0.f, 0,
                       nullptr, 0, e->dKV, e->nkv, st));
  LAUNCH(MHMR_CAT_HEAD, kv_add_rows(e->KV32, e->nkv, e->dKV, e->nkv, det_b, det_y, det_x, count, Pm, res, st));
  // token embedding (cross_attn_transformer.py:352-357)
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->query, Cq, count, Pm, e->C, e->Wte_q, Cq, e->te_const, kHphDim, nullptr, nullptr, 0.f,
                       0, nullptr, 0, e->xa, kHphDim, st));
  TRY(hph_decoder(e, det_b, count, st));
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->xa, kHphDim, count, Pm, kHphDim, e->Wdec, kHphDim, e->bdec, e->ndec, nullptr, nullptr, 0.f,
                       0, nullptr, 0, e->dec, e->ndec, st));
  const float focal_norm = static_cast<float>(e->cfg.img_size / (2.0 * tan(30.0 * 3.14159265358979323846 / 180.0)));
  LAUNCH(MHMR_CAT_HEAD, person_post(e->dec, e->ndec, nb, o->offset, K, e->Kinv, det_b, det_y, det_x, count, Pm, focal_norm,
                     o->rotmat, o->rotvec, o->shape, o->expression, o->dist_pp, o->dist, o->loc, o->transl,
                     e->K_det, st));
  {
    ProfScope ps_(e, MHMR_CAT_SMPLX, st);
    TRY(smplx_forward(e->body.bm, o->rotvec, o->shape, o->expression, o->transl, e->K_det, count, Pm, e->body.ws,
                      o->v3d, o->v2d, o->j3d, o->j2d, o->transl_pelvis, st));
  }
  e->launches += 3;
  return MHMR_OK;
}

// Multi_HMR.forward (multi_hmr_anny/multi_hmr.py:98-175) up to the body model's inputs.  K == nullptr: the regressed
// intrinsics are used.
int anny_head_forward(mhmr_engine* e, const ImgSrc& x, const float* K, int B, float det_thresh, int nms,
                      const int64_t* forced_idx, int forced_P, const mhmr_anny_outputs* o, cudaStream_t st) {
  const int D = e->D, N = e->N, T = e->T, res = e->res, Pm = e->cfg.max_persons, Bm = e->cfg.max_batch;
  const int nb = e->cfg.num_betas, dim = e->dec_dim, J = e->cfg.num_joints, BN = B * N, J6p = (6 * J + 3) & ~3;
  const AnnyHeadWeights& hw = e->anny_w;
  int* det_b = o->det_idx; int* det_y = o->det_idx + Pm; int* det_x = o->det_idx + 2 * Pm;
  int* count = e->count + 2;
  // detection (encoder.py:59-60, multi_hmr.py:116-124)
  TRY(detect(e, B, det_thresh, nms, forced_idx, forced_P, false, o->logits, o->scores_map, o->det_idx, e->det_score,
             o->count, st));
  // decoder tokens of every cell and the keys / values of every HPH layer
  TRY(run_plan(e, MHMR_CAT_GEMM_OTHER, e->dt_plan, BN, st));
  TRY(run_plan(e, MHMR_CAT_GEMM_OTHER, e->kv_plan, BN, st));
  // cls rows (camera) and person rows: fp32 refinement, or the bulk pass
  MHMR_CUDA_CHECK(cudaMemcpyAsync(e->anny_ints, &B, sizeof(int), cudaMemcpyHostToDevice, st));
  const float *xr = nullptr, *cls_src = e->cls_x;
  if (e->cfg.refine_central) {
    TRY(refine_streams(e, x, det_b, det_y, det_x, count, B, e->anny_ints + 1, st));
    xr = e->r_x + static_cast<size_t>(B) * D;
    cls_src = e->r_x;
  } else if (e->ln_fold) {
    LAUNCH(MHMR_CAT_HEAD, cls_gather(e->Xn16, e->Xlo, D, T, B, D, e->cls_x, st));
  } else {
    LAUNCH(MHMR_CAT_HEAD, cls_gather(e->X, nullptr, D, T, B, D, e->cls_x, st));
  }
  // field of view and intrinsics (encoder.py:50-56)
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(cls_src, D, e->anny_ints, Bm, D, hw.fov0_w, D, hw.fov0_b, D, e->norm_g, e->norm_b,
                                      1e-6f, 1, nullptr, 0, e->cls_h, D, st));
  LAUNCH(MHMR_CAT_HEAD, anny_camera(e->cls_h, D, hw.fov2_w, hw.fov2_b, hw.fov_max, K, B, e->cfg.img_size, o->fov,
                                    o->K_regressed, e->K_use, e->Kinv, st));
  ++e->launches;  // anny_camera = 2 kernels
  // queries: dec_to_token(final-normed feature) + dec_pos_emb at the detected cells (multi_hmr.py:131)
  LAUNCH(MHMR_CAT_HEAD, anny_gather(e->z32, xr, e->norm_g, e->norm_b, hw.dec_pos_emb, det_b, det_y, det_x, count, Pm, res,
                                    D, dim, e->zc, e->xa, st));
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->zc, D, count, Pm, D, hw.dt_w, D, hw.dt_b, dim, nullptr, nullptr, 0.f, 0, e->xa, dim,
                                      e->xa, dim, st));
  // HPH (hph.py:133-140)
  TRY(hph_decoder(e, det_b, count, st));
  // regressors: hidden layers of offset | dist | shape | pose at once, then the four output Linears
  float* hid = e->offh;
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(e->xa, dim, count, Pm, dim, e->W1, dim, e->b1, 4 * dim, nullptr, nullptr, 0.f, 1,
                                      nullptr, 0, hid, 4 * dim, st));
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(hid, 4 * dim, count, Pm, dim, hw.off2_w, dim, hw.off2_b, 2, nullptr, nullptr, 0.f, 0,
                                      nullptr, 0, o->offset, 2, st));
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(hid + dim, 4 * dim, count, Pm, dim, hw.dist2_w, dim, hw.dist2_b, 1, nullptr, nullptr,
                                      0.f, 0, nullptr, 0, o->dist_pp, 1, st));
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(hid + 2 * dim, 4 * dim, count, Pm, dim, hw.shape2_w, dim, hw.shape2_b, nb, nullptr,
                                      nullptr, 0.f, 0, nullptr, 0, o->shape, nb, st));
  LAUNCH(MHMR_CAT_HEAD, skinny_linear(hid + 3 * dim, 4 * dim, count, Pm, dim, hw.pose2_w, dim, e->b_pose2, 6 * J, nullptr,
                                      nullptr, 0.f, 0, nullptr, 0, e->dec, J6p, st));
  LAUNCH(MHMR_CAT_HEAD, anny_person_post(e->dec, J6p, J, hw.useful_rotmat, o->shape, nb, o->offset, o->dist_pp, e->K_use,
                                         e->Kinv, det_b, det_y, det_x, count, Pm, o->rotmat, o->rotmat_homo, o->rotvec,
                                         o->dist, o->loc, o->transl, o->K_det, st));
  return MHMR_OK;
}

}  // namespace

extern "C" {

int mhmr_create(const mhmr_config* cfg, mhmr_engine** out) {
  MHMR_REQUIRE(cfg != nullptr && out != nullptr, "null argument");
  MHMR_REQUIRE(cfg->arch >= 0 && cfg->arch <= 2, "arch must be 0 (S), 1 (B) or 2 (L)");
  MHMR_REQUIRE(cfg->img_size > 0 && cfg->img_size % 14 == 0, "Invalid img size");  // model.py:65
  MHMR_REQUIRE(cfg->max_batch > 0 && cfg->max_persons > 0, "capacities must be positive");
  MHMR_REQUIRE(cfg->head == MHMR_HEAD_SMPLX || cfg->head == MHMR_HEAD_ANNY, "head must be 0 (SMPL-X) or 1 (Anny)");
  if (cfg->head == MHMR_HEAD_SMPLX) {
    MHMR_REQUIRE(cfg->num_betas == 10 || cfg->num_betas == 11, "num_betas must be 10 or 11");  // model.py:384
    MHMR_REQUIRE(cfg->xat_depth >= 1 && cfg->xat_depth <= 8 && cfg->xat_num_heads >= 1, "bad HPH geometry");
    MHMR_REQUIRE(cfg->person_center_idx >= 0 && cfg->person_center_idx < 55,
                 "person_center must be one of the 55 kinematic joints");
    MHMR_REQUIRE(cfg->num_verts > 0, "num_verts must be positive");
  } else {
    // multi_hmr.py:28-36: the HPH kernels are built for dim_head = 32 (one lane per channel)
    MHMR_REQUIRE(cfg->xat_depth >= 1 && cfg->xat_num_heads >= 1, "bad HPH geometry");
    MHMR_REQUIRE(cfg->xat_dim > 0 && cfg->xat_dim % 32 == 0 && cfg->xat_mlp_dim > 0 && cfg->xat_mlp_dim % 32 == 0,
                 "xat_dim and xat_mlp_dim must be positive multiples of 32");
    MHMR_REQUIRE(cfg->num_joints >= 1 && cfg->num_betas >= 1, "num_joints and num_betas must be positive");
    MHMR_REQUIRE(cfg->person_center_idx >= 0 && cfg->person_center_idx < cfg->num_joints,
                 "person_center_idx must index a bone of the body model");
  }
  auto e = std::make_unique<mhmr_engine>();
  e->cfg = *cfg;
  const ArchSpec& a = kArch[cfg->arch];
  e->D = a.D; e->depth = a.depth;
  e->dec_dim = e->dec_mlp = kHphDim;
  if (cfg->head == MHMR_HEAD_ANNY) {
    e->enc = "encoder.backbone.";
    e->dec_dim = cfg->xat_dim;
    e->dec_mlp = cfg->xat_mlp_dim;
  }
  e->res = cfg->img_size / 14;
  e->N = e->res * e->res;
  e->T = e->N + 1;
  e->C = e->D + kCamDim;
  e->Cp = e->D + 128;                 // fp16 context pitch: D feature columns + 99 camera columns + zero pad
  e->Cq = (e->C + 3) & ~3;            // fp32 per-person pitch
  e->nkv = cfg->xat_depth * 2 * cfg->xat_num_heads * 32;
  MHMR_REQUIRE(e->nkv % 32 == 0, "HPH inner dim must be a multiple of 32");
  *out = e.release();
  return MHMR_OK;
}

int mhmr_destroy(mhmr_engine* h) {
  delete h;
  return MHMR_OK;
}

static int store_copy(std::map<std::string, DevBuf>& m, const char* key, const void* data, size_t bytes) {
  MHMR_REQUIRE(key != nullptr && data != nullptr && bytes > 0, "null/empty tensor");
  auto it = m.find(key);
  if (it != m.end()) {
    cudaFree(it->second.p);
    m.erase(it);
  }
  DevBuf b;
  b.bytes = bytes;
  MHMR_CUDA_CHECK(cudaMalloc(&b.p, bytes));
  MHMR_CUDA_CHECK(cudaMemcpy(b.p, data, bytes, cudaMemcpyDefault));
  m[key] = b;
  return MHMR_OK;
}

int mhmr_set_weight(mhmr_engine* h, const char* key, const float* data, int64_t numel) {
  MHMR_REQUIRE(h != nullptr, "null engine");
  if (h->finalized) { set_last_error("engine already finalized"); return MHMR_ERR_STATE; }
  return store_copy(h->weights, key, data, static_cast<size_t>(numel) * 4);
}

int mhmr_set_table_i32(mhmr_engine* h, const char* key, const int32_t* data, int64_t numel) {
  MHMR_REQUIRE(h != nullptr, "null engine");
  if (h->finalized) { set_last_error("engine already finalized"); return MHMR_ERR_STATE; }
  return store_copy(h->tables, key, data, static_cast<size_t>(numel) * 4);
}

int mhmr_finalize(mhmr_engine* h) {
  MHMR_REQUIRE(h != nullptr, "null engine");
  if (h->finalized) return MHMR_OK;
  cudaStream_t st = nullptr;
  TRY(finalize_vit(h, st));
  if (h->cfg.head == MHMR_HEAD_ANNY) {
    TRY(finalize_anny(h, st));
  } else {
    TRY(finalize_head(h, st));
    TRY(finalize_body(h, st));
  }
  MHMR_CUDA_CHECK(cudaStreamSynchronize(st));
  h->finalized = true;
  return MHMR_OK;
}

// checks of the engine, batch and forced persons that every forward entry makes; `entry` names it in the messages
static int check_forward(mhmr_engine* h, const void* out, int head, const char* entry, int B, const int64_t* forced_idx,
                         int forced_P) {
  MHMR_REQUIRE(h != nullptr && out != nullptr, "null argument");
  if (!h->finalized) { set_last_error(std::string(entry) + " before mhmr_finalize"); return MHMR_ERR_STATE; }
  MHMR_REQUIRE(h->cfg.head == head, std::string(entry) + " needs an engine created with head = " +
                                        (head == MHMR_HEAD_ANNY ? "MHMR_HEAD_ANNY" : "MHMR_HEAD_SMPLX"));
  MHMR_REQUIRE(B >= 1 && B <= h->cfg.max_batch, "batch exceeds max_batch");
  MHMR_REQUIRE(forced_idx == nullptr || (forced_P >= 0 && forced_P <= h->cfg.max_persons),
               "forced_P exceeds max_persons");
  return MHMR_OK;
}

static int forward_impl(mhmr_engine* h, const ImgSrc& x, const float* K, int B, float det_thresh,
                        int nms_kernel_size, const int64_t* forced_idx, int forced_P, const mhmr_outputs* out,
                        void* stream) {
  MHMR_REQUIRE(K != nullptr, "null argument");
  TRY(check_forward(h, out, MHMR_HEAD_SMPLX, "mhmr_forward", B, forced_idx, forced_P));
  MHMR_REQUIRE(out->scores_map && out->count && out->det_idx && out->det_score && out->offset && out->loc &&
                   out->dist_pp && out->dist && out->rotmat && out->rotvec && out->shape && out->expression &&
                   out->transl && out->transl_pelvis && out->v3d && out->j3d && out->j2d,
               "a required output buffer is null");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  h->launches = 0;
  TRY(vit_forward(h, x, B, out->z, st));
  return head_forward(h, x, K, B, det_thresh, nms_kernel_size, forced_idx, forced_P, out, st);
}

int mhmr_forward(mhmr_engine* h, const float* x, const float* K, int B, float det_thresh,
                 int nms_kernel_size, const int64_t* forced_idx, int forced_P, const mhmr_outputs* out,
                 void* stream) {
  MHMR_REQUIRE(x != nullptr, "null image");
  ImgSrc src;
  src.f32 = x;
  return forward_impl(h, src, K, B, det_thresh, nms_kernel_size, forced_idx, forced_P, out, stream);
}

int mhmr_forward_u8(mhmr_engine* h, const uint8_t* img_u8, const float* lut, const float* K, int B, float det_thresh,
                    int nms_kernel_size, const int64_t* forced_idx, int forced_P, const mhmr_outputs* out,
                    void* stream) {
  MHMR_REQUIRE(img_u8 != nullptr && lut != nullptr, "null image / table");
  ImgSrc src;
  src.u8 = img_u8;
  src.lut = lut;
  return forward_impl(h, src, K, B, det_thresh, nms_kernel_size, forced_idx, forced_P, out, stream);
}

static int forward_anny_impl(mhmr_engine* h, const ImgSrc& x, const float* K, int B, float det_thresh,
                             int nms_kernel_size, const int64_t* forced_idx, int forced_P, const mhmr_anny_outputs* out,
                             void* stream) {
  TRY(check_forward(h, out, MHMR_HEAD_ANNY, "mhmr_forward_anny", B, forced_idx, forced_P));
  // multi_hmr.py:118: an even kernel changes the pooled map's shape and the reference fails on the comparison
  MHMR_REQUIRE(forced_idx != nullptr || nms_kernel_size <= 1 || nms_kernel_size % 2 == 1,
               "nms_kernel_size must be odd");
  MHMR_REQUIRE(out->scores_map && out->logits && out->count && out->det_idx && out->K_regressed && out->fov &&
                   out->K_det && out->offset && out->loc && out->dist && out->dist_pp && out->shape && out->rotmat &&
                   out->rotmat_homo && out->rotvec && out->transl,
               "a required output buffer is null");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  h->launches = 0;
  TRY(vit_forward(h, x, B, out->z, st));
  return anny_head_forward(h, x, K, B, det_thresh, nms_kernel_size, forced_idx, forced_P, out, st);
}

int mhmr_forward_anny(mhmr_engine* h, const float* x, const float* K, int B, float det_thresh, int nms_kernel_size,
                      const int64_t* forced_idx, int forced_P, const mhmr_anny_outputs* out, void* stream) {
  MHMR_REQUIRE(x != nullptr, "null image");
  ImgSrc src;
  src.f32 = x;
  return forward_anny_impl(h, src, K, B, det_thresh, nms_kernel_size, forced_idx, forced_P, out, stream);
}

int mhmr_forward_anny_u8(mhmr_engine* h, const uint8_t* img_u8, const float* lut, const float* K, int B,
                         float det_thresh, int nms_kernel_size, const int64_t* forced_idx, int forced_P,
                         const mhmr_anny_outputs* out, void* stream) {
  MHMR_REQUIRE(img_u8 != nullptr && lut != nullptr, "null image / table");
  ImgSrc src;
  src.u8 = img_u8;
  src.lut = lut;
  return forward_anny_impl(h, src, K, B, det_thresh, nms_kernel_size, forced_idx, forced_P, out, stream);
}

int mhmr_anny_place(mhmr_engine* h, int P, int V, const float* bone_poses, const float* transl, const float* K_det,
                    float* v3d, float* j3d, float* v2d, float* j2d, float* transl_pelvis, void* stream) {
  MHMR_REQUIRE(h != nullptr, "null engine");
  MHMR_REQUIRE(h->cfg.head == MHMR_HEAD_ANNY, "mhmr_anny_place needs an Anny engine");
  MHMR_REQUIRE(P >= 0 && P <= h->cfg.max_persons && V >= 0, "P exceeds max_persons");
  MHMR_REQUIRE(bone_poses && transl && K_det && j3d && j2d && transl_pelvis && (V == 0 || v3d), "null argument");
  return anny_place(bone_poses, transl, K_det, h->cfg.person_center_idx, P, V, h->cfg.num_joints, v3d, j3d, v2d, j2d,
                    transl_pelvis, static_cast<cudaStream_t>(stream));
}

int mhmr_sync_count(mhmr_engine* h, void* stream, int* num_persons) {
  MHMR_REQUIRE(h != nullptr && num_persons != nullptr, "null argument");
  MHMR_CUDA_CHECK(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  *num_persons = *h->h_count;
  if (*h->h_count > h->cfg.max_persons) {
    set_last_error("detected " + std::to_string(*h->h_count) + " persons > max_persons " +
                   std::to_string(h->cfg.max_persons));
    return MHMR_ERR_CAPACITY;
  }
  return MHMR_OK;
}

int mhmr_vit_forward(mhmr_engine* h, const float* x, int B, float* z, void* stream) {
  MHMR_REQUIRE(h != nullptr && x != nullptr && z != nullptr, "null argument");
  if (!h->finalized) { set_last_error("mhmr_vit_forward before mhmr_finalize"); return MHMR_ERR_STATE; }
  MHMR_REQUIRE(B >= 1 && B <= h->cfg.max_batch, "batch exceeds max_batch");
  h->launches = 0;
  ImgSrc src;
  src.f32 = x;
  return vit_forward(h, src, B, z, static_cast<cudaStream_t>(stream));
}

int mhmr_op_vit_stream(mhmr_engine* h, const float* x, int B, int layers, float* out, void* stream) {
  MHMR_REQUIRE(h != nullptr && x != nullptr && out != nullptr, "null argument");
  if (!h->finalized) { set_last_error("mhmr_op_vit_stream before mhmr_finalize"); return MHMR_ERR_STATE; }
  MHMR_REQUIRE(B >= 1 && B <= h->cfg.max_batch, "batch exceeds max_batch");
  MHMR_REQUIRE(layers >= 0 && layers <= h->depth, "layers outside [0, depth]");
  h->launches = 0;
  ImgSrc src;
  src.f32 = x;
  return vit_forward(h, src, B, nullptr, static_cast<cudaStream_t>(stream), layers, out);
}

int mhmr_smplx_forward(mhmr_engine* h, int P, const float* rotvec, const float* shape,
                       const float* expression, const float* loc, const float* dist, const float* K_det,
                       float* v3d, float* v2d, float* j3d, float* j2d, float* transl, float* transl_pelvis,
                       void* stream) {
  MHMR_REQUIRE(h != nullptr, "null engine");
  if (!h->finalized) { set_last_error("mhmr_smplx_forward before mhmr_finalize"); return MHMR_ERR_STATE; }
  MHMR_REQUIRE(h->cfg.head == MHMR_HEAD_SMPLX, "mhmr_smplx_forward needs an SMPL-X engine");
  MHMR_REQUIRE(P >= 1 && P <= h->cfg.max_persons, "P exceeds max_persons");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DeviceBody& b = h->body;
  MHMR_CUDA_CHECK(cudaMemcpyAsync(b.count, &P, sizeof(int), cudaMemcpyHostToDevice, st));
  TRY(loc_to_transl(loc, dist, K_det, P, transl, st));
  return smplx_forward(b.bm, rotvec, shape, expression, transl, K_det, b.count, P, b.ws, v3d, v2d, j3d, j2d,
                       transl_pelvis, st);
}

int mhmr_smplx_backward(mhmr_engine* h, int P, const float* rotvec, const float* shape, const float* expression,
                        const float* loc, const float* dist, const float* K_det, const float* g_v3d, const float* g_v2d,
                        const float* g_j3d, const float* g_j2d, const float* g_transl, const float* g_transl_pelvis,
                        float* d_rotvec, float* d_shape, float* d_expression, float* d_loc, float* d_dist,
                        void* stream) {
  MHMR_REQUIRE(h != nullptr, "null engine");
  if (!h->finalized) { set_last_error("mhmr_smplx_backward before mhmr_finalize"); return MHMR_ERR_STATE; }
  MHMR_REQUIRE(h->cfg.head == MHMR_HEAD_SMPLX, "mhmr_smplx_backward needs an SMPL-X engine");
  MHMR_REQUIRE(P >= 1 && P <= h->cfg.max_persons, "P exceeds max_persons");
  MHMR_REQUIRE(rotvec && shape && expression && loc && dist && K_det && d_rotvec && d_shape && d_loc && d_dist,
               "null argument");
  BodyGrads g;
  g.v3d = g_v3d; g.v2d = g_v2d; g.j3d = g_j3d; g.j2d = g_j2d; g.tp = g_transl_pelvis;
  return smplx_backward(h->body.bm, h->body.gs, P, rotvec, shape, expression, loc, dist, K_det, g, g_transl, d_rotvec,
                        d_shape, d_expression, d_loc, d_dist, static_cast<cudaStream_t>(stream));
}

int mhmr_last_launch_count(mhmr_engine* h) { return h != nullptr ? h->launches : 0; }

int mhmr_set_profiling(mhmr_engine* h, int enable) {
  MHMR_REQUIRE(h != nullptr, "null engine");
  h->profiling = enable != 0;
  h->prof.clear();
  h->events_used = 0;
  return MHMR_OK;
}

int mhmr_get_profile(mhmr_engine* h, float* ms_by_category, int* launches_by_category) {
  MHMR_REQUIRE(h != nullptr && ms_by_category != nullptr && launches_by_category != nullptr, "null argument");
  for (int c = 0; c < MHMR_NUM_CATEGORIES; ++c) { ms_by_category[c] = 0.f; launches_by_category[c] = 0; }
  for (const auto& p : h->prof) {
    MHMR_CUDA_CHECK(cudaEventSynchronize(p.b));
    float ms = 0.f;
    MHMR_CUDA_CHECK(cudaEventElapsedTime(&ms, p.a, p.b));
    ms_by_category[p.cat] += ms;
    launches_by_category[p.cat] += 1;
  }
  h->prof.clear();
  h->events_used = 0;
  return MHMR_OK;
}

}  // extern "C"
