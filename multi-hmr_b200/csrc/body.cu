// Ground-truth body models of the evaluation protocols (reference Trainer.prepare_gt, train.py:58-134): the raw
// `smplx` forward -- SMPL male / female (3DPW, train.py:74-94) and SMPL-X neutral with 11 betas (BEDLAM, :95-110) --
// behind a handle independent of the engine, since an evaluation holds three of them at once.  The kernels are the
// engine's own (smplx_lbs.cu) instantiated for the body model's joint count.  This file folds the load-time tables of
// these handles and of the engine's SMPL-X layer (body_build) and validates the per-call sizes.
#include <memory>
#include <vector>

#include "kernels.cuh"

using namespace mhmr;

struct mhmr_body {
  int kind = 0;
  DeviceBody body;
};

namespace mhmr {

// What the vertex kernel takes: at most 32 blend-shape coefficients and 512 coefficient rows
static int body_limits(int joints, int L) {
  MHMR_REQUIRE(L <= 32, "at most 32 shape + expression coefficients");
  MHMR_REQUIRE(9 * (joints - 1) + L <= 512,
               "pose features + shape + expression coefficients exceed the vertex kernel's 512 rows");
  return MHMR_OK;
}

int body_build(DeviceBody* b, int joints, int V, int nb, int ne, int center_idx, int max_persons,
               const float* v_template, const float* shapedirs, const float* expr_dirs, const float* posedirs,
               const float* J_regressor, const float* lbs_weights, const int32_t* parents, const int32_t* extra_idx,
               const int32_t* lmk_tri, const float* lmk_bary, cudaStream_t st) {
  const int NJ = joints, L = nb + ne, PF = 9 * (NJ - 1), nl = (NJ == 55) ? 51 : 0;
  TRY(body_limits(NJ, L));
  // integer tables are validated on the host before anything reads them on the device
  std::vector<int32_t> hp(NJ), he(21), ht(3 * nl);
  MHMR_CUDA_CHECK(cudaMemcpy(hp.data(), parents, NJ * 4, cudaMemcpyDefault));
  MHMR_CUDA_CHECK(cudaMemcpy(he.data(), extra_idx, 21 * 4, cudaMemcpyDefault));
  if (nl) MHMR_CUDA_CHECK(cudaMemcpy(ht.data(), lmk_tri, 3 * nl * 4, cudaMemcpyDefault));
  MHMR_REQUIRE(hp[0] < 0, "parents[0] must be the root (-1)");
  for (int j = 1; j < NJ; ++j) MHMR_REQUIRE(hp[j] >= 0 && hp[j] < j, "parents[j] must precede j");
  for (int d, j = 1; j < NJ; ++j) {  // the prep kernel walks at most 16 ancestors
    d = 1;
    for (int a = j; hp[a] >= 0; a = hp[a]) ++d;
    MHMR_REQUIRE(d <= 16, "kinematic chain deeper than 16 joints");
  }
  for (int v : he) MHMR_REQUIRE(v >= 0 && v < V, "extra_joints_idxs out of range");
  for (int v : ht) MHMR_REQUIRE(v >= 0 && v < V, "lmk_tri out of range");

  SmplxDeviceModel& bm = b->bm;
  bm.V = V; bm.L = L; bm.num_betas = nb; bm.center_idx = center_idx;
  bm.num_joints = NJ; bm.pose_feat = PF; bm.n_lmk = nl;
  bm.ldp = (3 * V + 3) & ~3;
  float *sfull, *PDX, *vtp, *Jt, *Jd, *lwp, *bary = nullptr;
  int *par, *ext, *tri = nullptr;
  TRY(b->alloc(&sfull, static_cast<size_t>(3) * V * L, st));
  TRY(repack_f32(shapedirs, nb, 0, sfull, L, 0, 3 * V, nb, false, st));
  if (ne) TRY(repack_f32(expr_dirs, ne, 0, sfull, L, nb, 3 * V, ne, false, st));
  TRY(b->alloc(&PDX, static_cast<size_t>(PF + L) * bm.ldp, st));
  TRY(smplx_build_pdx(posedirs, sfull, PF, L, V, bm.ldp, PDX, st));
  TRY(b->alloc(&vtp, bm.ldp, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(vtp, v_template, 3ll * V * 4, cudaMemcpyDeviceToDevice, st));
  TRY(b->alloc(&Jt, NJ * 3, st));
  TRY(smplx_fold_jreg(J_regressor, v_template, NJ, V, 3, Jt, st));
  TRY(b->alloc(&Jd, static_cast<size_t>(NJ) * 3 * L, st));
  TRY(smplx_fold_jreg(J_regressor, sfull, NJ, V, 3 * L, Jd, st));
  // skinning weights padded to whole tiles (the vertex kernel bulk-copies one tile per CTA)
  const int tv = smplx_tile_verts();
  const int Vpad = (V + tv - 1) / tv * tv;
  TRY(b->alloc(&lwp, static_cast<size_t>(Vpad) * NJ, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(lwp, lbs_weights, static_cast<size_t>(V) * NJ * 4, cudaMemcpyDeviceToDevice, st));
  TRY(b->alloc(&par, NJ, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(par, hp.data(), NJ * 4, cudaMemcpyHostToDevice, st));
  TRY(b->alloc(&ext, 21, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(ext, he.data(), 21 * 4, cudaMemcpyHostToDevice, st));
  if (nl) {
    TRY(b->alloc(&tri, 3 * nl, st));
    MHMR_CUDA_CHECK(cudaMemcpyAsync(tri, ht.data(), 3 * nl * 4, cudaMemcpyHostToDevice, st));
    TRY(b->alloc(&bary, 3 * nl, st));
    MHMR_CUDA_CHECK(cudaMemcpyAsync(bary, lmk_bary, 3 * nl * 4, cudaMemcpyDeviceToDevice, st));
  }
  bm.PDX = PDX; bm.vt = vtp; bm.lbs_weights_padded = lwp; bm.Jt = Jt; bm.Jdirs = Jd;
  bm.parents = par; bm.extra_idx = ext; bm.lmk_tri = tri; bm.lmk_bary = bary;
  TRY(smplx_make_tmap(&bm));
  TRY(b->alloc(&b->ws.cf, static_cast<size_t>(max_persons) * (PF + L), st));
  TRY(b->alloc(&b->ws.Amat, static_cast<size_t>(max_persons) * NJ * 12, st));
  TRY(b->alloc(&b->ws.xf, static_cast<size_t>(max_persons) * 16, st));
  TRY(b->alloc(&b->ws.jposed, static_cast<size_t>(max_persons) * NJ * 3, st));
  TRY(b->alloc(&b->count, 1, st));
  // backward scratch and the vertex -> joint table (synchronises: loading finishes before hp / he / ht go out of
  // scope and before the caller may free its arrays)
  return smplx_grad_init(b, max_persons, st);
}

}  // namespace mhmr

namespace {

// Device copies of the caller's float arrays, which may be host or device memory: every folding kernel reads these,
// never the caller's pointers.  Freed when loading is done.
struct Staging {
  std::vector<void*> bufs;
  ~Staging() {
    for (void* p : bufs) cudaFree(p);
  }
  int copy(const float* src, size_t n, const float** out, cudaStream_t st) {
    void* p = nullptr;
    MHMR_CUDA_CHECK(cudaMalloc(&p, n * sizeof(float)));
    bufs.push_back(p);
    MHMR_CUDA_CHECK(cudaMemcpyAsync(p, src, n * sizeof(float), cudaMemcpyDefault, st));
    *out = static_cast<const float*>(p);
    return MHMR_OK;
  }
};

}  // namespace

extern "C" {

int mhmr_body_create(int kind, int num_verts, int num_betas, int max_persons, const float* v_template,
                     const float* shapedirs, const float* expr_dirs, const float* posedirs, const float* J_regressor,
                     const float* lbs_weights, const int32_t* parents, const int32_t* extra_joints_idxs,
                     const int32_t* lmk_tri, const float* lmk_bary, void* stream, mhmr_body** out) {
  MHMR_REQUIRE(out != nullptr, "null output handle");
  *out = nullptr;
  MHMR_REQUIRE(kind == MHMR_BODY_SMPL || kind == MHMR_BODY_SMPLX, "kind must be MHMR_BODY_SMPL or MHMR_BODY_SMPLX");
  MHMR_REQUIRE(num_verts >= 1 && num_betas >= 1 && max_persons >= 1, "sizes must be positive");
  MHMR_REQUIRE(v_template && shapedirs && posedirs && J_regressor && lbs_weights && parents && extra_joints_idxs,
               "null body-model array");
  MHMR_REQUIRE(kind == MHMR_BODY_SMPL || (expr_dirs && lmk_tri && lmk_bary),
               "SMPL-X needs expr_dirs, lmk_tri and lmk_bary");
  const bool x = kind == MHMR_BODY_SMPLX;
  const int V = num_verts, nb = num_betas, ne = x ? 10 : 0, NJ = x ? 55 : 24, PF = 9 * (NJ - 1);
  TRY(body_limits(NJ, nb + ne));  // before staging reads num_betas columns of shapedirs
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Staging stage;
  const float *vt, *sd, *ed = nullptr, *pd, *jr, *lw, *bary = nullptr;
  TRY(stage.copy(v_template, 3ll * V, &vt, st));
  TRY(stage.copy(shapedirs, 3ll * V * nb, &sd, st));
  if (x) TRY(stage.copy(expr_dirs, 3ll * V * ne, &ed, st));
  TRY(stage.copy(posedirs, static_cast<size_t>(PF) * 3 * V, &pd, st));
  TRY(stage.copy(J_regressor, static_cast<size_t>(NJ) * V, &jr, st));
  TRY(stage.copy(lbs_weights, static_cast<size_t>(V) * NJ, &lw, st));
  if (x) TRY(stage.copy(lmk_bary, 51 * 3, &bary, st));
  auto h = std::make_unique<mhmr_body>();
  h->kind = kind;
  TRY(body_build(&h->body, NJ, V, nb, ne, 0, max_persons, vt, sd, ed, pd, jr, lw, parents, extra_joints_idxs, lmk_tri,
                 bary, st));
  *out = h.release();
  return MHMR_OK;
}

int mhmr_body_destroy(mhmr_body* h) {
  delete h;
  return MHMR_OK;
}

int mhmr_body_info(const mhmr_body* h, int* num_verts, int* num_joints_out, int* num_pose_joints, int* num_betas,
                   int* num_expression) {
  MHMR_REQUIRE(h != nullptr, "null body model");
  const SmplxDeviceModel& bm = h->body.bm;
  if (num_verts) *num_verts = bm.V;
  if (num_joints_out) *num_joints_out = bm.num_joints + 21 + bm.n_lmk;
  if (num_pose_joints) *num_pose_joints = bm.num_joints;
  if (num_betas) *num_betas = bm.num_betas;
  if (num_expression) *num_expression = bm.L - bm.num_betas;
  return MHMR_OK;
}

int mhmr_body_forward(mhmr_body* h, int P, const float* full_pose, const float* betas, const float* expression,
                      const float* transl, const float* K, float* v3d, float* v2d, float* j3d, float* j2d,
                      float* transl_pelvis, void* stream) {
  MHMR_REQUIRE(h != nullptr, "null body model");
  MHMR_REQUIRE(P >= 0 && P <= h->body.gs.max_persons, "P exceeds the handle's max_persons");
  MHMR_REQUIRE(full_pose && betas && transl && K && v3d && j3d && j2d && transl_pelvis, "null argument");
  MHMR_REQUIRE(h->kind == MHMR_BODY_SMPL || expression != nullptr, "SMPL-X needs an expression array");
  if (P == 0) return MHMR_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DeviceBody& b = h->body;
  MHMR_CUDA_CHECK(cudaMemcpyAsync(b.count, &P, sizeof(int), cudaMemcpyHostToDevice, st));
  return body_forward_raw(b.bm, full_pose, betas, expression, transl, K, b.count, P, b.ws, v3d, v2d, j3d, j2d,
                          transl_pelvis, st);
}

int mhmr_body_backward(mhmr_body* h, int P, const float* full_pose, const float* betas, const float* expression,
                       const float* transl, const float* K, const float* g_v3d, const float* g_v2d, const float* g_j3d,
                       const float* g_j2d, const float* g_transl_pelvis, float* d_full_pose, float* d_betas,
                       float* d_expression, float* d_transl, void* stream) {
  MHMR_REQUIRE(h != nullptr, "null body model");
  MHMR_REQUIRE(P >= 0 && P <= h->body.gs.max_persons, "P exceeds the handle's max_persons");
  MHMR_REQUIRE(full_pose && betas && transl && K && d_full_pose && d_betas && d_transl, "null argument");
  MHMR_REQUIRE(h->kind == MHMR_BODY_SMPL || expression != nullptr, "SMPL-X needs an expression array");
  if (P == 0) return MHMR_OK;
  BodyGrads g;
  g.v3d = g_v3d; g.v2d = g_v2d; g.j3d = g_j3d; g.j2d = g_j2d; g.tp = g_transl_pelvis;
  return body_backward_raw(h->body.bm, h->body.gs, P, full_pose, betas, expression, transl, K, g, d_full_pose,
                           d_betas, h->kind == MHMR_BODY_SMPLX ? d_expression : nullptr, d_transl,
                           static_cast<cudaStream_t>(stream));
}

}  // extern "C"
