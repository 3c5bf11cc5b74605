// Ground-truth body models of the evaluation protocols (reference Trainer.prepare_gt, train.py:58-134): the raw
// `smplx` forward -- SMPL male / female (3DPW, train.py:74-94) and SMPL-X neutral with 11 betas (BEDLAM, :95-110) --
// behind a handle independent of the engine, since an evaluation holds three of them at once.  The kernels are the
// engine's own (smplx_lbs.cu) instantiated for the body model's joint count; this file only folds the load-time
// tables and validates the per-call sizes.
#include <vector>

#include "kernels.cuh"

using namespace mhmr;

struct mhmr_body {
  int kind = 0, V = 0, nb = 0, ne = 0, NJ = 0, max_persons = 0;
  SmplxDeviceModel bm;
  SmplxScratch ws;
  SmplxGradScratch gs;
  int* count = nullptr;
  std::vector<void*> allocs;
  ~mhmr_body() {
    for (void* p : allocs) cudaFree(p);
  }
  template <typename T>
  int alloc(T** out, size_t n) {
    void* p = nullptr;
    MHMR_CUDA_CHECK(cudaMalloc(&p, n * sizeof(T)));
    allocs.push_back(p);
    *out = static_cast<T*>(p);
    return MHMR_OK;
  }
};

#define TRY(expr)                   \
  do {                              \
    int rc_ = (expr);               \
    if (rc_ != MHMR_OK) return rc_; \
  } while (0)

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

int body_build(mhmr_body* h, const float* v_template, const float* shapedirs, const float* expr_dirs,
               const float* posedirs, const float* J_regressor, const float* lbs_weights, const int32_t* parents,
               const int32_t* extra_idx, const int32_t* lmk_tri, const float* lmk_bary, cudaStream_t st) {
  const int V = h->V, nb = h->nb, ne = h->ne, NJ = h->NJ, L = nb + ne, PF = 9 * (NJ - 1);
  const int nl = (h->kind == MHMR_BODY_SMPLX) ? 51 : 0;
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

  Staging stage;
  const float *vt_d, *sd_d, *ed_d = nullptr, *pd_d, *jr_d, *lw_d, *bary_d = nullptr;
  TRY(stage.copy(v_template, 3ll * V, &vt_d, st));
  TRY(stage.copy(shapedirs, 3ll * V * nb, &sd_d, st));
  if (ne) TRY(stage.copy(expr_dirs, 3ll * V * ne, &ed_d, st));
  TRY(stage.copy(posedirs, static_cast<size_t>(PF) * 3 * V, &pd_d, st));
  TRY(stage.copy(J_regressor, static_cast<size_t>(NJ) * V, &jr_d, st));
  TRY(stage.copy(lbs_weights, static_cast<size_t>(V) * NJ, &lw_d, st));
  if (nl) TRY(stage.copy(lmk_bary, 3 * nl, &bary_d, st));

  SmplxDeviceModel& bm = h->bm;
  bm.V = V; bm.L = L; bm.num_betas = nb; bm.center_idx = 0;
  bm.num_joints = NJ; bm.pose_feat = PF; bm.n_lmk = nl;
  bm.ldp = (3 * V + 3) & ~3;
  float *sfull, *PDX, *vtp, *Jt, *Jd, *lwp, *bary = nullptr;
  int *par, *ext, *tri = nullptr;
  TRY(h->alloc(&sfull, static_cast<size_t>(3) * V * L));
  TRY(repack_f32(sd_d, nb, 0, sfull, L, 0, 3 * V, nb, false, st));
  if (ne) TRY(repack_f32(ed_d, ne, 0, sfull, L, nb, 3 * V, ne, false, st));
  TRY(h->alloc(&PDX, static_cast<size_t>(PF + L) * bm.ldp));
  TRY(smplx_build_pdx(pd_d, sfull, PF, L, V, bm.ldp, PDX, st));
  TRY(h->alloc(&vtp, bm.ldp));
  MHMR_CUDA_CHECK(cudaMemsetAsync(vtp, 0, bm.ldp * 4, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(vtp, vt_d, 3ll * V * 4, cudaMemcpyDeviceToDevice, st));
  TRY(h->alloc(&Jt, NJ * 3));
  TRY(smplx_fold_jreg(jr_d, vt_d, NJ, V, 3, Jt, st));
  TRY(h->alloc(&Jd, static_cast<size_t>(NJ) * 3 * L));
  TRY(smplx_fold_jreg(jr_d, sfull, NJ, V, 3 * L, Jd, st));
  const int tv = smplx_tile_verts();
  const int Vpad = (V + tv - 1) / tv * tv;
  TRY(h->alloc(&lwp, static_cast<size_t>(Vpad) * NJ));
  MHMR_CUDA_CHECK(cudaMemsetAsync(lwp, 0, static_cast<size_t>(Vpad) * NJ * 4, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(lwp, lw_d, static_cast<size_t>(V) * NJ * 4, cudaMemcpyDeviceToDevice, st));
  TRY(h->alloc(&par, NJ));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(par, hp.data(), NJ * 4, cudaMemcpyHostToDevice, st));
  TRY(h->alloc(&ext, 21));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(ext, he.data(), 21 * 4, cudaMemcpyHostToDevice, st));
  if (nl) {
    TRY(h->alloc(&tri, 3 * nl));
    MHMR_CUDA_CHECK(cudaMemcpyAsync(tri, ht.data(), 3 * nl * 4, cudaMemcpyHostToDevice, st));
    TRY(h->alloc(&bary, 3 * nl));
    MHMR_CUDA_CHECK(cudaMemcpyAsync(bary, bary_d, 3 * nl * 4, cudaMemcpyDeviceToDevice, st));
  }
  bm.PDX = PDX; bm.vt = vtp; bm.lbs_weights_padded = lwp; bm.Jt = Jt; bm.Jdirs = Jd;
  bm.parents = par; bm.extra_idx = ext; bm.lmk_tri = tri; bm.lmk_bary = bary;
  TRY(smplx_make_tmap(&bm));
  const int Pm = h->max_persons;
  TRY(h->alloc(&h->ws.cf, static_cast<size_t>(Pm) * (PF + L)));
  TRY(h->alloc(&h->ws.Amat, static_cast<size_t>(Pm) * NJ * 12));
  TRY(h->alloc(&h->ws.xf, static_cast<size_t>(Pm) * 16));
  TRY(h->alloc(&h->ws.jposed, static_cast<size_t>(Pm) * NJ * 3));
  TRY(h->alloc(&h->count, 1));
  // backward scratch and the vertex -> joint table (synchronises: loading finishes before the staging buffers are
  // freed and before the caller may free its arrays)
  return smplx_grad_init(bm, Pm, [h](void** p, size_t bytes) {
    uint8_t* q = nullptr;
    const int rc = h->alloc(&q, bytes);
    *p = q;
    return rc;
  }, &h->gs, st);
}

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
  const int ne = (kind == MHMR_BODY_SMPLX) ? 10 : 0;
  MHMR_REQUIRE(num_betas + ne <= 32, "at most 32 shape + expression coefficients");
  MHMR_REQUIRE(9 * ((kind == MHMR_BODY_SMPLX) ? 54 : 23) + num_betas + ne <= 512,
               "pose features + shape + expression coefficients exceed the vertex kernel's 512 rows");
  MHMR_REQUIRE(v_template && shapedirs && posedirs && J_regressor && lbs_weights && parents && extra_joints_idxs,
               "null body-model array");
  MHMR_REQUIRE(kind == MHMR_BODY_SMPL || (expr_dirs && lmk_tri && lmk_bary),
               "SMPL-X needs expr_dirs, lmk_tri and lmk_bary");
  auto* h = new mhmr_body();
  h->kind = kind; h->V = num_verts; h->nb = num_betas; h->ne = ne; h->max_persons = max_persons;
  h->NJ = (kind == MHMR_BODY_SMPLX) ? 55 : 24;
  const int rc = body_build(h, v_template, shapedirs, expr_dirs, posedirs, J_regressor, lbs_weights, parents,
                            extra_joints_idxs, lmk_tri, lmk_bary, static_cast<cudaStream_t>(stream));
  if (rc != MHMR_OK) {
    delete h;
    return rc;
  }
  *out = h;
  return MHMR_OK;
}

int mhmr_body_destroy(mhmr_body* h) {
  delete h;
  return MHMR_OK;
}

int mhmr_body_info(const mhmr_body* h, int* num_verts, int* num_joints_out, int* num_pose_joints, int* num_betas,
                   int* num_expression) {
  MHMR_REQUIRE(h != nullptr, "null body model");
  if (num_verts) *num_verts = h->V;
  if (num_joints_out) *num_joints_out = h->NJ + 21 + h->bm.n_lmk;
  if (num_pose_joints) *num_pose_joints = h->NJ;
  if (num_betas) *num_betas = h->nb;
  if (num_expression) *num_expression = h->ne;
  return MHMR_OK;
}

int mhmr_body_forward(mhmr_body* h, int P, const float* full_pose, const float* betas, const float* expression,
                      const float* transl, const float* K, float* v3d, float* v2d, float* j3d, float* j2d,
                      float* transl_pelvis, void* stream) {
  MHMR_REQUIRE(h != nullptr, "null body model");
  MHMR_REQUIRE(P >= 0 && P <= h->max_persons, "P exceeds the handle's max_persons");
  MHMR_REQUIRE(full_pose && betas && transl && K && v3d && j3d && j2d && transl_pelvis, "null argument");
  MHMR_REQUIRE(h->ne == 0 || expression != nullptr, "SMPL-X needs an expression array");
  if (P == 0) return MHMR_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MHMR_CUDA_CHECK(cudaMemcpyAsync(h->count, &P, sizeof(int), cudaMemcpyHostToDevice, st));
  return body_forward_raw(h->bm, full_pose, betas, expression, transl, K, h->count, P, h->ws, v3d, v2d, j3d, j2d,
                          transl_pelvis, st);
}

int mhmr_body_backward(mhmr_body* h, int P, const float* full_pose, const float* betas, const float* expression,
                       const float* transl, const float* K, const float* g_v3d, const float* g_v2d, const float* g_j3d,
                       const float* g_j2d, const float* g_transl_pelvis, float* d_full_pose, float* d_betas,
                       float* d_expression, float* d_transl, void* stream) {
  MHMR_REQUIRE(h != nullptr, "null body model");
  MHMR_REQUIRE(P >= 0 && P <= h->max_persons, "P exceeds the handle's max_persons");
  MHMR_REQUIRE(full_pose && betas && transl && K && d_full_pose && d_betas && d_transl, "null argument");
  MHMR_REQUIRE(h->ne == 0 || expression != nullptr, "SMPL-X needs an expression array");
  if (P == 0) return MHMR_OK;
  BodyGrads g;
  g.v3d = g_v3d; g.v2d = g_v2d; g.j3d = g_j3d; g.j2d = g_j2d; g.tp = g_transl_pelvis;
  return body_backward_raw(h->bm, h->gs, P, full_pose, betas, expression, transl, K, g, d_full_pose, d_betas,
                           h->ne ? d_expression : nullptr, d_transl, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
