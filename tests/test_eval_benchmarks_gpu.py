"""The 3DPW / EHF / BEDLAM evaluation protocols on the device: ground-truth body models (mhmr_body_*) and the pair
regression (mhmr_eval_regress) against float64 references, `metrics.evaluate` against the goldens of the reference's
own Trainer.evaluate, an end-to-end run on engine predictions, and a sensitivity check for each plausible mistake."""
import os

import numpy as np
import pytest
import torch

from oracle import eval_bench_ref as R
from oracle import smplx_ref

pytestmark = pytest.mark.gpu
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def assets():
    return R.eval_assets(0)


@pytest.fixture(scope="module")
def dev_assets(assets, cuda_device):
    from multihmr_b200 import metrics

    return metrics.EvalAssets(assets["smplx"], assets["smpl_male"], assets["smpl_female"], assets["smplx2smpl"],
                              assets["j_regressor_h36m"], device=cuda_device)


def _fp64_body(bm, kind, full_pose, betas, transl, expression=None, extra=None):
    """smplx.SMPL / smplx.SMPLX forward in float64 (oracle/smplx_ref.lbs is dtype-generic)."""
    d = lambda k: bm[k].double()
    if kind == "smpl":
        comps, dirs = betas.double(), d("shapedirs")[..., :10]
    else:
        sd = torch.cat([bm["shapedirs"], bm["shapedirs_extra"]], -1)[..., :11].double()
        comps, dirs = torch.cat([betas, expression], -1).double(), torch.cat([sd, d("expr_dirs")], -1)
    v, j = smplx_ref.lbs(comps, full_pose.double().reshape(betas.shape[0], -1), d("v_template"), dirs, d("posedirs"),
                         d("J_regressor"), bm["parents"].long(), d("lbs_weights"))
    ids = bm["extra_joints_idxs"].long() if extra is None else extra
    j = torch.cat([j, v[:, ids]], 1)
    if kind == "smplx":
        j = torch.cat([j, smplx_ref.vertices2landmarks(v, bm["faces"].long(), bm["lmk_faces_idx"].long(),
                                                      bm["lmk_bary_coords"].double())], 1)
    t = transl.double().unsqueeze(1)
    return v + t, j + t


def _project(x, K):
    return R.perspective_projection(x, K.double())


# |v| <= 8 m; each output is a few dozen fp32 roundings (2^-24 relative) away from the fp64 value: the 486 + 21-term
# blend sums of terms <= 5e-3, the <= 9-deep chain of 3x3 products, the 4-term skinning sum.  30 roundings of 8 m
# = 1.4e-5 m; 3D tolerance 3e-5 m.  Projection: f / z ~ 388 / 5.5 px per metre, times 2 for the x/z, y/z terms.
TOL3 = 3e-5
TOL2 = 2 * 388 / 5.5 * TOL3 + 1e-3


def _body_case(kind, n, seed):
    g = torch.Generator().manual_seed(seed)
    nj = 24 if kind == "smpl" else 55
    pose = torch.randn(n, nj, 3, generator=g) * 0.3
    pose[:, 0] = torch.randn(n, 3, generator=g) * 0.8  # non-zero global orient
    betas = torch.randn(n, 10 if kind == "smpl" else 11, generator=g)
    transl = torch.randn(n, 3, generator=g) * 0.5 + torch.tensor([0.0, 0.0, 6.0])
    f = 388.0
    K = torch.tensor([[f, 0, 224.0], [0, f, 224.0], [0, 0, 1.0]]).repeat(n, 1, 1)
    expr = torch.randn(n, 10, generator=g) * 0.5
    return pose, betas, transl, K, expr


def _err(a, b):
    return (a.double().cpu() - b.double().cpu()).abs().max().item()


@pytest.mark.parametrize("gender", ["male", "female"])
def test_smpl_body_forward_vs_fp64(assets, dev_assets, gender, cuda_device):
    bm = assets[f"smpl_{gender}"]
    pose, betas, transl, K, _ = _body_case("smpl", 5, 1 if gender == "male" else 2)
    out = dev_assets[f"smpl_{gender}"](pose, betas, transl, K)
    v, j = _fp64_body(bm, "smpl", pose, betas, transl)
    assert out["v3d"].shape == (5, 6890, 3) and out["j3d"].shape == (5, 45, 3)
    ev, ej = _err(out["v3d"], v), _err(out["j3d"], j)
    e2 = _err(out["j2d"], _project(j, K))
    print(f"SMPL {gender}: v {ev / TOL3:.3f}, j {ej / TOL3:.3f}, j2d {e2 / TOL2:.3f} of tolerance")
    assert ev <= TOL3 and ej <= TOL3 and e2 <= TOL2
    assert _err(out["transl_pelvis"], j[:, 0]) <= TOL3
    # sensitivity: each plausible mistake falls outside the tolerance
    other = assets["smpl_female" if gender == "male" else "smpl_male"]
    assert _err(out["v3d"], _fp64_body(other, "smpl", pose, betas, transl)[0]) > 10 * TOL3       # genders swapped
    p0 = pose.clone()
    p0[:, 0] = 0
    assert _err(out["v3d"], _fp64_body(bm, "smpl", p0, betas, transl)[0]) > 10 * TOL3          # global orient dropped
    assert _err(out["v3d"], _fp64_body(bm, "smpl", pose, betas, 2 * transl)[0]) > 10 * TOL3    # transl added twice
    rev = bm["extra_joints_idxs"].long().flip(0)
    assert _err(out["j3d"], _fp64_body(bm, "smpl", pose, betas, transl, extra=rev)[1]) > 10 * TOL3  # extras reversed


def test_smplx_body_forward_vs_fp64(assets, dev_assets, cuda_device):
    bm = assets["smplx"]
    pose, betas, transl, K, expr = _body_case("smplx", 4, 3)
    pose[:, 23:25] = torch.randn(4, 2, 3) * 0.3  # eye poses
    out = dev_assets["smplx"](pose, betas, transl, K, expression=expr)
    v, j = _fp64_body(bm, "smplx", pose, betas, transl, expr)
    assert out["v3d"].shape == (4, 10475, 3) and out["j3d"].shape == (4, 127, 3)
    ev, ej, e2 = _err(out["v3d"], v), _err(out["j3d"], j), _err(out["j2d"], _project(j, K))
    print(f"SMPL-X: v {ev / TOL3:.3f}, j {ej / TOL3:.3f}, j2d {e2 / TOL2:.3f} of tolerance")
    assert ev <= TOL3 and ej <= TOL3 and e2 <= TOL2
    p0 = pose.clone()
    p0[:, 23:25] = 0
    assert _err(out["v3d"], _fp64_body(bm, "smplx", p0, betas, transl, expr)[0]) > 10 * TOL3   # eyes dropped
    p0 = pose.clone()
    p0[:, 0] = 0
    assert _err(out["v3d"], _fp64_body(bm, "smplx", p0, betas, transl, expr)[0]) > 10 * TOL3   # global orient dropped


def test_regression_vs_fp64(cuda_device):
    from multihmr_b200 import metrics

    g = torch.Generator().manual_seed(6)
    N, Rr = 700, 17
    A = torch.rand(Rr, N, generator=g) * (torch.rand(Rr, N, generator=g) < 0.05)
    A[4] = 0
    A[4, :40] = torch.randn(40, generator=g)  # a row with negative weights that does not sum to 1
    X = torch.randn(5, N, 3, generator=g) + torch.tensor([0.3, -0.2, 6.0])
    c = torch.randn(5, 3, generator=g) + torch.tensor([0.0, 0.0, 6.0])
    pairs = torch.tensor([[3, 1], [0, 4], [2, 2]], dtype=torch.int32, device=cuda_device)
    n_pairs = torch.tensor([3], dtype=torch.int32, device=cuda_device)
    csr = metrics.CSR(A, cuda_device)
    rows = metrics.H36M_TO_J14
    for side in (0, 1):
        out, _ = metrics.regress(csr, X.to(cuda_device), pairs, n_pairs, side, c.to(cuda_device), rows=rows, root=0)
        for m, pr in enumerate(pairs.tolist()):
            s = pr[side]
            xc = X[s].double() - c[s].double()
            y = A.double() @ xc
            ref = (y - y[[0]])[rows]
            # fp32: <= 3 products per lane + 5 shuffle levels + the centring, each 2^-24 relative of sum |w| |x - c|
            tol = 12 * 2 ** -24 * ((A.double().abs() @ xc.abs())[rows] + (A.double().abs() @ xc.abs())[0]).max().item()
            err = (out[m].double().cpu() - ref).abs().max().item()
            assert err <= tol, (side, m, err, tol)
            wrong = A.double() @ X[s].double() - c[s].double()  # regressing before centring
            assert ((wrong - wrong[[0]])[rows] - out[m].double().cpu()).abs().max().item() > 10 * tol
    # the projection
    K = torch.tensor([[400.0, 0, 200], [0, 380, 210], [0, 0, 1]]).repeat(5, 1, 1)
    out, o2 = metrics.regress(csr, X.to(cuda_device), pairs, n_pairs, 1, None, K=K.to(cuda_device))
    ref = _project((A.double() @ X[pairs[0, 1].item()].double()).unsqueeze(0), K[:1])[0]
    assert (o2[0].double().cpu() - ref).abs().max().item() < 1e-3


def test_new_entries_reject_bad_sizes(dev_assets, cuda_device):
    from multihmr_b200 import _lib, metrics

    csr = dev_assets.j_regressor_h36m
    X = torch.zeros(2, 6890, 3, device=cuda_device)
    pairs = torch.zeros(49, 2, dtype=torch.int32, device=cuda_device)
    n = torch.ones(1, dtype=torch.int32, device=cuda_device)
    with pytest.raises(AssertionError, match="48 pairs"):
        metrics.regress(csr, X, pairs, n, 0)
    with pytest.raises(AssertionError, match="root row"):
        metrics.regress(csr, X, pairs[:2], n, 0, rows=[1, 2], root=17)
    with pytest.raises(AssertionError, match="side"):
        metrics.regress(csr, X, pairs[:2], n, 2)
    body = dev_assets["smpl_male"]
    z = torch.zeros(49, 24, 3)
    with pytest.raises(ValueError):
        body(z, torch.zeros(49, 10), torch.zeros(49, 3), torch.zeros(49, 3, 3))
    lib = _lib.load()
    rc = lib.mhmr_body_forward(body._h, 49, None, None, None, None, None, None, None, None, None, None, None)
    assert rc == -2
    bad = dict(R.eval_assets(0)["smpl_male"])
    bad["parents"] = bad["parents"].clone()
    bad["parents"][5] = 7  # a parent after its child
    with pytest.raises(AssertionError, match="precede"):
        metrics.BodyModel(bad, "smpl", device=cuda_device)
    # SMPL-X with 22 betas: 486 + 22 + 10 coefficient rows exceed the vertex kernel's 512, refused at creation
    with pytest.raises(AssertionError, match="512 rows"):
        metrics.BodyModel(R.eval_assets(0)["smplx"], "smplx", num_betas=22, device=cuda_device)
    with pytest.raises(ValueError, match="rows must lie"):
        metrics.regress(csr, X, pairs[:2], n, 0, rows=[1, 17])


def test_body_create_from_host_arrays(assets, dev_assets, cuda_device):
    """mhmr_body_create takes host or device arrays: a handle built from host (CPU) tensors gives the same meshes as
    one built from device tensors."""
    from multihmr_b200 import _lib
    from multihmr_b200._lib import call, stream

    bm = assets["smplx"]
    sd = torch.cat([bm["shapedirs"], bm["shapedirs_extra"]], -1)[..., :11].float().contiguous()
    f32 = lambda t: t.float().contiguous()
    i32 = lambda t: t.to(torch.int32).contiguous()
    arrs = [f32(bm["v_template"]), sd, f32(bm["expr_dirs"]), f32(bm["posedirs"]), f32(bm["J_regressor"]),
            f32(bm["lbs_weights"]), i32(bm["parents"]), i32(bm["extra_joints_idxs"]),
            i32(bm["faces"].long()[bm["lmk_faces_idx"].long()]), f32(bm["lmk_bary_coords"])]
    h = torch.zeros(1, dtype=torch.int64)
    call("mhmr_body_create", 1, bm["v_template"].shape[0], 11, 8, *arrs, stream(), h)
    h = h.item()
    try:
        pose, betas, transl, K, expr = _body_case("smplx", 3, 5)
        ref = dev_assets["smplx"](pose, betas, transl, K, expression=expr)
        d = lambda t, n: t.to(cuda_device).float().reshape(3, n).contiguous()
        # the inputs stay referenced for the call (a temporary's block could be handed to the next one)
        ins = [d(pose, 165), d(betas, 11), d(expr, 10), d(transl, 3), d(K, 9)]
        out = {k: torch.empty_like(v) for k, v in ref.items()}
        call("mhmr_body_forward", h, 3, *ins, out["v3d"], None, out["j3d"], out["j2d"], out["transl_pelvis"], stream())
        for k in ref:
            assert torch.equal(out[k], ref[k]), k
    finally:
        _lib.load().mhmr_body_destroy(h)


def _stub(cases, dev):
    persons = [[{k: v.to(dev) for k, v in p.items()} for p in c[2]] for c in cases]
    it = iter(persons)
    return lambda x, **kw: next(it)


@pytest.mark.parametrize("dataset", ["3dpw", "ehf", "bedlam"])
def test_evaluate_vs_golden(assets, dev_assets, dataset, cuda_device):
    from multihmr_b200 import metrics

    cases = R.make_cases(dataset, assets)
    res = metrics.evaluate(_stub(cases, cuda_device), [(c[0], c[1]) for c in cases], dev_assets, dataset)
    ev = res["evaluator"]
    with np.load(os.path.join(GOLDEN_DIR, f"eval_{dataset}.npz")) as g:
        gold = {k: g[k] for k in g.files}
    for k in ("precision", "recall", "f1_score"):
        assert res[k] == float(gold[f"meter_{k}"]), k
    # fp32 device body model and regression vs the CPU reference: meshes agree to ~1e-5 m, errors to ~1e-2 mm
    for k in ("pve", "pa_pve", "mpjpe", "pa_mpjpe"):
        got = np.asarray(ev.values.get(k, []), dtype=np.float64)
        ref = gold[f"pairs_{k}"]
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        tol = 2e-2 + 1e-4 * np.abs(ref)
        assert (np.abs(got - ref) <= tol).all(), (k, got, ref)
        assert abs(res[k] - float(gold[f"meter_{k}"])) <= 2e-2 + 1e-4 * abs(float(gold[f"meter_{k}"])), k
    if dataset == "3dpw":
        # J17 instead of J14 falls outside the tolerance
        saved = R.H36M_TO_J14
        try:
            R.H36M_TO_J14 = R.H36M_TO_J17
            _, v17 = R.evaluate(cases, R.shim_models(assets), assets["smplx2smpl"], assets["j_regressor_h36m"],
                                dataset, R.IMG_SIZE)
        finally:
            R.H36M_TO_J14 = saved
        assert np.abs(np.asarray(ev.values["mpjpe"]) - v17["mpjpe"]).max() > 0.1
        # genders swapped in the ground truth changes the errors beyond the tolerance
        sw = [(x, dict(y, smpl_gender_id=3 - y["smpl_gender_id"]), p) for x, y, p in cases]
        res2 = metrics.evaluate(_stub(sw, cuda_device), [(c[0], c[1]) for c in sw], dev_assets, dataset)
        got2 = np.asarray(res2["evaluator"].values["pve"])
        assert got2.shape != gold["pairs_pve"].shape or np.abs(got2 - gold["pairs_pve"]).max() > 0.1


def test_end_to_end_3dpw_shaped_on_engine_predictions(assets, cuda_device):
    """Engine predictions on a golden case; ground truth from the device SMPL-X body model with parameters that
    reproduce the engine's own meshes (global orient inside the chain, transl = pelvis - rest pelvis), moved to SMPL
    by the transfer matrix: PVE / MPJPE below 1 mm and recall 100, through the 3DPW path (SMPL regression, H36M)."""
    import parity_util as pu
    from multihmr_b200 import metrics

    case, sd, bm, x, K, _ = pu.build_inputs("s_224_S_detect")
    m = pu.build_engine(case, sd, bm)
    persons = m(x, K=K, det_thresh=0.3, nms_kernel_size=3)
    assert len(persons) >= 2
    body = metrics.BodyModel(bm, "smplx", num_betas=10, device=cuda_device)
    P = len(persons)
    rv = torch.stack([p["rotvec"] for p in persons]).float()
    zero = torch.zeros(P, 2, 3, device=cuda_device)
    # engine order [root, body 21, lhand 15, rhand 15, jaw] -> smplx order [global, body 21, jaw, eyes, hands]
    full = torch.cat([rv[:, :22], rv[:, 52:53], zero, rv[:, 22:52]], 1)
    betas = torch.stack([p["shape"] for p in persons]).float()
    expr = torch.stack([p["expression"] for p in persons]).float()
    vs = bm["v_template"].double() + torch.einsum("vcl,pl->pvc", torch.cat([bm["shapedirs"], bm["expr_dirs"]], -1).double(),
                                                  torch.cat([betas, expr], 1).double().cpu())
    rest_pelvis = torch.einsum("v,pvc->pc", bm["J_regressor"][0].double(), vs)
    pel = torch.stack([p["transl_pelvis"].reshape(3) for p in persons]).double().cpu()
    transl = (pel - rest_pelvis).float()
    # every image of this case has the same K; all persons of the batch are evaluated at once, as in
    # test_eval_metrics.py::test_evaluator_on_engine_outputs
    assert torch.equal(K[0], K[-1])
    ev = metrics.Evaluator(smplx2smpl=assets["smplx2smpl"], j_regressor_h36m=assets["j_regressor_h36m"],
                           device=cuda_device)
    gt = body(full, betas, transl, K[0].expand(P, 3, 3), expression=expr)
    assert (gt["v3d"] - torch.stack([p["v3d"] for p in persons])).abs().max().item() < 1e-4
    T = metrics.CSR(assets["smplx2smpl"], cuda_device)
    ar = torch.arange(P, dtype=torch.int32, device=cuda_device)
    same = torch.stack([ar, ar], 1).contiguous()
    smpl_v, _ = metrics.regress(T, gt["v3d"], same, torch.tensor([P], dtype=torch.int32, device=cuda_device), 1)
    gt_smpl = dict(j2d=gt["j2d"], v3d=smpl_v, transl_pelvis=gt["transl_pelvis"])
    ev.update(persons, gt_smpl)
    s = ev.summary()
    print(s)
    assert s["recall"] == 100.0 and s["precision"] == 100.0
    assert s["pve"] < 1.0 and s["pa_pve"] < 1.0 and s["mpjpe"] < 1.0 and s["pa_mpjpe"] < 1.0
