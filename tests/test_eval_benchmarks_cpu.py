"""The 3DPW / EHF / BEDLAM evaluation protocols on the CPU: the restatement oracle/eval_bench_ref.py against the goldens
of the reference's own Trainer.evaluate (oracle/make_golden_eval.py), the SMPL restatement against a float64
evaluation of the SMPL formula, the chumpy-free pickle loader and the CSR build of the regressors."""
import os
import pickle
import sys
import types

import numpy as np
import pytest
import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def assets():
    from oracle import eval_bench_ref

    return eval_bench_ref.eval_assets(0)


@pytest.mark.parametrize("dataset", ["3dpw", "ehf", "bedlam"])
def test_restatement_equals_golden(assets, dataset):
    from oracle import eval_bench_ref as R

    cases = R.make_cases(dataset, assets)
    meters, vals = R.evaluate(cases, R.shim_models(assets), assets["smplx2smpl"], assets["j_regressor_h36m"], dataset,
                              R.IMG_SIZE)
    with np.load(os.path.join(GOLDEN_DIR, f"eval_{dataset}.npz")) as g:
        for k in R.METERS:
            # the restatement's sparse SMPL-X -> SMPL product rounds differently from the reference's dense one
            assert abs(meters[k] - float(g[f"meter_{k}"])) <= 1e-4, (k, meters[k], float(g[f"meter_{k}"]))
        for k in ("pve", "pa_pve", "mpjpe", "pa_mpjpe"):
            assert vals[k].shape == g[f"pairs_{k}"].shape, k
            assert np.abs(vals[k] - g[f"pairs_{k}"]).max(initial=0.0) <= 1e-4, k
    if dataset == "3dpw":
        assert vals["mpjpe"].size > 0
    else:
        assert vals["mpjpe"].size == 0


def _rodrigues64(r):
    ang = np.linalg.norm(r + 1e-8)
    k = r / ang
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * Kx @ Kx


def smpl_fp64(bm, pose, betas, transl):
    """The SMPL formula in float64 numpy, written out joint by joint: v_shaped = T + S b, J = Jr v_shaped,
    v_posed = v_shaped + P (R_j - I), G_j = G_parent [R_j | J_j - J_parent], v = sum_j w_j G_j [v_posed - J_j],
    joints = [G_j translation | v[extra ids]], all + transl."""
    f = lambda k: bm[k].double().numpy()
    V = f("v_template").shape[0]
    vs = f("v_template") + np.einsum("vcl,l->vc", f("shapedirs")[..., :10], betas)
    J = f("J_regressor") @ vs
    Rs = [_rodrigues64(pose[j]) for j in range(24)]
    feat = np.concatenate([(Rs[j] - np.eye(3)).reshape(-1) for j in range(1, 24)])
    vp = vs + (feat @ f("posedirs")).reshape(V, 3)
    par = bm["parents"].tolist()
    G = []
    for j in range(24):
        T = np.eye(4)
        T[:3, :3] = Rs[j]
        T[:3, 3] = J[j] - (J[par[j]] if j else 0)
        G.append(T if j == 0 else G[par[j]] @ T)
    A = np.stack([g @ np.block([[np.eye(3), -J[j][:, None]], [np.zeros((1, 3)), np.ones((1, 1))]])
                  for j, g in enumerate(G)])
    Tv = np.einsum("vj,jab->vab", f("lbs_weights"), A)
    v = np.einsum("vab,vb->va", Tv[:, :3, :3], vp) + Tv[:, :3, 3]
    joints = np.concatenate([np.stack([g[:3, 3] for g in G]), v[bm["extra_joints_idxs"].numpy()]])
    return v + transl, joints + transl


def test_smpl_restatement_vs_float64_formula(assets):
    from oracle import eval_bench_ref as R

    g = torch.Generator().manual_seed(3)
    for gender in ("male", "female"):
        bm = assets[f"smpl_{gender}"]
        pose = torch.randn(2, 24, 3, generator=g) * 0.4
        betas = torch.randn(2, 10, generator=g)
        transl = torch.randn(2, 3, generator=g) + torch.tensor([0.0, 0.0, 6.0])
        out = R.SMPLShim(bm)(global_orient=pose[:, 0], body_pose=pose[:, 1:], betas=betas, transl=transl)
        assert out.vertices.shape == (2, 6890, 3) and out.joints.shape == (2, 45, 3)
        for i in range(2):
            v, j = smpl_fp64(bm, pose[i].double().numpy(), betas[i].double().numpy(), transl[i].double().numpy())
            # fp32 restatement: |v| <= 8 m, a few dozen roundings of 2^-24 relative each
            assert np.abs(out.vertices[i].double().numpy() - v).max() < 2e-5
            assert np.abs(out.joints[i].double().numpy() - j).max() < 2e-5


def _pickle_with_fake_module(obj_factory, module, name):
    """Pickle an object whose class claims to live at module.name (no such package needs to be installed)."""
    mod = types.ModuleType(module)
    cls = type(name, (), {"__module__": module})
    setattr(mod, name, cls)
    parts = module.split(".")
    saved = {m: sys.modules.get(m) for m in [".".join(parts[: i + 1]) for i in range(len(parts))]}
    for i in range(len(parts)):
        sys.modules.setdefault(".".join(parts[: i + 1]), types.ModuleType(".".join(parts[: i + 1])))
    sys.modules[module] = mod
    try:
        return pickle.dumps(obj_factory(cls), protocol=2)
    finally:
        for m, v in saved.items():
            if v is None:
                sys.modules.pop(m, None)
            else:
                sys.modules[m] = v


def test_chumpy_free_loader(tmp_path):
    from multihmr_b200 import api

    rng = np.random.default_rng(0)
    sd = rng.normal(size=(6, 3, 10))

    def make(Ch):
        ch = Ch()
        ch.__dict__.update(x=sd, _dirty_vars=set())  # what chumpy.ch.Ch pickles: its value in 'x'
        return {"shapedirs": ch, "v_template": rng.normal(size=(6, 3)), "kintree_table": np.zeros((2, 24), np.int64)}

    p = tmp_path / "smpl.pkl"
    p.write_bytes(_pickle_with_fake_module(make, "chumpy.ch", "Ch"))
    d = api.load_body_model_pickle(str(p))
    assert isinstance(d["shapedirs"], np.ndarray) and np.array_equal(d["shapedirs"], sd)
    assert d["v_template"].shape == (6, 3)

    bad = tmp_path / "bad.pkl"
    bad.write_bytes(_pickle_with_fake_module(lambda C: {"x": C()}, "evil.payload", "Thing"))
    with pytest.raises(pickle.UnpicklingError):
        api.load_body_model_pickle(str(bad))

    class Reduce:
        def __reduce__(self):
            return (os.system, ("true",))

    bad.write_bytes(pickle.dumps({"matrix": Reduce()}, protocol=2))
    with pytest.raises(pickle.UnpicklingError):
        api.load_body_model_pickle(str(bad))


def test_csr_build_reproduces_dense_product():
    from multihmr_b200 import metrics, synth

    g = torch.Generator().manual_seed(4)
    A = torch.randn(17, 500, generator=g) * (torch.rand(17, 500, generator=g) < 0.1)
    A[3] = 0.0  # an empty row
    A[5, 7] = -0.75  # negative weights are kept
    X = torch.randn(500, 3, generator=g, dtype=torch.float64)
    csr = metrics.CSR(A, device="cpu")
    assert csr.shape == (17, 500) and csr.rowptr.dtype == torch.int32 and csr.col.dtype == torch.int32
    assert int(csr.rowptr[-1]) == int((A != 0).sum())
    assert torch.equal(csr.to_dense(), A)
    assert torch.allclose(csr.to_dense().double() @ X, A.double() @ X, rtol=0, atol=1e-12)
    T = synth.make_smplx2smpl(0)
    ct = metrics.CSR(T, device="cpu")
    assert ct.shape == (6890, 10475) and int(ct.rowptr[-1]) == 3 * 6890
    assert torch.allclose(ct.to_dense().sum(1), torch.ones(6890), atol=1e-6)
    H = synth.make_j_regressor_h36m(0)
    assert (H >= 0).all() and torch.allclose(H.sum(1), torch.ones(17), atol=1e-6)
