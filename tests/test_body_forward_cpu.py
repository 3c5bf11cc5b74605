"""The premises of tests/test_body_forward_gpu.py, checked without a GPU: on the exact bodies every intermediate of the
fp64 forward lies on the 2^-12 grid well inside fp32's 24 bits, so fp32 arithmetic in any order reproduces it (the
fp32 oracle does, bit for bit); the forward bound covers the fp32 oracle on random bodies; and every planted mistake
moves the fp64 reference outside that bound."""
import pytest
import torch

import body_forward_util as bf
import body_grad_util as bg
from oracle import smplx_ref

STEP = 2.0 ** -12


def _on_grid(name, t):
    s = t.double() / STEP
    assert torch.equal(s, s.round()), f"{name} leaves the 2^-12 grid"
    assert s.abs().max().item() < 2.0 ** 24, f"{name} needs more than 24 bits"


def _lbs(bm, pose, comps, nb, dt):
    d = lambda k: torch.as_tensor(bm[k]).to(dt)
    dirs = bg.smplx_dirs(bm, nb, dt, "cpu")
    return smplx_ref.lbs(comps.to(dt), pose.to(dt).reshape(pose.shape[0], -1), d("v_template"), dirs, d("posedirs"),
                         d("J_regressor"), torch.as_tensor(bm["parents"]).long(), d("lbs_weights"))


@pytest.mark.parametrize("kind", ["smpl", "smplx"])
@pytest.mark.parametrize("V", [5, 73, "real"])
def test_exact_bodies_are_exact(kind, V):
    V = bf.V_REAL[kind] if V == "real" else V
    for nb in bf.NB_EDGES[kind]:
        bm = bf.exact_body(kind, V, nb, seed=V + nb)
        pose, betas, transl, K, expr = bf.exact_inputs(kind, 3, nb, seed=nb)
        comps = betas if expr is None else torch.cat([betas, expr], -1)
        dt = torch.float64
        dirs = bg.smplx_dirs(bm, nb, dt, "cpu")
        v_shaped = torch.as_tensor(bm["v_template"]).double() + torch.einsum("bl,mkl->bmk", comps.double(), dirs)
        J = torch.einsum("bik,ji->bjk", v_shaped, torch.as_tensor(bm["J_regressor"]).double())
        rot = smplx_ref.batch_rodrigues(pose.double().reshape(-1, 3))
        assert torch.equal(rot, torch.eye(3, dtype=dt).expand_as(rot)), "R = I exactly at a zero rotation"
        Gt, A = smplx_ref.batch_rigid_transform(rot.view(3, -1, 3, 3), J, torch.as_tensor(bm["parents"]).long())
        assert torch.equal(Gt, J), "the chain telescopes to the rest joints"
        eye = torch.eye(4, dtype=dt).expand_as(A)
        assert torch.equal(A, eye), "every skinning transform is [I | 0]"
        assert torch.equal(torch.as_tensor(bm["lbs_weights"]).double().sum(1), torch.ones(V, dtype=dt))
        ref = bg.raw_outputs(bm, pose.double(), betas.double(), transl.double(), K.double(),
                             None if expr is None else expr.double())
        for name, t in (("v_shaped", v_shaped), ("J", J), ("v3d", ref["v3d"]), ("j3d", ref["j3d"]),
                        ("transl_pelvis", ref["transl_pelvis"])):
            _on_grid(name, t)
        # the fp32 oracle, summing in its own order, gives the same bits
        v64, j64 = _lbs(bm, pose, comps, nb, torch.float64)
        v32, j32 = _lbs(bm, pose, comps, nb, torch.float32)
        assert torch.equal(v32.double(), v64) and torch.equal(j32.double(), j64)


def _fp32_outputs(ref_fn, args):
    return ref_fn(*[None if a is None else a.float() for a in args])


@pytest.mark.parametrize("kind", ["smpl", "smplx"])
def test_bound_covers_fp32_oracle(kind):
    """The fp32 oracle (torch on the CPU, its own summation order) lies inside the bound of the device forward."""
    nb = bf.NB_EDGES[kind][1]
    bm = bf.random_body(kind, nb)
    pose, betas, transl, K, expr = bf.random_inputs(kind, 3, nb)
    ref, tol = bf.raw_reference(bm, pose, betas, transl, K, expr, "cpu")
    got = bg.raw_outputs(bm, pose, betas, transl, K, expr)
    r = bf.worst_ratio(got, ref, tol)
    print(f"{kind} fp32 oracle worst err/tol: " + ", ".join(f"{k} {v:.3f}" for k, v in r.items()))
    assert max(r.values()) <= 1.0, r


def test_bound_covers_fp32_oracle_placed():
    from multihmr_b200 import synth

    bm = synth.make_body_model(1)
    args = bf.placed_inputs(5)
    ref, tol = bf.placed_reference(bm, *args, "cpu")
    got = bg.placed_outputs(bm, *args)
    r = bf.worst_ratio(got, ref, tol)
    print("placed fp32 oracle worst err/tol: " + ", ".join(f"{k} {v:.3f}" for k, v in r.items()))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("kind", ["smpl", "smplx"])
def test_mistakes_leave_the_bound(kind):
    """Each planted mistake moves the fp64 reference by more than the bound somewhere."""
    nb = bf.NB_EDGES[kind][1]
    bm = bf.random_body(kind, nb)
    P = 2 * bf.PB[kind] + 1
    args = bf.random_inputs(kind, P, nb)
    ref, tol = bf.raw_reference(bm, *args, "cpu")
    for name in bf.MISTAKES:
        if name == "second_pass":
            wrong = bf.second_pass_from_first(ref, bf.PB[kind])
        else:
            m = bf.mistaken_inputs(name, kind, bm, args)
            if m is None:
                continue
            wrong, _ = bf.raw_reference(m[0], *m[1], "cpu")
        r = max(bf.worst_ratio(wrong, ref, tol).values())
        print(f"{kind} {name}: {r:.1f}")
        assert r > 1.0, name
