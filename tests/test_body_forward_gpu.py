"""Forward of the body models on the device (mhmr_body_forward for SMPL / SMPL-X, mhmr_smplx_forward for the engine's
placed SMPL-X layer) against the fp64 reference (body_grad_util.raw_outputs / placed_outputs), across the vertex
kernel's edges: vertex tiles of 72 (full, single partial, one past), person passes of 8 (SMPL) / 16 (SMPL-X) up to
80 persons, and coefficient row counts KT = 9 (NJ - 1) + num_betas (+ 10) from 208 to the 512-row limit.

  * Exact bodies (body_forward_util.exact_body): v3d, j3d and transl_pelvis equal the reference bit for bit; v2d / j2d
    within the rounding of the projection.
  * Random bodies: every output within the bound derived from the kernels' accumulation lengths
    (body_forward_util.forward_bound); each planted mistake of the reference falls outside it.
  * Invariants: repeated calls and batch position (pass, capacity) change no bit; a NaN person leaves the others'
    bits alone; v2d is the projection of the call's own v3d.
Every output lands in a canvas with SENTINEL guard bands before and after the P persons (up to the handle's
capacity), which must come back untouched."""
import math

import pytest
import torch

import body_forward_util as bf
import parity_util as pu
from fp64_util import SENTINEL

pytestmark = pytest.mark.gpu
GUARD = 64
CAP = 80
V_SWEEP = (5, 71, 72, 73, 144, 145, "real")


def _stream():
    from ctypes import c_void_p

    return c_void_p(torch.cuda.current_stream().cuda_stream)


def _canvases(shapes, P, cap, dev):
    """{name: (flat canvas, [P, *shape] view)}: GUARD sentinels, cap persons' rows of sentinels, GUARD sentinels."""
    out = {}
    for k, s in shapes.items():
        n = math.prod(s)
        buf = torch.full((2 * GUARD + cap * n,), SENTINEL, device=dev)
        out[k] = (buf, buf[GUARD:GUARD + P * n].view(P, *s))
    return out


def _check_guards(cv, P):
    for k, (buf, view) in cv.items():
        n = view[0].numel() if P else 0
        assert (buf[:GUARD] == SENTINEL).all(), f"{k}: write before the first person"
        assert (buf[GUARD + P * n:] == SENTINEL).all(), f"{k}: write past person {P - 1} (or past the last vertex)"


def _body(bm, kind, nb, dev, cap=CAP):
    from multihmr_b200 import metrics

    return metrics.BodyModel(bm, kind, nb, cap, dev)


def raw_forward(body, pose, betas, transl, K, expr, with_v2d=True):
    """mhmr_body_forward into sentinel canvases; returns the outputs (guards checked)."""
    from ctypes import c_int

    from multihmr_b200._lib import check, ptr

    P = int(betas.shape[0])
    fp, b, tr, Kd, ex = body._inputs(pose, betas, transl, K, expr)
    V, J = body.num_verts, body.num_joints
    shapes = dict(v3d=(V, 3), v2d=(V, 2), j3d=(J, 3), j2d=(J, 2), transl_pelvis=(3,))
    if not with_v2d:
        shapes.pop("v2d")
    cv = _canvases(shapes, P, body.max_persons, body.device)
    o = lambda k: ptr(cv[k][1]) if k in cv else None
    check(body._lib.mhmr_body_forward(body._h, c_int(P), ptr(fp), ptr(b), ptr(ex), ptr(tr), ptr(Kd), o("v3d"),
                                      o("v2d"), o("j3d"), o("j2d"), o("transl_pelvis"), _stream()),
          "mhmr_body_forward")
    torch.cuda.synchronize()
    _check_guards(cv, P)
    return {k: v[1] for k, v in cv.items()}


def placed_forward(m, rotvec, shape, loc, dist, K, expr):
    from ctypes import c_int

    from multihmr_b200._lib import check, ptr

    m.finalize()
    x = m._smplx_inputs(rotvec, shape, loc, dist, K, expr)
    P, V = int(rotvec.shape[0]), m.num_verts
    shapes = dict(v3d=(V, 3), v2d=(V, 2), j3d=(127, 3), j2d=(127, 2), transl=(3,), transl_pelvis=(3,))
    cv = _canvases(shapes, P, m.max_persons, m.device)
    check(m._lib.mhmr_smplx_forward(m._handle, c_int(P), ptr(x[0]), ptr(x[1]), ptr(x[5]), ptr(x[2]), ptr(x[3]),
                                    ptr(x[4]), *[ptr(cv[k][1]) for k in shapes], _stream()), "mhmr_smplx_forward")
    torch.cuda.synchronize()
    _check_guards(cv, P)
    return {k: v[1] for k, v in cv.items()}


def _report(label, r):
    print(f"{label} worst err/tol: " + ", ".join(f"{k} {v:.3f}" for k, v in r.items()))


# ------------------------------------------------------------------------------------------------ 1. exact bodies
@pytest.mark.parametrize("kind", ["smpl", "smplx"])
@pytest.mark.parametrize("V", V_SWEEP)
def test_exact_bodies_bit_for_bit(kind, V, cuda_device):
    V = bf.V_REAL[kind] if V == "real" else V
    for nb in bf.NB_EDGES[kind]:
        bm = bf.exact_body(kind, V, nb, seed=V + nb)
        body = _body(bm, kind, nb, cuda_device)
        worst2 = 0.0
        for P in bf.persons_sweep(kind):
            pose, betas, transl, K, expr = bf.exact_inputs(kind, P, nb, seed=P)
            got = raw_forward(body, pose, betas, transl, K, expr)
            ref, _ = bf.raw_reference(bm, pose, betas, transl, K, expr, cuda_device)
            for k in ("v3d", "j3d", "transl_pelvis"):
                bad = got[k].double() != ref[k]
                assert not bad.any(), (f"{kind} V={V} nb={nb} P={P} {k}: {int(bad.sum())} elements differ, first at "
                                       f"{bad.nonzero()[0].tolist()}")
            for k, src in (("v2d", "v3d"), ("j2d", "j3d")):
                tol = bf.projection_bound(ref[src], K.to(cuda_device), torch.zeros_like(ref[src][..., 0]))
                r = ((got[k].double() - ref[k]).abs() / tol).max().item()
                worst2 = max(worst2, r)
                assert r <= 1.0, (kind, V, nb, P, k, r)
        print(f"exact {kind} V={V} nb={nb} (KT={9 * (bf.NJ[kind] - 1) + nb + (10 if kind == 'smplx' else 0)}): "
              f"3-D outputs bit for bit at P={bf.persons_sweep(kind)}, 2-D worst err/tol {worst2:.3f}")
        del body


# ------------------------------------------------------------------------------------------------ 2. random bodies
@pytest.fixture(scope="module")
def random_bodies(cuda_device):
    out = {}
    for kind in ("smpl", "smplx"):
        for nb in bf.NB_EDGES[kind]:
            bm = bf.random_body(kind, nb)
            out[kind, nb] = (bm, _body(bm, kind, nb, cuda_device))
    return out


@pytest.mark.parametrize("kind", ["smpl", "smplx"])
@pytest.mark.parametrize("nb_i", [0, 1, 2])
def test_raw_forward_vs_fp64(random_bodies, kind, nb_i, cuda_device):
    nb = bf.NB_EDGES[kind][nb_i]
    bm, body = random_bodies[kind, nb]
    for P in bf.persons_sweep(kind):
        args = bf.random_inputs(kind, P, nb, seed=P + nb)
        got = raw_forward(body, *args)
        ref, tol = bf.raw_reference(bm, *args, cuda_device)
        r = bf.worst_ratio(got, ref, tol)
        _report(f"{kind} nb={nb} P={P}", r)
        assert all(torch.isfinite(t).all() for t in got.values())
        assert max(r.values()) <= 1.0, r
        # v2d is the projection of the call's own v3d
        own = bf.project(got["v3d"].double(), args[3])
        tol2 = bf.projection_bound(got["v3d"].double(), args[3], torch.zeros_like(own[..., 0]))
        assert ((got["v2d"].double() - own).abs() / tol2).max().item() <= 1.0


@pytest.mark.parametrize("kind", ["smpl", "smplx"])
def test_raw_forward_sensitivity(random_bodies, kind, cuda_device):
    nb = bf.NB_EDGES[kind][1]
    bm, body = random_bodies[kind, nb]
    P = 2 * bf.PB[kind] + 1
    args = bf.random_inputs(kind, P, nb, seed=77)
    got = raw_forward(body, *args)
    ref, tol = bf.raw_reference(bm, *args, cuda_device)
    assert max(bf.worst_ratio(got, ref, tol).values()) <= 1.0
    for name in bf.MISTAKES:
        if name == "second_pass":
            wrong = bf.second_pass_from_first(ref, bf.PB[kind])
        else:
            mis = bf.mistaken_inputs(name, kind, bm, args)
            if mis is None:
                continue
            wrong, _ = bf.raw_reference(mis[0], *mis[1], cuda_device)
        r = max(bf.worst_ratio(got, wrong, tol).values())
        print(f"{kind} mistaken reference {name}: err/tol {r:.1f}")
        assert r > 1.0, name


@pytest.fixture(scope="module")
def engine(cuda_device):
    case, sd, bm, x, K, _ = pu.build_inputs("s_224_S_forced")
    return pu.build_engine(case, sd, bm, max_persons=CAP), bm


@pytest.mark.parametrize("P", [1, 15, 16, 17, 33, 40, 80])
def test_placed_forward_vs_fp64(engine, P, cuda_device):
    m, bm = engine
    args = bf.placed_inputs(P, seed=P)
    got = placed_forward(m, *args)
    ref, tol = bf.placed_reference(bm, *args, cuda_device)
    r = bf.worst_ratio(got, ref, tol)
    _report(f"placed P={P}", r)
    assert max(r.values()) <= 1.0, r
    if P >= 17:
        for name in bf.MISTAKES:
            if name == "second_pass":
                wrong = bf.second_pass_from_first(ref, 16)
            else:
                mis = bf.mistaken_inputs(name, "smplx", bm, args)
                wrong, _ = bf.placed_reference(mis[0], *mis[1], cuda_device)
            rw = max(bf.worst_ratio(got, wrong, tol).values())
            print(f"placed P={P} mistaken reference {name}: err/tol {rw:.1f}")
            assert rw > 1.0, name


# ------------------------------------------------------------------------------------------------ 3. invariants
def _same(a, b, idx=None):
    return all(torch.equal(a[k] if idx is None else a[k][idx], b[k]) for k in b)


@pytest.mark.parametrize("kind", ["smpl", "smplx"])
def test_repeat_position_and_nan_isolation(random_bodies, kind, cuda_device):
    nb = bf.NB_EDGES[kind][1]
    bm, body = random_bodies[kind, nb]
    small = _body(bm, kind, nb, cuda_device, cap=1)
    args = bf.random_inputs(kind, CAP, nb, seed=5)
    a = raw_forward(body, *args)
    assert _same(a, raw_forward(body, *args)), "repeated call"
    pb = bf.PB[kind]
    sub = lambda i: [None if t is None else t[i:i + 1] for t in args]
    for i in sorted({0, pb - 1, pb, pb + 1, 2 * pb, 40, CAP - 1}):
        assert _same(a, raw_forward(body, *sub(i)), slice(i, i + 1)), f"person {i} alone (capacity {CAP})"
        assert _same(a, raw_forward(small, *sub(i)), slice(i, i + 1)), f"person {i} alone (capacity 1)"
    bad = [None if t is None else t.clone() for t in args]
    for i in (pb, CAP - 1):
        bad[0][i] = float("nan")
    b = raw_forward(body, *bad)
    keep = torch.ones(CAP, dtype=torch.bool, device=cuda_device)
    keep[[pb, CAP - 1]] = False
    assert all(torch.equal(a[k][keep], b[k][keep]) for k in a), "a NaN person changed another person's outputs"
    assert not torch.isfinite(b["v3d"][pb]).any()


def test_placed_repeat_and_position(engine, cuda_device):
    m, _ = engine
    args = bf.placed_inputs(CAP, seed=9)
    a = placed_forward(m, *args)
    assert _same(a, placed_forward(m, *args))
    for i in (0, 15, 16, 17, 33, CAP - 1):
        one = [t[i:i + 1] for t in args]
        assert _same(a, placed_forward(m, *one), slice(i, i + 1)), f"person {i} alone"
