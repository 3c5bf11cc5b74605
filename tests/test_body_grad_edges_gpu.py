"""Backward of the body models (mhmr_body_backward, mhmr_smplx_backward) against fp64 autograd at the gradient
kernels' own edges: vertex tiles of body_grad_util.GTV = 80 (a one-vertex tile, V a multiple of 80, the real bodies'
partial last tiles), coefficient rows KT = 208 / 217 / 239 (SMPL, up to the beta[32] limit) and 497 / 507 / 512 (SMPL-X,
up to kKTMax), person passes of GPB = 16 (P = 15, 16, 17, 33 and a capacity of 80), and the rotation-derivative
branches (the Taylor switch at a = 0.5, the placed root's first-order form below 1e-6 rad, |r| = pi and beyond).

Every gradient lands in a canvas with SENTINEL guard bands sized to the handle's capacity, which must come back
untouched.  Exact bodies at zero pose give all four gradients bit for bit.  Otherwise each element must lie within
body_grad_util.tolerance (the per-person bound) and within body_grad_util.backward_bound (the per-element
running-error bound); each planted mistake of body_grad_util.body lies more than twice the latter away.  Invariants: bitwise repeat, batch position across a pass boundary, a call with P = 17
after one with P = 80, NaN isolation, and P = 0 writing nothing."""
import math

import pytest
import torch

import body_forward_util as bf
import body_grad_util as bg
import parity_util as pu
from fp64_util import SENTINEL

pytestmark = pytest.mark.gpu
GUARD = 64
CAP = 80
PERSONS = (1, 15, 16, 17, 33)
V_SMALL = (5, 79, 80, 81, 160, 161)


def _canvas(shape, P, cap, dev):
    n = math.prod(shape)
    buf = torch.full((2 * GUARD + cap * n,), SENTINEL, device=dev)
    return buf, buf[GUARD:GUARD + P * n].view(P, *shape)


def _check(buf, view, P, name):
    n = view[0].numel() if P else 0
    assert (buf[:GUARD] == SENTINEL).all(), f"{name}: write before the first person"
    assert (buf[GUARD + P * n:] == SENTINEL).all(), f"{name}: write past person {P - 1}"


def raw_backward(body, args, up):
    """mhmr_body_backward into sentinel canvases: [d_full_pose, d_betas, d_transl(, d_expression)]."""
    from multihmr_b200._lib import call, stream

    pose, betas, transl, K, expr = args
    P = int(betas.shape[0])
    fp, b, tr, Kd, ex = body._inputs(pose, betas, transl, K, expr)
    shapes = dict(fp=(body.num_pose_joints * 3,), b=(body.num_betas,), tr=(3,), ex=(10,))
    if ex is None:
        shapes.pop("ex")
    cv = {k: _canvas(s, P, body.max_persons, body.device) for k, s in shapes.items()}
    g = lambda k: None if up.get(k) is None else up[k].to(body.device, torch.float32).contiguous()
    call("mhmr_body_backward", body._h, P, fp, b, ex, tr, Kd, g("v3d"), g("v2d"), g("j3d"), g("j2d"),
         g("transl_pelvis"), cv["fp"][1], cv["b"][1], cv["ex"][1] if "ex" in cv else None, cv["tr"][1], stream())
    torch.cuda.synchronize()
    for k, (buf, view) in cv.items():
        _check(buf, view, P, k)
    return [cv[k][1] for k in ("fp", "b", "tr", "ex") if k in cv]


def raw_reference(bm, args, up, dev, **mistake):
    """fp64 autograd of bg.raw_outputs: (gradients, gradients under |upstream|) in the order of raw_backward."""
    pose, betas, transl, K, expr = args
    d = lambda t: None if t is None else t.to(dev, torch.float64).requires_grad_()
    ins = [d(pose), d(betas), d(transl)] + ([d(expr)] if expr is not None else [])
    out = bg.raw_outputs(bm, ins[0], ins[1], ins[2], K.to(dev, torch.float64), ins[3] if expr is not None else None,
                         **mistake)
    up = {k: v.to(dev) for k, v in up.items()}
    return bg.vjp(out, up, ins), bg.vjp(out, {k: v.abs() for k, v in up.items()}, ins)


RAW_NAMES = ("d_full_pose", "d_betas", "d_transl", "d_expression")


def raw_ratios(bm, args, up, got, dev):
    """worst err / bg.tolerance and err / bg.backward_bound over the gradients."""
    ref, ref_abs = raw_reference(bm, args, up, dev)
    NJ = args[0].shape[1]
    n = bg.n_seq(torch.as_tensor(bm["v_template"]).shape[0], NJ)
    f64 = [None if a is None else a.to(dev, torch.float64) for a in args]
    with torch.no_grad():
        _, bound = bg.backward_bound(bm, f64, {k: v.to(dev) for k, v in up.items()})
    old = new = 0.0
    for a, r, ra, name in zip(got, ref, ref_abs, RAW_NAMES):
        err = (a.double().reshape(r.shape) - r).abs()
        old = max(old, (err / bg.tolerance(r, ra, n)).max().item())
        new = max(new, (err / bound[name].reshape(r.shape)).max().item())
    return old, new


def _upstreams(P, V, J, g, outs=("all", "v3d", "j3d", "j2d", "transl_pelvis")):
    for which in outs:
        up = bg.upstream(P, V, J, g, which)
        up.pop("transl", None)
        yield which, up


def _body(bm, kind, nb, dev, cap=CAP):
    from multihmr_b200 import metrics

    return metrics.BodyModel(bm, kind, nb, cap, dev)


_njout = bg.num_output_joints


# ------------------------------------------------------------------------------------------------ 1. tile edges
@pytest.mark.parametrize("kind", ["smpl", "smplx"])
@pytest.mark.parametrize("V", V_SMALL)
def test_small_bodies_at_tile_edges(kind, V, cuda_device):
    """exact_body's tables (one-vertex last tile at V = 81 / 161, whole tiles at 80 / 160) with random poses and
    upstream gradients, every nb edge and P across the pass boundary."""
    report = []
    for nb in bf.NB_EDGES[kind]:
        bm = bf.exact_body(kind, V, nb, seed=V + nb)
        body = _body(bm, kind, nb, cuda_device)
        g = torch.Generator().manual_seed(V * 7 + nb)
        worst = [0.0, 0.0]
        for P in PERSONS:
            args = bf.random_inputs(kind, P, nb, seed=P + nb)
            for which, up in _upstreams(P, V, _njout(kind), g, ("all", "v3d", "j2d")):
                got = raw_backward(body, args, up)
                assert all(torch.isfinite(t).all() for t in got), (nb, P, which)
                old, new = raw_ratios(bm, args, up, got, cuda_device)
                worst = [max(worst[0], old), max(worst[1], new)]
                assert old <= 1.0 and new <= 1.0, (kind, V, nb, P, which, old, new)
        report.append(f"nb={nb} {worst[0]:.3f} / {worst[1]:.4f}")
        del body
    print(f"{kind} V={V} worst err/tol (per-person / per-element): " + ", ".join(report))


# ------------------------------------------------------------------------------------------------ 0. exact bodies
def _exact_case(kind, V, nb, P, bm, seed):
    """Zero pose, betas / expressions in {-1, 0, 1}, and integer upstream gradients: v3d on 6 entries (+-1), j3d on 3
    entries (+-1) among the body and vertex-picked joints and (SMPL-X) one landmark entry (+-4, so its barycentric
    1/2, 1/4 shares stay integers), transl_pelvis on one coordinate (+-1)."""
    g = torch.Generator().manual_seed(seed)
    pose, _, transl, K, _ = bf.exact_inputs(kind, P, nb, seed)
    betas = torch.randint(-1, 2, (P, nb), generator=g).float()
    expr = torch.randint(-1, 2, (P, 10), generator=g).float() if kind == "smplx" else None
    NJ, J = bf.NJ[kind], bg.num_output_joints(kind)
    sign = lambda *s: torch.randint(0, 2, s, generator=g).float() * 2 - 1
    up = dict(v3d=torch.zeros(P, V, 3), j3d=torch.zeros(P, J, 3), transl_pelvis=torch.zeros(P, 3))
    for p in range(P):
        for _ in range(6):
            up["v3d"][p, torch.randint(0, V, (1,), generator=g), torch.randint(0, 3, (1,), generator=g)] += sign(1)
        for _ in range(3):
            up["j3d"][p, torch.randint(0, NJ + 21, (1,), generator=g), torch.randint(0, 3, (1,), generator=g)] += sign(1)
        if kind == "smplx":
            up["j3d"][p, torch.randint(NJ + 21, J, (1,), generator=g), torch.randint(0, 3, (1,), generator=g)] += 4 * sign(1)
        up["transl_pelvis"][p, torch.randint(0, 3, (1,), generator=g)] = sign(1)
    return (pose, betas, transl, K, expr), up


def _exact_precondition(bm, kind, args, up):
    """G X (2 + 2 depth) < 2^9 per person, with G the person's sum of |upstream| after the vertex -> joint scatter, X
    the largest |v_shaped| or |J| and depth the chain's.  Why it suffices: at zero pose every rotation is I and every
    skinning transform [I | 0] exactly, the tables sit on 2^-10 (J_regressor 2^-2, weights 2^-3, v_shaped and J on
    2^-10 / 2^-12) and the scattered output gradient g_o is an integer, so every product of the backward is a multiple
    of 2^-15 (g_A_t J, g_G_t t_j, Jdirs g_J; g_cf and g_A_R are coarser).  The largest partial sum is the root's g_G_R,
    sum_j |g_A_R,j| + |g_A_t,j| |J_j| + |g_G_t,j| |t_j| <= G X + G X + depth G 2 X; below 2^-15 2^24 = 2^9 every partial
    sum, in any order, is exact in fp32.  At r = 0 rotvec_grad returns <g, K(e_k)> exactly (A = 1, K(r) = 0), and the
    fp64 reference is (sin a / a) <g, K(e_k)>, a = sqrt(3) 1e-8, which rounds to the same fp32 value.  So d_full_pose,
    d_betas, d_expression and d_transl all equal the fp64 reference rounded to fp32."""
    pose, betas, transl, K, expr = args
    V = torch.as_tensor(bm["v_template"]).shape[0]
    NJ = bf.NJ[kind]
    M, _ = bg.scatter_table(bm, NJ, bg.num_output_joints(kind), V, torch.float64, "cpu")
    go = up["v3d"].double() + torch.einsum("vj,pjc->pvc", M, up["j3d"].double())
    G = go.abs().sum((1, 2)) + up["j3d"][:, :NJ].double().abs().sum((1, 2)) + up["transl_pelvis"].double().abs().sum(1)
    comps = betas if expr is None else torch.cat([betas, expr], -1)
    dirs = bg.smplx_dirs(bm, betas.shape[1], torch.float64, "cpu")
    vs = torch.as_tensor(bm["v_template"]).double() + torch.einsum("bl,mkl->bmk", comps.double(), dirs)
    Jx = torch.einsum("bik,ji->bjk", vs, torch.as_tensor(bm["J_regressor"]).double())
    X = torch.maximum(vs.abs().amax((1, 2)), Jx.abs().amax((1, 2)))
    par = bf.parents(kind)
    depth = [0] * NJ
    for j, p in enumerate(par):
        depth[j] = 0 if p < 0 else depth[p] + 1
    worst = (G * X * (2 + 2 * max(depth))).max().item()
    assert worst < 2 ** 9, worst
    return worst


@pytest.mark.parametrize("kind", ["smpl", "smplx"])
@pytest.mark.parametrize("V", V_SMALL)
def test_exact_bodies_bit_for_bit(kind, V, cuda_device):
    """Every gradient equals the fp64 reference rounded to fp32, bit for bit (argument: _exact_precondition), at
    every nb edge and P across the pass boundary."""
    for nb in bf.NB_EDGES[kind]:
        bm = bf.exact_body(kind, V, nb, seed=V + nb)
        body = _body(bm, kind, nb, cuda_device)
        margin = 0.0
        for P in PERSONS:
            args, up = _exact_case(kind, V, nb, P, bm, seed=100 * V + 10 * nb + P)
            margin = max(margin, _exact_precondition(bm, kind, args, up))
            got = raw_backward(body, args, up)
            ref, _ = raw_reference(bm, args, up, cuda_device)
            for a, r, name in zip(got, ref, RAW_NAMES):
                bad = a.reshape(r.shape) != r.float()
                assert not bad.any(), (f"{kind} V={V} nb={nb} P={P} {name}: {int(bad.sum())} elements differ, first "
                                       f"at {bad.nonzero()[0].tolist()}")
        print(f"exact {kind} V={V} nb={nb}: all four gradients bit for bit at P={PERSONS} "
              f"(largest partial-sum bound {margin:.0f} < 512)")
        del body


# ------------------------------------------------------------------------------------------------ 2. real bodies
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
def test_real_bodies_at_row_and_pass_edges(random_bodies, kind, nb_i, cuda_device):
    nb = bf.NB_EDGES[kind][nb_i]
    bm, body = random_bodies[kind, nb]
    g = torch.Generator().manual_seed(31 + nb)
    for P in PERSONS + (CAP,):
        args = bf.random_inputs(kind, P, nb, seed=P + nb)
        worst = {}
        for which, up in _upstreams(P, body.num_verts, body.num_joints, g,
                                    ("all", "v3d", "j2d") if P == CAP else ("all", "v3d", "j3d", "j2d", "transl_pelvis")):
            got = raw_backward(body, args, up)
            old, new = raw_ratios(bm, args, up, got, cuda_device)
            worst[which] = (old, new)
            assert old <= 1.0 and new <= 1.0, (kind, nb, P, which, old, new)
        print(f"{kind} nb={nb} P={P} worst err/tol (per-person / per-element): "
              + ", ".join(f"{k} {a:.3f}/{b:.4f}" for k, (a, b) in worst.items()))


# ------------------------------------------------------------------------------------------------ 3. rotation branches
BODY_ANGLES = (0.0, 1e-8, 1e-4, 0.5 * (1 - 2.0 ** -20), 0.5 * (1 + 2.0 ** -20), math.pi - 1e-3, math.pi, 4.0)


@pytest.mark.parametrize("kind", ["smpl", "smplx"])
def test_rotation_branches(random_bodies, kind, cuda_device):
    """Every body joint of person p at |r| = BODY_ANGLES[p] (random axes), the Taylor switch of rotvec_grad from both
    sides at 2^-20 relative (the fp32 angle is within a few u, so both sides stay on theirs)."""
    nb = bf.NB_EDGES[kind][1]
    bm, body = random_bodies[kind, nb]
    P = len(BODY_ANGLES)
    args = list(bf.random_inputs(kind, P, nb, seed=3))
    g = torch.Generator().manual_seed(17)
    axis = torch.randn(P, bf.NJ[kind], 3, generator=g, dtype=torch.float64)
    axis = axis / axis.norm(dim=-1, keepdim=True)
    args[0] = (axis * torch.tensor(BODY_ANGLES, dtype=torch.float64).view(P, 1, 1)).float()
    for which, up in _upstreams(P, body.num_verts, body.num_joints, g):
        got = raw_backward(body, args, up)
        old, new = raw_ratios(bm, args, up, got, cuda_device)
        print(f"{kind} rotation branches, upstream {which}: worst err/tol {old:.3f} / {new:.4f}")
        assert old <= 1.0 and new <= 1.0, (which, old, new)


@pytest.fixture(scope="module")
def engine(cuda_device):
    case, sd, bm, x, K, _ = pu.build_inputs("s_224_S_forced")
    return pu.build_engine(case, sd, bm, max_persons=CAP), bm


ROOT_ANGLES = (0.0, 5e-7, 1e-6 * (1 - 2.0 ** -20), 1e-6 * (1 + 2.0 ** -20), 2e-6, 0.5 * (1 - 2.0 ** -20),
               0.5 * (1 + 2.0 ** -20))


def placed_backward(m, args, up):
    from multihmr_b200._lib import call, stream

    m.finalize()
    x = m._smplx_inputs(*args)
    P = int(args[0].shape[0])
    shapes = dict(rot=(53, 3), shape=(x[1].shape[1],), expr=(10,), loc=(2,), dist=())
    cv = {k: _canvas(s, P, m.max_persons, m.device) for k, s in shapes.items()}
    g = lambda k: None if up.get(k) is None else up[k].to(m.device, torch.float32).contiguous()
    call("mhmr_smplx_backward", m._handle, P, x[0], x[1], x[5], x[2], x[3], x[4], g("v3d"), g("v2d"), g("j3d"),
         g("j2d"), g("transl"), g("transl_pelvis"), cv["rot"][1], cv["shape"][1], cv["expr"][1], cv["loc"][1],
         cv["dist"][1], stream())
    torch.cuda.synchronize()
    for k, (buf, view) in cv.items():
        _check(buf, view, P, k)
    return [cv[k][1] for k in ("rot", "shape", "loc", "dist", "expr")]


def placed_ratios(bm, args, up, got, dev):
    d = lambda t: t.to(dev, torch.float64).requires_grad_()
    ins = [d(a) for a in args]
    ins_ = ins[:4] + [ins[5]]
    out = bg.placed_outputs(bm, *ins[:4], args[4].to(dev, torch.float64), ins[5])
    upd = {k: v.to(dev) for k, v in up.items()}
    ref = bg.vjp(out, upd, ins_)
    ref_abs = bg.vjp(out, {k: v.abs() for k, v in upd.items()}, ins_)
    with torch.no_grad():
        _, bound = bg.backward_bound(bm, [a.to(dev, torch.float64) for a in args], upd, placed=True)
    n = bg.n_seq(torch.as_tensor(bm["v_template"]).shape[0], 55)
    old = new = 0.0
    for a, r, ra, name in zip(got, ref, ref_abs, ("d_rotvec", "d_shape", "d_loc", "d_dist", "d_expression")):
        err = (a.double().reshape(r.shape) - r).abs()
        old = max(old, (err / bg.tolerance(r, ra, n)).max().item())
        new = max(new, (err / bound[name].reshape(r.shape)).max().item())
    return old, new


@pytest.mark.parametrize("P", PERSONS)
def test_placed_at_pass_edges_and_root_branches(engine, P, cuda_device):
    """The placed layer through an engine of capacity 80; person p's root at |r| = ROOT_ANGLES[p % 7]."""
    m, bm = engine
    args = list(bf.placed_inputs(P, seed=40 + P))
    g = torch.Generator().manual_seed(50 + P)
    unit = torch.randn(P, 3, generator=g, dtype=torch.float64)
    unit = unit / unit.norm(dim=-1, keepdim=True)
    ang = torch.tensor([ROOT_ANGLES[p % len(ROOT_ANGLES)] for p in range(P)], dtype=torch.float64)
    args[0] = args[0].clone()
    args[0][:, 0] = (unit * ang[:, None]).float()
    worst = {}
    for which in ("all", "v3d", "v2d", "j3d", "j2d", "transl", "transl_pelvis"):
        up = bg.upstream(P, m.num_verts, 127, g, which)
        got = placed_backward(m, args, up)
        worst[which] = placed_ratios(bm, args, up, got, cuda_device)
        assert max(worst[which]) <= 1.0, (P, which, worst[which])
    print(f"placed P={P} worst err/tol (per-person / per-element): "
          + ", ".join(f"{k} {a:.3f}/{b:.4f}" for k, (a, b) in worst.items()))


# ------------------------------------------------------------------------------------------------ 4. planted mistakes
NEW_MISTAKES = ("last_tile", "last_coef_row", "lmk_corner", "extra_last_vertex", "leaf_parent", "second_pass")


@pytest.mark.parametrize("kind", ["smpl", "smplx"])
def test_planted_mistakes(kind, cuda_device):
    """At the largest nb and P = 2 GPB + 1, sparse upstream (the instance of test_body_grad_bound_cpu's separation
    test): the device lies inside both bounds of the true reference, and each mistaken reference is more than twice
    the bound away from the true one, so the device lies outside the bound around it."""
    nb = bf.NB_EDGES[kind][2]
    bm = bg.edge_body(kind, nb)
    body = _body(bm, kind, nb, cuda_device)
    P = 2 * bg.GPB + 1
    args = bf.random_inputs(kind, P, nb, seed=4)
    g = torch.Generator().manual_seed(5)
    up = bg.upstream(P, body.num_verts, body.num_joints, g, "all", sparse=True)
    up.pop("transl")
    got = raw_backward(body, args, up)
    ref, ref_abs = raw_reference(bm, args, up, cuda_device)
    n = bg.n_seq(body.num_verts, bf.NJ[kind])
    tol = [bg.tolerance(r, ra, n) for r, ra in zip(ref, ref_abs)]
    with torch.no_grad():
        _, bd = bg.backward_bound(bm, [None if a is None else a.to(cuda_device, torch.float64) for a in args],
                                  {k: v.to(cuda_device) for k, v in up.items()})
    new = [bd[k].reshape(r.shape) for k, r in zip(RAW_NAMES, ref)]
    ratio = lambda x, want, b: max(((a.double().reshape(r.shape) - r).abs() / t).max().item()
                                   for a, r, t in zip(x, want, b))
    assert ratio(got, ref, tol) <= 1.0 and ratio(got, ref, new) <= 1.0
    for name in NEW_MISTAKES:
        if name == "lmk_corner" and kind == "smpl":
            continue
        if name == "second_pass":
            wrong = [t.clone() for t in ref]
            for t in wrong:
                t[bg.GPB:2 * bg.GPB] = t[:bg.GPB]
        else:
            wrong, _ = raw_reference(bm, args, up, cuda_device, **{name: True})
        r_old, r_new = ratio(got, wrong, tol), ratio(wrong, ref, new)
        print(f"{kind} mistaken reference {name}: device err/tol {r_old:.1f} (per-person), "
              f"|wrong - ref| / bound {r_new:.2f} (per-element)")
        assert r_old > 1.0 and r_new > 2.0, name


# ------------------------------------------------------------------------------------------------ 5. invariants
def test_invariants(random_bodies, cuda_device):
    kind = "smplx"
    nb = bf.NB_EDGES[kind][1]
    bm, body = random_bodies[kind, nb]
    g = torch.Generator().manual_seed(99)
    args = bf.random_inputs(kind, CAP, nb, seed=5)
    up = bg.upstream(CAP, body.num_verts, body.num_joints, g, "all")
    up.pop("transl")
    a = raw_backward(body, args, up)
    assert all(torch.equal(x, y) for x, y in zip(a, raw_backward(body, args, up))), "repeated call"
    sub = lambda lo, hi: ([None if t is None else t[lo:hi] for t in args], {k: v[lo:hi] for k, v in up.items()})
    # P = 17 right after P = 80 equals a fresh handle's P = 17 and the first 17 persons of the P = 80 call
    b17 = raw_backward(body, *sub(0, 17))
    fresh = _body(bm, kind, nb, cuda_device)
    f17 = raw_backward(fresh, *sub(0, 17))
    assert all(torch.equal(x, y) for x, y in zip(b17, f17)), "P = 17 after P = 80 differs from a fresh call"
    assert all(torch.equal(x[:17], y) for x, y in zip(a, b17)), "a person's gradient depends on the call's P"
    # batch position across a pass boundary: persons 15..17 alone and as a batch starting at 15
    for lo, hi in ((15, 16), (16, 17), (15, 18), (bg.GPB, 2 * bg.GPB + 1)):
        s = raw_backward(body, *sub(lo, hi))
        assert all(torch.equal(x[lo:hi], y) for x, y in zip(a, s)), (lo, hi)
    # NaN upstream on one person and NaN pose on another leave the others' bits alone
    bad_args = [None if t is None else t.clone() for t in args]
    bad_up = {k: v.clone() for k, v in up.items()}
    bad_up["v3d"][bg.GPB] = float("nan")
    bad_args[0][CAP - 1] = float("nan")
    c = raw_backward(body, bad_args, bad_up)
    keep = torch.ones(CAP, dtype=torch.bool, device=cuda_device)
    keep[[bg.GPB, CAP - 1]] = False
    assert all(torch.equal(x[keep], y[keep]) for x, y in zip(a, c)), "a NaN person changed another person's gradients"
    # P = 0 writes nothing
    from multihmr_b200._lib import call, stream

    fp, bb, tr, Kd, ex = body._inputs(*[None if t is None else t[:1] for t in args])
    outs = [_canvas(s, 1, CAP, cuda_device) for s in ((body.num_pose_joints * 3,), (nb,), (10,), (3,))]
    call("mhmr_body_backward", body._h, 0, fp, bb, ex, tr, Kd, up["v3d"][:1].to(cuda_device), None, None, None, None,
         *[o[1] for o in outs], stream())
    torch.cuda.synchronize()
    assert all((o[0] == SENTINEL).all() for o in outs), "P = 0 wrote to an output"
