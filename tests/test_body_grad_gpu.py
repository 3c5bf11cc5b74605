"""Backward of the body models on the device (mhmr_body_backward, mhmr_smplx_backward) against the fp64 autograd of
the oracle: every input gradient per element within a bound derived from the kernels' accumulation lengths
(body_grad_util.tolerance), for random upstream gradients on all outputs and on each output alone; each planted
mistake of the reference falls outside the bound; bitwise determinism and batch independence; the autograd
wrappers; a fitting loop."""
import math

import pytest
import torch

import body_grad_util as bg
import parity_util as pu

pytestmark = pytest.mark.gpu
OUTS_RAW = ("all", "v3d", "v2d", "j3d", "j2d", "transl_pelvis")


@pytest.fixture(scope="module")
def assets():
    from oracle import eval_bench_ref as R

    return R.eval_assets(0)


@pytest.fixture(scope="module")
def bodies(assets, cuda_device):
    from multihmr_b200 import metrics

    return {"smplx": metrics.BodyModel(assets["smplx"], "smplx", 11, 48, cuda_device),
            "smpl": metrics.BodyModel(assets["smpl_male"], "smpl", 10, 48, cuda_device)}


@pytest.fixture(scope="module")
def engine(cuda_device):
    case, sd, bm, x, K, _ = pu.build_inputs("s_224_S_forced")
    return pu.build_engine(case, sd, bm, max_persons=32), bm


def _raw_case(kind, P, seed):
    g = torch.Generator().manual_seed(seed)
    NJ, nb = (55, 11) if kind == "smplx" else (24, 10)
    pose = bg.poses(P, NJ, g)
    betas = torch.randn(P, nb, generator=g)
    betas[-1] *= 4.0  # large shape coefficients
    transl = torch.randn(P, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 6.0])
    K = torch.tensor([[388.0, 0, 224.0], [0, 388.0, 224.0], [0, 0, 1.0]]).repeat(P, 1, 1)
    expr = torch.randn(P, 10, generator=g) * 0.5 if kind == "smplx" else None
    return pose, betas, transl, K, expr, g


def _placed_case(P, seed):
    from multihmr_b200 import synth

    g = torch.Generator().manual_seed(seed)
    rotvec = bg.poses(P, 53, g)
    rotvec[-1, 0] = 0.0  # small-angle branch of the root rotation
    shape = torch.randn(P, 10, generator=g)
    shape[-1] *= 4.0
    expr = torch.randn(P, 10, generator=g) * 0.5
    loc = torch.rand(P, 2, generator=g) * 200 + 10
    dist = torch.rand(P, generator=g) * 5 + 1.5
    K = synth.make_cameras(P, 224, jitter=True, seed=P)
    return rotvec, shape, loc, dist, K, expr, g


def _raw_ref(bm, dev, pose, betas, transl, K, expr, up, **mistake):
    d = lambda t: None if t is None else t.to(dev, torch.float64).requires_grad_()
    ins = [d(pose), d(betas), d(transl)] + ([d(expr)] if expr is not None else [])
    out = bg.raw_outputs(bm, ins[0], ins[1], ins[2], K.to(dev, torch.float64), ins[3] if expr is not None else None,
                         **mistake)
    ref = bg.vjp(out, up, ins)
    ref_abs = bg.vjp(out, {k: v.abs() for k, v in up.items()}, ins)
    return ref, ref_abs


def _raw_got(body, pose, betas, transl, K, expr, up):
    x = body._inputs(pose, betas, transl, K, expr)
    d_fp, d_b, d_ex, d_tr = body._backward(*x, g_v3d=up.get("v3d"), g_v2d=up.get("v2d"), g_j3d=up.get("j3d"),
                                           g_j2d=up.get("j2d"), g_transl_pelvis=up.get("transl_pelvis"))
    return [d_fp, d_b, d_tr] + ([d_ex] if expr is not None else [])


def _ratio(got, ref, ref_abs, n):
    worst = 0.0
    for a, r, ra in zip(got, ref, ref_abs):
        tol = bg.tolerance(r, ra, n)
        err = (a.double().reshape(r.shape) - r).abs()
        worst = max(worst, (err / tol).max().item())
    return worst


@pytest.mark.parametrize("kind,P", [("smplx", 1), ("smplx", 16), ("smplx", 17), ("smplx", 48), ("smpl", 1),
                                    ("smpl", 9)])
def test_raw_backward_vs_fp64(assets, bodies, kind, P, cuda_device):
    bm = assets["smplx" if kind == "smplx" else "smpl_male"]
    body = bodies[kind]
    pose, betas, transl, K, expr, g = _raw_case(kind, P, 100 + P)
    n = bg.n_seq(body.num_verts, body.num_pose_joints)
    report = []
    for which in OUTS_RAW:
        up = bg.upstream(P, body.num_verts, body.num_joints, g, which)
        up.pop("transl", None)
        up = {k: v.to(cuda_device) for k, v in up.items()}
        got = _raw_got(body, pose, betas, transl, K, expr, up)
        ref, ref_abs = _raw_ref(bm, cuda_device, pose, betas, transl, K, expr, up)
        r = _ratio(got, ref, ref_abs, n)
        report.append(f"{which} {r:.3f}")
        assert all(torch.isfinite(t).all() for t in got)
        assert r <= 1.0, (which, r)
    print(f"{kind} P={P} worst err/tol: " + ", ".join(report))


def test_raw_backward_sensitivity(assets, bodies, cuda_device):
    bm, body = assets["smplx"], bodies["smplx"]
    P = 4
    pose, betas, transl, K, expr, g = _raw_case("smplx", P, 7)
    up = bg.upstream(P, body.num_verts, body.num_joints, g, "all", sparse=True)
    up = {k: up[k].to(cuda_device) for k in ("v3d", "j3d")}
    got = _raw_got(body, pose, betas, transl, K, expr, up)
    n = bg.n_seq(body.num_verts, 55)
    ref, ref_abs = _raw_ref(bm, cuda_device, pose, betas, transl, K, expr, up)
    assert _ratio(got, ref, ref_abs, n) <= 1.0
    mistakes = dict(no_posedirs=True, j_const=True, parent_swap=18, rod_t=True, no_scatter=True)
    for name, val in mistakes.items():
        wrong, _ = _raw_ref(bm, cuda_device, pose, betas, transl, K, expr, up, **{name: val})
        r = _ratio(got, wrong, ref_abs, n)
        print(f"mistaken reference {name}: err/tol {r:.1f}")
        assert r > 1.0, name


def _placed_ref(bm, dev, rotvec, shape, loc, dist, K, expr, up, **mistake):
    d = lambda t: t.to(dev, torch.float64).requires_grad_()
    ins = [d(rotvec), d(shape), d(loc), d(dist), d(expr)]
    out = bg.placed_outputs(bm, *ins[:4], K.to(dev, torch.float64), ins[4], **mistake)
    return bg.vjp(out, up, ins), bg.vjp(out, {k: v.abs() for k, v in up.items()}, ins)


def _placed_got(m, rotvec, shape, loc, dist, K, expr, up):
    x = m._smplx_inputs(rotvec, shape, loc, dist, K, expr)
    d_rot, d_shape, d_loc, d_dist, d_expr = m._smplx_backward(
        x, g_v3d=up.get("v3d"), g_v2d=up.get("v2d"), g_j3d=up.get("j3d"), g_j2d=up.get("j2d"),
        g_transl=up.get("transl"), g_transl_pelvis=up.get("transl_pelvis"))
    return [d_rot, d_shape, d_loc, d_dist, d_expr]


@pytest.mark.parametrize("P", [1, 5, 16, 23])
def test_placed_backward_vs_fp64(engine, P, cuda_device):
    m, bm = engine
    rotvec, shape, loc, dist, K, expr, g = _placed_case(P, 200 + P)
    n = bg.n_seq(m.num_verts, 55)
    report = []
    for which in OUTS_RAW + ("transl",):
        up = {k: v.to(cuda_device) for k, v in bg.upstream(P, m.num_verts, 127, g, which).items()}
        got = _placed_got(m, rotvec, shape, loc, dist, K, expr, up)
        ref, ref_abs = _placed_ref(bm, cuda_device, rotvec, shape, loc, dist, K, expr, up)
        r = _ratio(got, ref, ref_abs, n)
        report.append(f"{which} {r:.3f}")
        assert r <= 1.0, (which, r)
    print(f"placed P={P} worst err/tol: " + ", ".join(report))
    # the head-joint centre treated as constant falls outside the bound
    up = {k: v.to(cuda_device) for k, v in bg.upstream(P, m.num_verts, 127, g, "all", sparse=True).items()}
    got = _placed_got(m, rotvec, shape, loc, dist, K, expr, up)
    ref, ref_abs = _placed_ref(bm, cuda_device, rotvec, shape, loc, dist, K, expr, up)
    wrong, _ = _placed_ref(bm, cuda_device, rotvec, shape, loc, dist, K, expr, up, center_const=True)
    assert _ratio(got, ref, ref_abs, n) <= 1.0 < _ratio(got, wrong, ref_abs, n)


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def test_bitwise_repeat_and_batch_independence(bodies, engine, cuda_device):
    body = bodies["smplx"]
    P = 48
    pose, betas, transl, K, expr, g = _raw_case("smplx", P, 5)
    up = {k: v.to(cuda_device) for k, v in bg.upstream(P, body.num_verts, body.num_joints, g, "all").items()}
    up.pop("transl")
    a = _raw_got(body, pose, betas, transl, K, expr, up)
    assert _same(a, _raw_got(body, pose, betas, transl, K, expr, up))
    perm = torch.randperm(P, generator=g)
    sub = lambda d, idx: {k: v[idx.to(v.device)] for k, v in d.items()}
    b = _raw_got(body, pose[perm], betas[perm], transl[perm], K[perm], expr[perm], sub(up, perm))
    assert _same([t[perm.to(t.device)] for t in a], b)
    for i in (0, 17, 47):
        one = torch.tensor([i])
        c = _raw_got(body, pose[one], betas[one], transl[one], K[one], expr[one], sub(up, one))
        assert _same([t[i:i + 1] for t in a], c)
    m, _ = engine
    P = 23
    rotvec, shape, loc, dist, K, expr, g = _placed_case(P, 9)
    up = {k: v.to(cuda_device) for k, v in bg.upstream(P, m.num_verts, 127, g, "all").items()}
    a = _placed_got(m, rotvec, shape, loc, dist, K, expr, up)
    assert _same(a, _placed_got(m, rotvec, shape, loc, dist, K, expr, up))
    perm = torch.randperm(P, generator=g)
    b = _placed_got(m, rotvec[perm], shape[perm], loc[perm], dist[perm], K[perm], expr[perm], sub(up, perm))
    assert _same([t[perm.to(t.device)] for t in a], b)
    one = torch.tensor([11])
    c = _placed_got(m, rotvec[one], shape[one], loc[one], dist[one], K[one], expr[one], sub(up, one))
    assert _same([t[11:12] for t in a], c)


def test_autograd_wrappers_match_entries(bodies, engine, cuda_device):
    body = bodies["smplx"]
    P = 3
    pose, betas, transl, K, expr, g = _raw_case("smplx", P, 11)
    x = body._inputs(pose, betas, transl, K, expr)
    direct = body._forward(*x)
    with torch.no_grad():
        ng = body(pose, betas, transl, K, expr)
    plain = body(pose, betas, transl, K, expr)
    leaves = [t.clone().requires_grad_() for t in (pose, betas, transl, expr)]
    out = body(leaves[0], leaves[1], leaves[2], K, leaves[3])
    for k in direct:
        assert torch.equal(direct[k], ng[k]) and torch.equal(direct[k], plain[k]) and torch.equal(direct[k], out[k])
        assert not ng[k].requires_grad and not plain[k].requires_grad and out[k].requires_grad
    up = {k: torch.randn(out[k].shape, generator=g).to(cuda_device) for k in ("v3d", "j3d", "j2d", "transl_pelvis")}
    gr = torch.autograd.grad(sum((out[k] * up[k]).sum() for k in up), leaves)
    d = _raw_got(body, pose, betas, transl, K, expr, up)
    for a, b, leaf in zip(gr, [d[0], d[1], d[2], d[3]], leaves):
        assert a.shape == leaf.shape and a.dtype == leaf.dtype and a.device == leaf.device
        assert torch.equal(a.to(cuda_device).reshape(-1), b.reshape(-1))
    # no expression: no expression gradient; K requiring grad raises
    out = body(leaves[0], leaves[1], leaves[2], K)
    assert out["v3d"].requires_grad
    with pytest.raises(NotImplementedError):
        body(leaves[0], betas, transl, K.clone().requires_grad_(), expr)
    with pytest.raises(ValueError):
        body(torch.zeros(49, 55, 3, requires_grad=True), torch.zeros(49, 11), torch.zeros(49, 3), K[:1].repeat(49, 1, 1))

    m, _ = engine
    rotvec, shape, loc, dist, K, expr, g = _placed_case(4, 12)
    xs = m._smplx_inputs(rotvec, shape, loc, dist, K, expr)
    direct = m._smplx_forward(*xs)
    with torch.no_grad():
        ng = m.smplx(rotvec, shape, loc, dist, K, expr)
    leaves = [t.clone().requires_grad_() for t in (rotvec, shape, loc, dist, expr)]
    out = m.smplx(leaves[0], leaves[1], leaves[2], leaves[3], K, leaves[4])
    for k in direct:
        assert torch.equal(direct[k], ng[k]) and torch.equal(direct[k], out[k]), k
        assert out[k].requires_grad and not ng[k].requires_grad
    up = {k: torch.randn(out[k].shape, generator=g).to(cuda_device)
          for k in ("v3d", "v2d", "j3d", "j2d", "transl", "transl_pelvis")}
    gr = torch.autograd.grad(sum((out[k] * up[k]).sum() for k in up), leaves)
    up["transl_pelvis"] = up["transl_pelvis"][:, 0]
    d = _placed_got(m, rotvec, shape, loc, dist, K, expr, up)
    for a, b, leaf in zip(gr, d, leaves):
        assert a.shape == leaf.shape and a.dtype == leaf.dtype and a.device == leaf.device
        assert torch.equal(a.to(cuda_device).reshape(-1), b.reshape(-1))
    with pytest.raises(NotImplementedError):
        m.smplx(leaves[0], shape, loc, dist, K.clone().requires_grad_(), expr)


def test_entries_reject_bad_arguments(bodies, engine, cuda_device):
    from ctypes import c_int, c_void_p

    from multihmr_b200._lib import MhmrError, check, ptr

    body = bodies["smpl"]
    x = body._inputs(*_raw_case("smpl", 2, 3)[:5])
    d = [torch.empty_like(t) for t in (x[0], x[1], x[2])]
    call = lambda P, fp: body._lib.mhmr_body_backward(body._h, c_int(P), ptr(fp), ptr(x[1]), None, ptr(x[2]),
                                                      ptr(x[3]), None, None, None, None, None, ptr(d[0]), ptr(d[1]),
                                                      None, ptr(d[2]), c_void_p(0))
    for P, fp in ((49, x[0]), (-1, x[0]), (2, None)):
        with pytest.raises((AssertionError, MhmrError)):
            check(call(P, fp), "mhmr_body_backward")
    m, _ = engine
    xs = m._smplx_inputs(*_placed_case(2, 3)[:6])
    with pytest.raises((AssertionError, MhmrError)):
        check(m._lib.mhmr_smplx_backward(m._handle, c_int(33), *[ptr(t) for t in xs[:2]], ptr(xs[5]), ptr(xs[2]),
                                         ptr(xs[3]), ptr(xs[4]), *([None] * 6), *[ptr(torch.empty_like(t)) for t in
                                                                                  (xs[0], xs[1], xs[5], xs[2], xs[3])],
                                         c_void_p(0)), "mhmr_smplx_backward")


def _fit(grad_fn, forward, params, target, steps=200):
    opt = torch.optim.Adam(params, lr=0.01)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.98)
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        loss = grad_fn(params, target)
        losses.append(float(loss))
        opt.step()
        sched.step()
    return losses


def test_fitting_loop(assets, bodies, cuda_device):
    """Adam on full_pose, betas and transl of 4 SMPL-X persons from a perturbed start, against vertices and joints
    made by the forward from known parameters.  The same loop with the fp64 oracle's gradients reduces the loss by
    well over 100x in 200 steps (printed below); the device gradients must do as well."""
    body, bm = bodies["smplx"], assets["smplx"]
    P = 4
    g = torch.Generator().manual_seed(21)
    pose = torch.randn(P, 55, 3, generator=g) * 0.3
    betas = torch.randn(P, 11, generator=g)
    transl = torch.randn(P, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 6.0])
    K = torch.tensor([[388.0, 0, 224.0], [0, 388.0, 224.0], [0, 0, 1.0]]).repeat(P, 1, 1)
    expr = torch.zeros(P, 10)
    with torch.no_grad():
        t = body(pose, betas, transl, K, expr)
    target = (t["v3d"], t["j3d"])
    start = [pose + torch.randn(P, 55, 3, generator=g) * 0.05, betas + torch.randn(P, 11, generator=g) * 0.3,
             transl + torch.randn(P, 3, generator=g) * 0.02]

    def loss_dev(params, target):
        out = body(params[0], params[1], params[2], K, expr)
        return ((out["v3d"] - target[0]) ** 2).sum(-1).mean() + ((out["j3d"] - target[1]) ** 2).sum(-1).mean()

    d64 = lambda t: t.to(cuda_device, torch.float64)
    tgt64 = (d64(target[0]), d64(target[1]))
    K64, e64 = d64(K), d64(expr)

    def loss_ref(params, target):
        out = bg.raw_outputs(bm, params[0], params[1], params[2], K64, e64)
        return ((out["v3d"] - target[0]) ** 2).sum(-1).mean() + ((out["j3d"] - target[1]) ** 2).sum(-1).mean()

    def run(fn, params):
        def step(p, t):
            loss = fn(p, t)
            loss.backward()
            return loss.detach()
        return _fit(step, None, params, None)

    ref = run(lambda p, _: loss_ref(p, tgt64), [d64(s).requires_grad_() for s in start])
    dev = run(lambda p, _: loss_dev(p, target), [s.to(cuda_device).requires_grad_() for s in start])
    print(f"fitting: fp64 oracle {ref[0]:.3e} -> {ref[-1]:.3e} ({ref[0] / ref[-1]:.0f}x), "
          f"device {dev[0]:.3e} -> {dev[-1]:.3e} ({dev[0] / dev[-1]:.0f}x)")
    assert ref[0] / ref[-1] >= 100.0
    assert dev[0] / dev[-1] >= 100.0
