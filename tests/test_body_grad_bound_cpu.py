"""The per-element bound of the body-model backward (body_grad_util.backward_bound) and the planted mistakes of
body_grad_util.body, in fp64 on the CPU:

  * the bound's restatement of the kernels' stages computes the fp64 autograd gradients (so its magnitudes and error
    terms follow the arithmetic the device does), raw SMPL / SMPL-X at real size and at tile edges, and placed;
  * the Taylor truncation of rotvec_grad below TAYLOR_BELOW stays within TAYLOR_TRUNC (2 a)^8;
  * each planted mistake moves some gradient element by more than twice the per-element bound (bg.backward_bound) and
    twice the per-person bound (bg.tolerance) at the edge shape where it matters, so a device result inside either
    bound is outside it for the mistaken reference (triangle inequality);
  * the median ratio of the two bounds per gradient is printed."""

import pytest
import torch

import body_forward_util as bf
import body_grad_util as bg

RAW = ("d_full_pose", "d_betas", "d_transl", "d_expression")


def _grads(bm, args, up, **mistake):
    pose, betas, transl, K, expr = args
    d = lambda t: None if t is None else t.double().requires_grad_()
    ins = [d(pose), d(betas), d(transl)] + ([d(expr)] if expr is not None else [])
    out = bg.raw_outputs(bm, ins[0], ins[1], ins[2], K.double(), ins[3] if expr is not None else None, **mistake)
    return bg.vjp(out, up, ins), bg.vjp(out, {k: v.abs() for k, v in up.items()}, ins)


_edge_body, _njout = bg.edge_body, bg.num_output_joints


@pytest.mark.parametrize("kind,V", [("smplx", None), ("smpl", None), ("smplx", 81), ("smpl", 161)])
def test_restatement_is_the_gradient(kind, V):
    nb = bf.NB_EDGES[kind][2]
    bm = _edge_body(kind, nb, V)
    V = torch.as_tensor(bm["v_template"]).shape[0]
    P = 3
    args = bf.random_inputs(kind, P, nb, seed=2)
    g = torch.Generator().manual_seed(4)
    for which in ("all", "v3d", "j2d", "transl_pelvis"):
        up = bg.upstream(P, V, _njout(kind), g, which)
        up.pop("transl", None)
        ref, _ = _grads(bm, args, up)
        got, bound = bg.backward_bound(bm, [None if a is None else a.double() for a in args], up)
        for name, r in zip(RAW, ref):
            a = got[name].reshape(r.shape)
            assert ((a - r).abs().max() <= 1e-6 * r.abs().max() + 1e-300), (which, name)
            assert (bound[name] >= 0).all() and torch.isfinite(bound[name]).all()


def test_placed_restatement_is_the_gradient():
    bm = bf.random_body("smplx", 10)
    args = bf.placed_inputs(4, seed=3)
    g = torch.Generator().manual_seed(5)
    for which in ("all", "v2d", "transl"):
        up = bg.upstream(4, 10475, 127, g, which)
        d = lambda t: t.double().requires_grad_()
        ins = [d(a) for a in args]
        out = bg.placed_outputs(bm, *ins[:4], args[4].double(), ins[5])
        ref = bg.vjp(out, up, ins[:4] + [ins[5]])
        got, bound = bg.backward_bound(bm, [a.double() for a in args], up, placed=True)
        for name, r in zip(("d_rotvec", "d_shape", "d_loc", "d_dist", "d_expression"), ref):
            assert ((got[name].reshape(r.shape) - r).abs().max() <= 1e-6 * r.abs().max()), (which, name)


def test_taylor_truncation():
    a = torch.linspace(0.3, bg.TAYLOR_BELOW, 200, dtype=torch.float64)
    ser, _ = bg._rot_coefs(a, torch.ones_like(a, dtype=torch.bool))
    clo, _ = bg._rot_coefs(a, torch.zeros_like(a, dtype=torch.bool))
    worst = max(((x - y).abs() / (bg.TAYLOR_TRUNC * (2 * a) ** 8)).max().item() for x, y in zip(ser, clo))
    print(f"Taylor truncation / bound: {worst:.3f}")
    assert worst <= 1.0


MISTAKES = ("last_tile", "last_coef_row", "lmk_corner", "extra_last_vertex", "leaf_parent", "second_pass")


@pytest.mark.parametrize("kind", ["smplx", "smpl"])
def test_planted_mistakes_separate(kind):
    """P = 2 GPB + 1 (second_pass), the largest nb (last_coef_row at KT = 512 / 239), the real body's partial last
    tile (10475 = 130 * 80 + 75, 6890 = 86 * 80 + 10), sparse upstream on every output."""
    nb = bf.NB_EDGES[kind][2]
    bm = _edge_body(kind, nb)
    V = torch.as_tensor(bm["v_template"]).shape[0]
    P = 2 * bg.GPB + 1
    args = bf.random_inputs(kind, P, nb, seed=4)
    g = torch.Generator().manual_seed(5)
    up = bg.upstream(P, V, _njout(kind), g, "all", sparse=True)
    up.pop("transl")
    ref, ref_abs = _grads(bm, args, up)
    n = bg.n_seq(V, bf.NJ[kind])
    old = [bg.tolerance(r, ra, n) for r, ra in zip(ref, ref_abs)]
    _, bd = bg.backward_bound(bm, [None if a is None else a.double() for a in args], up)
    new = [bd[k].reshape(r.shape) for k, r in zip(RAW, ref)]
    print(f"{kind}: median per-person / per-element bound: "
          + ", ".join(f"{k} {(o / b).median().item():.2f}" for k, o, b in zip(RAW, old, new)))
    for name in MISTAKES:
        if name == "lmk_corner" and kind == "smpl":
            continue
        if name == "second_pass":
            wrong = [t.clone() for t in ref]
            for t in wrong:
                t[bg.GPB:2 * bg.GPB] = t[:bg.GPB]
        else:
            wrong, _ = _grads(bm, args, up, **{name: True})
        sep = lambda tol: max(((w - r).abs() / t).max().item() for w, r, t in zip(wrong, ref, tol))
        s_old, s_new = sep(old), sep(new)
        print(f"{kind} {name}: separation {s_old:.1f} (per-person bound), {s_new:.2f} (per-element bound)")
        assert s_old > 2.0 and s_new > 2.0, name
