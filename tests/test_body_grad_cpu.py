"""The fp64 references of the body-model backward: the autograd of the oracle (smplx_ref.lbs for SMPL and SMPL-X,
multihmr_ref.smpl_layer_forward for the placed layer) agrees with central differences, including rotation rows at
exactly 0, at 1e-4 rad and near pi; and the restatement in body_grad_util that the GPU tests differentiate (with
its mistake switches off) computes the oracle's values."""
import math

import pytest
import torch

import body_grad_util as bg
from oracle import multihmr_ref, smplx_ref

torch.set_grad_enabled(True)


def _bm(kind):
    from multihmr_b200 import synth

    return synth.make_body_model(0) if kind == "smplx" else synth.make_smpl_body_model(0, "male")


def _oracle_raw(bm, kind, pose, betas, transl, K, expr):
    """smplx.SMPL / SMPL-X forward through oracle/smplx_ref.lbs (as tests/test_eval_benchmarks_gpu.py states it)."""
    d = lambda k: torch.as_tensor(bm[k]).double()
    if kind == "smpl":
        comps, dirs = betas, d("shapedirs")[..., :10]
    else:
        sd = torch.cat([d("shapedirs"), d("shapedirs_extra")], -1)[..., :11]
        comps, dirs = torch.cat([betas, expr], -1), torch.cat([sd, d("expr_dirs")], -1)
    v, j = smplx_ref.lbs(comps, pose.reshape(pose.shape[0], -1), d("v_template"), dirs, d("posedirs"),
                         d("J_regressor"), torch.as_tensor(bm["parents"]).long(), d("lbs_weights"))
    j = torch.cat([j, v[:, torch.as_tensor(bm["extra_joints_idxs"]).long()]], 1)
    if kind == "smplx":
        j = torch.cat([j, smplx_ref.vertices2landmarks(v, bm["faces"].long(), bm["lmk_faces_idx"].long(),
                                                      d("lmk_bary_coords"))], 1)
    t = transl.unsqueeze(1)
    v, j = v + t, j + t
    pp = multihmr_ref.perspective_projection
    return dict(v3d=v, v2d=pp(v, K), j3d=j, j2d=pp(j, K), transl_pelvis=j[:, 0])


def _central(f, x, idx, h=1e-6):
    out = []
    for i in idx:
        xp, xm = x.detach().clone(), x.detach().clone()
        xp.view(-1)[i] += h
        xm.view(-1)[i] -= h
        out.append((f(xp) - f(xm)) / (2 * h))
    return torch.stack(out)


def _check(f, inputs, coords):
    """Autograd of the scalar f(*inputs) against central differences at the listed flat coordinates."""
    xs = [t.detach().clone().requires_grad_() for t in inputs]
    grads = torch.autograd.grad(f(*xs), xs)
    worst = 0.0
    for k, (x, g) in enumerate(zip(xs, grads)):
        idx = coords[k]
        fk = lambda xk: f(*[xk if i == k else t.detach() for i, t in enumerate(xs)]).detach()
        num = _central(fk, x, idx)
        ana = g.reshape(-1)[idx]
        scale = ana.abs().max().item() + 1e-12
        err = (num - ana).abs().max().item() / scale
        worst = max(worst, err)
        assert torch.isfinite(ana).all()
        assert err < 1e-5, (k, err)
    return worst


def _pose_coords(NJ, rows, g, extra=6):
    rnd = torch.randperm(NJ * 3, generator=g)[:extra].tolist()
    return sorted(set([r * 3 + c for r in rows for c in range(3)] + rnd))


@pytest.mark.parametrize("kind", ["smplx", "smpl"])
def test_raw_oracle_autograd_vs_central_differences(kind):
    bm = _bm(kind)
    g = torch.Generator().manual_seed(3)
    P, NJ, nb = 2, (55 if kind == "smplx" else 24), (11 if kind == "smplx" else 10)
    pose = bg.poses(P, NJ, g).double()        # person 0: zero rows from NJ/2; rows 3 / 4: |r| = 1e-4, pi - 1e-3
    betas = torch.randn(P, nb, generator=g).double()
    transl = (torch.randn(P, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 6.0])).double()
    K = torch.tensor([[388.0, 0, 224.0], [0, 388.0, 224.0], [0, 0, 1.0]]).double().repeat(P, 1, 1)
    expr = (torch.randn(P, 10, generator=g) * 0.5).double() if kind == "smplx" else None
    V = int(bm["v_template"].shape[0])
    J = NJ + 21 + (51 if kind == "smplx" else 0)
    up = bg.upstream(P, V, J, g, "all")
    up.pop("transl")
    up = {k: v.double() for k, v in up.items()}

    def f(pose, betas, transl, *ex):
        out = _oracle_raw(bm, kind, pose, betas, transl, K, ex[0] if ex else None)
        return sum((out[k] * up[k]).sum() for k in up)

    inputs = [pose, betas, transl] + ([expr] if expr is not None else [])
    zero_row = NJ - 1  # inside person 0's zero rows
    coords = [_pose_coords(NJ, [0, 3, 4, zero_row, NJ + 3, NJ + 4], g), list(range(nb * P)), list(range(3 * P))]
    if expr is not None:
        coords.append(list(range(0, 10 * P, 3)))
    print(f"{kind}: worst relative deviation {_check(f, inputs, coords):.2e}")
    # the restatement the GPU tests differentiate computes the oracle's values
    ref = _oracle_raw(bm, kind, pose, betas, transl, K, expr)
    mine = bg.raw_outputs(bm, pose, betas, transl, K, expr)
    for k in ref:
        assert (ref[k] - mine[k]).abs().max().item() < 1e-9, k


def test_placed_oracle_autograd_vs_central_differences():
    from multihmr_b200 import synth

    bm = synth.make_body_model(0)
    g = torch.Generator().manual_seed(4)
    P = 2
    rotvec = bg.poses(P, 53, g).double()
    rotvec[1, 0] = torch.tensor([1.0, -2.0, 0.5]).double() / math.sqrt(5.25) * (math.pi - 1e-3)
    shape = torch.randn(P, 10, generator=g).double()
    expr = (torch.randn(P, 10, generator=g) * 0.5).double()
    loc = (torch.rand(P, 2, generator=g) * 200 + 10).double()
    dist = (torch.rand(P, generator=g) * 5 + 1.5).double()
    K = synth.make_cameras(P, 224, jitter=True, seed=P).double()
    shim = smplx_ref.SMPLXShim(bm, 10).double()
    up = {k: v.double() for k, v in bg.upstream(P, 10475, 127, g, "all").items()}

    def f(rotvec, shape, loc, dist, expr):
        out = multihmr_ref.smpl_layer_forward(shim, rotvec, shape, loc, dist[:, None], K, expr, 15)
        out["transl_pelvis"] = out["transl_pelvis"][:, 0]
        return sum((out[k] * up[k]).sum() for k in up)

    coords = [_pose_coords(53, [0, 3, 4, 52, 53, 56, 57], g), list(range(10 * P)), list(range(2 * P)),
              list(range(P)), list(range(0, 10 * P, 3))]
    print(f"placed: worst relative deviation {_check(f, [rotvec, shape, loc, dist, expr], coords):.2e}")
    ref = multihmr_ref.smpl_layer_forward(shim, rotvec, shape, loc, dist[:, None], K, expr, 15)
    mine = bg.placed_outputs(bm, rotvec, shape, loc, dist, K, expr)
    for k in mine:
        r = ref[k][:, 0] if k == "transl_pelvis" else ref[k]
        assert (r - mine[k]).abs().max().item() < 1e-9, k
