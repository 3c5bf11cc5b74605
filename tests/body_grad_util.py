"""fp64 autograd references of the body-model backward (mhmr_body_backward / mhmr_smplx_backward): the raw smplx
body model (oracle/smplx_ref.lbs) and the placed SMPL-X layer (oracle/multihmr_ref.smpl_layer_forward), restated with
switches that plant the mistakes the GPU tests must detect, plus the inputs and the error bound shared by the tests."""
import math

import torch

from oracle import multihmr_ref, roma_ref, smplx_ref

U = 2.0 ** -24


def _rodrigues(r, transpose_grad):
    R = smplx_ref.batch_rodrigues(r)
    if transpose_grad:  # same values, derivative of R^T
        Rt = R.transpose(1, 2)
        R = R.detach() + (Rt - Rt.detach())
    return R


def body(bm, full_pose, comps, dirs, *, no_posedirs=False, j_const=False, parent_swap=None, rod_t=False,
         no_scatter=False):
    """smplx forward (no transl): vertices [P,V,3] and joints [P, NJ + 21 (+ 51), 3], dtype of the inputs.
    comps = [betas | expression], dirs = the matching [V,3,L] directions."""
    dt, dev = comps.dtype, comps.device
    d = lambda k: torch.as_tensor(bm[k]).to(dev, dt)
    P = comps.shape[0]
    v_shaped = d("v_template") + torch.einsum("bl,mkl->bmk", comps, dirs)
    Jr = d("J_regressor")
    J = torch.einsum("bik,ji->bjk", v_shaped.detach() if j_const else v_shaped, Jr)
    NJ = Jr.shape[0]
    rot = _rodrigues(full_pose.reshape(-1, 3), rod_t).view(P, NJ, 3, 3)
    pf = (rot[:, 1:] - torch.eye(3, dtype=dt, device=dev)).reshape(P, -1)
    v_posed = v_shaped if no_posedirs else v_shaped + (pf @ d("posedirs")).view(P, -1, 3)
    parents = torch.as_tensor(bm["parents"]).long().clone()
    if parent_swap is not None:
        parents[parent_swap] = parents[parents[parent_swap]]
    J_posed, A = smplx_ref.batch_rigid_transform(rot, J, parents)
    T = (d("lbs_weights") @ A.view(P, NJ, 16)).view(P, -1, 4, 4)
    homo = torch.cat([v_posed, torch.ones_like(v_posed[..., :1])], 2)
    verts = (T @ homo.unsqueeze(-1))[:, :, :3, 0]
    vs = verts.detach() if no_scatter else verts
    joints = [J_posed, vs[:, torch.as_tensor(bm["extra_joints_idxs"]).long()]]
    if "lmk_faces_idx" in bm and NJ == 55:
        joints.append(smplx_ref.vertices2landmarks(vs, torch.as_tensor(bm["faces"]).long().to(dev),
                                                   torch.as_tensor(bm["lmk_faces_idx"]).long().to(dev),
                                                   d("lmk_bary_coords")))
    return verts, torch.cat(joints, 1)


def smplx_dirs(bm, nb, dt, dev):
    sd = torch.as_tensor(bm["shapedirs"])
    if sd.shape[-1] < nb:
        sd = torch.cat([sd, torch.as_tensor(bm["shapedirs_extra"])[..., : nb - sd.shape[-1]]], -1)
    sd = sd[..., :nb]
    if "expr_dirs" in bm and torch.as_tensor(bm["parents"]).numel() == 55:
        sd = torch.cat([sd, torch.as_tensor(bm["expr_dirs"])], -1)
    return sd.to(dev, dt)


def raw_outputs(bm, full_pose, betas, transl, K, expression=None, **mistake):
    """mhmr_body_forward's outputs: v3d, v2d, j3d, j2d, transl_pelvis."""
    comps = betas if expression is None else torch.cat([betas, expression], -1)
    v, j = body(bm, full_pose, comps, smplx_dirs(bm, betas.shape[1], betas.dtype, betas.device), **mistake)
    t = transl.unsqueeze(1)
    v, j = v + t, j + t
    pp = multihmr_ref.perspective_projection
    return dict(v3d=v, v2d=pp(v, K), j3d=j, j2d=pp(j, K), transl_pelvis=j[:, 0])


def placed_outputs(bm, rotvec, shape, loc, dist, K, expression, center=15, center_const=False, **mistake):
    """SMPL_Layer.forward (multihmr_ref.smpl_layer_forward) over `body`: v3d, v2d, j3d, j2d, transl,
    transl_pelvis.  dist [P]."""
    P = rotvec.shape[0]
    z = rotvec.new_zeros(P, 1, 3)
    full_pose = torch.cat([z, rotvec[:, 1:22], rotvec[:, 52:53], z, z, rotvec[:, 22:37], rotvec[:, 37:52]], 1)
    dirs = smplx_dirs(bm, shape.shape[1], shape.dtype, shape.device)
    v, j = body(bm, full_pose, torch.cat([shape, expression], -1), dirs, **mistake)
    R = roma_ref.rotvec_to_rotmat(rotvec[:, 0])
    pelvis = j[:, [0]]
    j = (R.unsqueeze(1) @ (j - pelvis).unsqueeze(-1)).squeeze(-1)
    v = (R.unsqueeze(1) @ (v - pelvis).unsqueeze(-1)).squeeze(-1)
    transl = multihmr_ref.inverse_perspective_projection(loc.unsqueeze(1), K, dist.reshape(P, 1, 1))[:, 0]
    c = j[:, [center]]
    c = c.detach() if center_const else c
    v, j = v - c + transl.unsqueeze(1), j - c + transl.unsqueeze(1)
    pp = multihmr_ref.perspective_projection
    return dict(v3d=v, v2d=pp(v, K), j3d=j, j2d=pp(j, K), transl=transl, transl_pelvis=j[:, 0])


def vjp(outputs, grads, inputs):
    """Input gradients of sum_k <grads[k], outputs[k]> (keys absent from grads contribute nothing)."""
    loss = sum((outputs[k] * g.to(outputs[k].device, outputs[k].dtype)).sum() for k, g in grads.items()
               if g is not None)
    gr = torch.autograd.grad(loss, inputs, allow_unused=True, retain_graph=True)
    return [torch.zeros_like(x) if d is None else d for d, x in zip(gr, inputs)]


def poses(P, NJ, g, scale=0.4):
    """Random rotations of scale 0.4 with the special rows the backward must get right: zero rows (flat hands,
    fixed zero joints), |r| = 1e-4 and |r| = pi - 1e-3."""
    r = torch.randn(P, NJ, 3, generator=g) * scale
    unit = lambda n: (lambda x: x / x.norm(dim=-1, keepdim=True))(torch.randn(n, 3, generator=g))
    r[0, NJ // 2:] = 0.0
    if NJ > 4:
        r[:, 3] = unit(P) * 1e-4
        r[:, 4] = unit(P) * (math.pi - 1e-3)
    if P > 1:
        r[1, 1:] = 0.0
    return r


def upstream(P, V, J, g, which, sparse=False):
    """Random upstream gradients for all outputs ('all') or one output alone; 2-D gradients per pixel are scaled
    down by the ~70 px / m of the test cameras so every term carries similar weight.  `sparse`: g_v3d on 64
    vertices only (the sensitivity checks, where the vertex sum would hide the mistake)."""
    shapes = dict(v3d=(P, V, 3), v2d=(P, V, 2), j3d=(P, J, 3), j2d=(P, J, 2), transl_pelvis=(P, 3), transl=(P, 3))
    scale = dict(v2d=1e-2, j2d=1e-2)
    out = {}
    for k, s in shapes.items():
        if which == "all" or which == k:
            out[k] = torch.randn(*s, generator=g) * scale.get(k, 1.0)
    if sparse and "v3d" in out:
        keep = torch.zeros(V, dtype=torch.bool)
        keep[torch.randperm(V, generator=g)[:64]] = True
        out["v3d"] = out["v3d"] * keep[None, :, None]
    return out


def tolerance(ref, ref_abs, n_seq, per_person_rows=True):
    """Per-element bound of an fp32 gradient against the fp64 one.  Every gradient element is a chain of fp32
    sums; the longest is n_seq additions deep (the per-tile vertex sums, the tile sum, the kinematic chain and the
    J(beta) sum), each within one rounding u of its running value, so the error is below n_seq u times the sum of
    the magnitudes of the terms.  That sum is bounded by the person's largest gradient element under |upstream|
    (ref_abs, no sign cancellation in the vertex and joint sums) plus the element itself; a factor 4 covers the
    recomputed forward quantities (v_posed, the skinning transforms, the projection) that enter the products."""
    a = ref_abs.abs().reshape(ref_abs.shape[0], -1)
    row = a.amax(1, keepdim=True) if per_person_rows else a
    return 4 * n_seq * U * (ref.abs().reshape(ref.shape[0], -1) + row).reshape(ref.shape)


def n_seq(V, NJ):
    """Longest fp32 accumulation of the backward (DESIGN.md §9): 60 per-tile vertex terms (4-way split of 80 vertices
    plus the 8-way column split of 240 columns), the tile sum, the chain (NJ joints) and the 3 NJ terms of J(beta)."""
    tiles = (V + 79) // 80
    return 60 + tiles + NJ + 3 * NJ
