"""Body models, inputs and the error bound of the body-model forward tests (mhmr_body_forward, mhmr_smplx_forward).

Exact bodies: every table on a dyadic grid (v_template, shapedirs, expr_dirs, posedirs, transl on multiples of 2^-10;
J_regressor rows 1/2, 1/4, 1/4 of three vertices; skinning weights 1/2, 1/4, 1/8, 1/8; landmark barycentrics 1/2,
1/4, 1/4), integer betas and expressions, zero full pose.  Rodrigues of a zero rotation is I exactly, the kinematic
chain telescopes to [I | J_j] and every skinning transform is [I | 0], so each sum of the forward is exact in fp32 and
the device's v3d / j3d / transl_pelvis equal the fp64 reference bit for bit.

Random bodies: `forward_bound` bounds each output element of the fp32 forward against the fp64 reference from the
kernels' accumulation lengths (smplx_lbs.cu); `mistaken_reference` plants the mistakes the bound must expose."""
import math

import torch

import body_grad_util as bg
from oracle import multihmr_ref, roma_ref, smplx_ref

U = 2.0 ** -24
GRID = 2.0 ** -10
TV = 72                               # vertices per CTA of the vertex kernel (smplx_lbs.cu kTV)
PB = {"smpl": 8, "smplx": 16}         # persons per pass over the coefficient matrix
NJ = {"smpl": 24, "smplx": 55}
V_REAL = {"smpl": 6890, "smplx": 10475}
NB_EDGES = {"smpl": (1, 10, 32), "smplx": (1, 11, 16)}   # KT = 208 / 217 / 239 and 497 / 507 / 512 rows
CAM = torch.tensor([[256.0, 0.0, 128.0], [0.0, 256.0, 128.0], [0.0, 0.0, 1.0]])


def persons_sweep(kind):
    pb = PB[kind]
    return (1, pb - 1, pb, pb + 1, 2 * pb + 1, 80)


def parents(kind):
    from multihmr_b200 import synth

    return list(synth.SMPL_PARENTS if kind == "smpl" else synth.SMPLX_PARENTS)


def exact_body(kind, V, nb, seed=0):
    """Dyadic body-model dict of V >= 3 vertices and nb shape directions (see the module docstring)."""
    g = torch.Generator().manual_seed(seed)
    nj = NJ[kind]
    grid = lambda m, *s: (torch.randint(-m, m + 1, s, generator=g).double() * GRID).float()
    bm = {"v_template": grid(256, V, 3), "shapedirs": grid(16, V, 3, nb), "posedirs": grid(16, 9 * (nj - 1), 3 * V)}
    pick = lambda n, k: torch.argsort(torch.rand(n, V if k == 3 else nj, generator=g), 1)[:, :k]
    Jr = torch.zeros(nj, V)
    Jr.scatter_(1, pick(nj, 3), torch.tensor([0.5, 0.25, 0.25]).expand(nj, 3).contiguous())
    W = torch.zeros(V, nj)
    W.scatter_(1, pick(V, 4), torch.tensor([0.5, 0.25, 0.125, 0.125]).expand(V, 4).contiguous())
    bm.update(J_regressor=Jr, lbs_weights=W, parents=torch.tensor(parents(kind), dtype=torch.int64))
    extra = torch.randint(0, V, (21,), generator=g)
    extra[0], extra[1] = V - 1, 0
    bm["extra_joints_idxs"] = extra
    if kind == "smplx":
        bm["expr_dirs"] = grid(16, V, 3, 10)
        F = 64
        bm["faces"] = torch.argsort(torch.rand(F, V, generator=g), 1)[:, :3]
        bm["faces"][0] = torch.tensor([V - 1, 0, 1])
        bm["lmk_faces_idx"] = torch.randint(0, F, (51,), generator=g)
        bm["lmk_faces_idx"][0] = 0
        bary = torch.tensor([[0.5, 0.25, 0.25], [0.25, 0.5, 0.25], [0.25, 0.25, 0.5]])
        bm["lmk_bary_coords"] = bary[torch.randint(0, 3, (51,), generator=g)]
    return bm


def exact_inputs(kind, P, nb, seed=0):
    """Zero full pose, integer betas / expressions in [-3, 3], transl on the grid with z in [4, 5]."""
    g = torch.Generator().manual_seed(1000 + seed)
    pose = torch.zeros(P, NJ[kind], 3)
    betas = torch.randint(-3, 4, (P, nb), generator=g).float()
    transl = torch.randint(-256, 257, (P, 3), generator=g).float() * GRID
    transl[:, 2] = 4.0 + torch.randint(0, 1025, (P,), generator=g).float() * GRID
    expr = torch.randint(-3, 4, (P, 10), generator=g).float() if kind == "smplx" else None
    return pose, betas, transl, CAM.repeat(P, 1, 1), expr


def random_body(kind, nb, seed=0):
    """synth's SMPL / SMPL-X body model at its real size with shapedirs extended to nb directions."""
    from multihmr_b200 import synth

    bm = dict(synth.make_body_model(seed) if kind == "smplx" else synth.make_smpl_body_model(seed, "male"))
    sd = torch.as_tensor(bm["shapedirs"])
    if kind == "smplx":
        sd = torch.cat([sd, torch.as_tensor(bm["shapedirs_extra"])], -1)
    if sd.shape[-1] < nb:
        g = torch.Generator().manual_seed(5000 + seed)
        sd = torch.cat([sd, torch.randn(sd.shape[0], 3, nb - sd.shape[-1], generator=g) * 0.01], -1)
    bm["shapedirs"] = sd[..., :nb].contiguous()
    return bm


def random_inputs(kind, P, nb, seed=0):
    """bg.poses (zero rows, |r| = 1e-4, |r| = pi - 1e-3) with a non-zero global orient and, from person 2 on, the
    last joint turned by ~1.5 rad (its pose features are the last posedirs rows), betas with the last person's x4,
    transl ~6 m ahead."""
    g = torch.Generator().manual_seed(2000 + seed)
    nj = NJ[kind]
    pose = bg.poses(P, nj, g)
    pose[:, 0] = torch.randn(P, 3, generator=g) * 0.8
    pose[2:, nj - 1] = torch.tensor([1.5, 0.0, 0.0]) + torch.randn(P - 2 if P > 2 else 0, 3, generator=g) * 0.1
    betas = torch.randn(P, nb, generator=g)
    betas[-1] *= 4.0
    transl = torch.randn(P, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 6.0])
    K = torch.tensor([[388.0, 0, 224.0], [0, 388.0, 224.0], [0, 0, 1.0]]).repeat(P, 1, 1)
    expr = torch.randn(P, 10, generator=g) * 0.5 if kind == "smplx" else None
    return pose, betas, transl, K, expr


ROOT_SPECIAL = (5e-7, 0.0, 2e-6)  # either side of the placed layer's th < 1e-6 first-order branch


def placed_inputs(P, seed=0):
    from multihmr_b200 import synth

    g = torch.Generator().manual_seed(3000 + seed)
    rotvec = bg.poses(P, 53, g)
    unit = torch.randn(P, 3, generator=g)
    unit = unit / unit.norm(dim=-1, keepdim=True)
    for p in range(P):
        if p % 5 < 3:
            rotvec[p, 0] = unit[p] * ROOT_SPECIAL[p % 5]
    rotvec[2:, 51] = torch.tensor([1.5, 0.0, 0.0])  # last right-hand joint: its features are the last posedirs rows
    shape = torch.randn(P, 10, generator=g)
    shape[-1] *= 4.0
    expr = torch.randn(P, 10, generator=g) * 0.5
    loc = torch.rand(P, 2, generator=g) * 200 + 10
    dist = torch.rand(P, generator=g) * 5 + 1.5
    K = synth.make_cameras(P, 224, jitter=True, seed=P)
    return rotvec, shape, loc, dist, K, expr


# ------------------------------------------------------------------------------------------------ the bound
def projection_bound(o, K, do):
    """Per-element bound of K[:2] . (o / o_z) in fp32 (two quotients, two products, two sums: 4 u of the terms) when
    the camera-space point o carries an error of at most do per coordinate: |d(x / z)| <= (dx + |x / z| dz) /
    (|z| - dz).  o [P,N,3] fp64, K [P,3,3], do [P,N]."""
    K = K.to(o.device, o.dtype)
    z = o[..., 2]
    u, w = o[..., 0] / z, o[..., 1] / z
    den = z.abs() - do
    du, dw = (do + u.abs() * do) / den, (do + w.abs() * do) / den
    out = []
    for r in range(2):
        k0, k1, k2 = (K[:, r, c, None] for c in range(3))
        out.append(k0.abs() * du + k1.abs() * dw + 4 * U * ((k0 * u).abs() + (k1 * w).abs() + k2.abs()))
    return torch.stack(out, -1)


def forward_bound(bm, full_pose, comps, nb, transl, K, placed=None, center=15):
    """Per-element bound of the fp32 forward (body_prep_kernel, smplx_vertex_kernel, smplx_joints_kernel) against
    the fp64 one, from the accumulation lengths of the kernels.  Inputs fp64 on one device: full_pose [P,NJ,3] in
    smplx order, comps = [betas | expression], transl [P,3] (placed: the fp64 transl of loc / dist), K [P,3,3].
    placed = dict(R=root rotations [P,3,3], dtr=[P] bound of the device's transl) for the engine's layer.
    With u = 2^-24 (norms are 2-norms, |.| entries; a rotation, and a row of one, has norm 1):

      * Rodrigues (sqrtf, a quotient per axis component, sinf / cosf within 2 ulp, KK, three sums): the angle within
        3.5 u relative, sin within 15 u and 1 - cos within 12 u absolute (the angle error times ang <= pi), KK within
        12 u, so each entry of R within eR = 72 u.  The same for the placed layer's root rotation.
      * v_posed = v_template + sum_k cf_k PDX_k: each of 8 row lanes sums KT / 8 rows in fp32, 3 shuffle levels and
        the template follow: (KT / 8 + 4) u of sum |terms|, plus eR sum_k<PF |posedirs_k| for the pose features.
      * J = Jt + Jdirs beta, folded at load time (V / 256 terms per thread, 5 shuffle levels, 8 warp partials) and
        L terms per call: dJ = (V / 256 + 14 + L) u of sum_v |J_regressor| |v_shaped terms|.
      * The chain, walked joint by joint: G_j = G_parent [R_j | t_j], t_j = J_j - J_parent.  The rotation part's
        error norm grows by 3 eR + 9 u per level (eG_j = depth_j (3 eR + 9 u)); the translation's by
        eG_parent |t_j| + 2 sqrt(3) dJ + 4 u (sqrt(3) |t_j| + |G_t,parent|).  A_j's translation G_t - G_R J_j adds
        eG_j |J_j| + sqrt(3) dJ + 4 u (|G_t,j| + sqrt(3) |J_j|).
      * Skinning, an NJ-term sum: dT_v = sum_j w_vj dA_j + NJ u max|A|; then q = T [v_posed; 1] (3 terms + 1).
      * Placement: raw, + transl (1 rounding); placed, R (q - pelvis) - R (J_c - pelvis) + transl.
      * Vertex-picked joints copy the vertex; landmarks add 3 barycentric products (3 u).
      * Projection: projection_bound.
    Returns a dict of fp64 bounds shaped like the outputs (v3d, v2d, j3d, j2d, transl_pelvis[, transl])."""
    dt, dev = comps.dtype, comps.device
    d = lambda k: torch.as_tensor(bm[k]).to(dev, dt)
    P = comps.shape[0]
    dirs = bg.smplx_dirs(bm, nb, dt, dev)
    L = dirs.shape[-1]
    vt, posedirs, Jr, W = d("v_template"), d("posedirs"), d("J_regressor"), d("lbs_weights")
    V, nj = vt.shape[0], Jr.shape[0]
    par = [int(x) for x in torch.as_tensor(bm["parents"]).tolist()]
    KT = 9 * (nj - 1) + L
    rot = smplx_ref.batch_rodrigues(full_pose.reshape(-1, 3)).view(P, nj, 3, 3)
    pf = (rot[:, 1:] - torch.eye(3, dtype=dt, device=dev)).reshape(P, -1)
    blend_abs = torch.einsum("bl,mkl->bmk", comps.abs(), dirs.abs())
    v_shaped = vt + torch.einsum("bl,mkl->bmk", comps, dirs)
    v_posed = v_shaped + (pf @ posedirs).view(P, V, 3)
    S_vp = vt.abs() + (pf.abs() @ posedirs.abs()).view(P, V, 3) + blend_abs
    J = torch.einsum("bik,ji->bjk", v_shaped, Jr)
    SJ = torch.einsum("bik,ji->bjk", vt.abs() + blend_abs, Jr.abs()).amax((1, 2))
    Gt, A = smplx_ref.batch_rigid_transform(rot, J, torch.tensor(par))
    T = (W @ A.view(P, nj, 16)).view(P, V, 4, 4)
    q = (T[..., :3, :3] @ v_posed.unsqueeze(-1)).squeeze(-1) + T[..., :3, 3]
    m = lambda t, dims: t.abs().amax(dims)
    n2 = lambda t: t.norm(dim=-1)
    s3 = math.sqrt(3.0)
    eR = 72 * U
    lvl = 3 * eR + 9 * U
    dJ = (math.ceil(V / 256) + 14 + L) * U * SJ
    depth, eG, dGt, dAt = [], [], [], []
    for j, p in enumerate(par):
        depth.append(1 if p < 0 else depth[p] + 1)
        eG.append(depth[j] * lvl)
        if p < 0:
            dGt.append(dJ.clone())
        else:
            t = n2(J[:, j] - J[:, p])
            dGt.append(dGt[p] + eG[p] * t + 2 * s3 * dJ + 4 * U * (s3 * t + m(Gt[:, p], -1)))
        dAt.append(dGt[j] + eG[j] * n2(J[:, j]) + s3 * dJ + 4 * U * (m(Gt[:, j], -1) + s3 * n2(J[:, j])))
    eG = torch.tensor(eG, dtype=dt, device=dev)
    dGt, dAt = torch.stack(dGt, 1), torch.stack(dAt, 1)
    Atm = m(A[:, :, :3, 3], (1, 2))
    dTR = W @ eG + nj * U                                      # [V]
    dTt = dAt @ W.t() + nj * U * Atm[:, None]                  # [P, V]
    dvp = ((KT / 8 + 4) * U * S_vp + eR * posedirs.abs().sum(0).view(V, 3)).amax(-1)
    vp1 = v_posed.abs().sum(-1)
    dq = dTR * vp1 + s3 * dvp + dTt + 4 * U * (vp1 + Atm[:, None])
    tr = transl.unsqueeze(1)
    if placed is None:
        v, jk = q + tr, Gt + tr
        dv, djk = dq + U * m(v, -1), dGt + U * m(jk, -1)
    else:
        R, dtr = placed["R"], placed["dtr"][:, None]
        pel = Gt[:, :1]
        dc = Gt[:, center] - Gt[:, 0]
        cen = (R @ dc.unsqueeze(-1)).squeeze(-1).unsqueeze(1)
        dcen = 3 * eR * n2(dc) + s3 * (dGt[:, center] + dGt[:, 0]) + 4 * U * dc.abs().sum(-1)

        def place(x, dx):
            xp = x - pel
            dxp = dx + dGt[:, :1] + U * m(xp, -1)
            o = (R.unsqueeze(1) @ xp.unsqueeze(-1)).squeeze(-1) - cen + tr
            do = 3 * eR * n2(xp) + s3 * dxp + dcen[:, None] + 4 * U * (xp.abs().sum(-1) + m(cen, -1) + m(tr, -1)) + dtr
            return o, do

        v, dv = place(q, dq)
        jk, djk = place(Gt, dGt)
    extra = torch.as_tensor(bm["extra_joints_idxs"]).long().to(dev)
    joints, dj = [jk, v[:, extra]], [djk, dv[:, extra]]
    if nj == 55:
        tri = torch.as_tensor(bm["faces"]).long()[torch.as_tensor(bm["lmk_faces_idx"]).long()].to(dev)
        lmk = torch.einsum("blfi,lf->bli", v[:, tri], d("lmk_bary_coords"))
        joints.append(lmk)
        dj.append(dv[:, tri].amax(-1) + 3 * U * m(v[:, tri], (-1, -2)))
    j, dj = torch.cat(joints, 1), torch.cat(dj, 1)
    out = dict(v3d=dv.unsqueeze(-1).expand(P, V, 3), v2d=projection_bound(v, K, dv),
               j3d=dj.unsqueeze(-1).expand(*j.shape), j2d=projection_bound(j, K, dj),
               transl_pelvis=dj[:, :1].expand(P, 3))
    if placed is not None:
        out["transl"] = placed["dtr"][:, None].expand(P, 3)
    return out


def transl_bound(loc, dist, K):
    """The engine's transl = (K^-1 [loc; 1]) dist in fp32 by cofactors: 16 u of sum |K^-1| |[loc; 1]| dist."""
    p = torch.cat([loc, torch.ones_like(loc[:, :1])], -1)
    t = (torch.inverse(K).abs() @ p.abs().unsqueeze(-1)).squeeze(-1) * dist.reshape(-1, 1)
    return 16 * U * t.amax(-1)


def raw_reference(bm, pose, betas, transl, K, expr, dev):
    """bg.raw_outputs in fp64 on `dev` and the forward bound for the same inputs."""
    f = lambda t: None if t is None else t.to(dev, torch.float64)
    pose, betas, transl, K, expr = map(f, (pose, betas, transl, K, expr))
    ref = bg.raw_outputs(bm, pose, betas, transl, K, expr)
    comps = betas if expr is None else torch.cat([betas, expr], -1)
    return ref, forward_bound(bm, pose, comps, betas.shape[1], transl, K)


def placed_reference(bm, rotvec, shape, loc, dist, K, expr, dev):
    f = lambda t: t.to(dev, torch.float64)
    rotvec, shape, loc, dist, K, expr = map(f, (rotvec, shape, loc, dist, K, expr))
    ref = bg.placed_outputs(bm, rotvec, shape, loc, dist, K, expr)
    z = rotvec.new_zeros(rotvec.shape[0], 1, 3)
    full = torch.cat([z, rotvec[:, 1:22], rotvec[:, 52:53], z, z, rotvec[:, 22:37], rotvec[:, 37:52]], 1)
    placed = dict(R=roma_ref.rotvec_to_rotmat(rotvec[:, 0]), dtr=transl_bound(loc, dist, K))
    return ref, forward_bound(bm, full, torch.cat([shape, expr], -1), shape.shape[1], ref["transl"], K, placed)


# ------------------------------------------------------------------------------------------------ mistakes
MISTAKES = ("last_pdx_row", "last_posedirs_row", "expr_shift", "second_pass", "last_tile_weights", "root_transposed")


def mistaken_inputs(name, kind, bm, args):
    """The reference's inputs with one mistake planted (None: the mistake is applied to the outputs instead).
    args: raw (pose, betas, transl, K, expr) or placed (rotvec, shape, loc, dist, K, expr) as kind 'placed'."""
    bm, args = dict(bm), [None if a is None else a.clone() for a in args]
    if name == "last_pdx_row":            # the last coefficient row: last expression direction, or last beta
        if kind == "smpl":
            args[1][:, -1] = 0.0
        else:
            args[-1][:, -1] = 0.0
    elif name == "last_posedirs_row":     # row 485 (SMPL-X) / 206 (SMPL) of posedirs
        pd = torch.as_tensor(bm["posedirs"]).clone()
        pd[-1] = 0.0
        bm["posedirs"] = pd
    elif name == "expr_shift":            # expression coefficient e lands in column e + 1
        if kind == "smpl":
            return None
        e = args[-1]
        args[-1] = torch.cat([torch.zeros_like(e[:, :1]), e[:, :-1]], -1)
    elif name == "last_tile_weights":     # the last vertex tile skinned with the previous tile's weights
        W = torch.as_tensor(bm["lbs_weights"]).clone()
        V = W.shape[0]
        v0 = (V - 1) // TV * TV
        W[v0:] = W[v0 - TV:v0 - TV + (V - v0)]
        bm["lbs_weights"] = W
    elif name == "root_transposed":       # R^T of the global orient (raw) / root rotation (placed): r -> -r
        args[0][:, 0] = -args[0][:, 0]
    else:
        return None
    return bm, args


def second_pass_from_first(ref, pb):
    """Outputs whose persons pb .. 2 pb - 1 are those of persons 0 .. pb - 1."""
    out = {}
    for k, t in ref.items():
        t = t.clone()
        n = min(pb, t.shape[0] - pb)
        t[pb:pb + n] = t[:n]
        out[k] = t
    return out


def worst_ratio(got, ref, tol, keys=None):
    """max over elements of |got - ref| / tol per output (fp64)."""
    keys = keys or [k for k in ref if k in got]
    return {k: ((got[k].double().to(ref[k].device) - ref[k]).abs() / tol[k]).max().item() for k in keys}


def project(x, K):
    return multihmr_ref.perspective_projection(x, K.to(x.device, x.dtype))
