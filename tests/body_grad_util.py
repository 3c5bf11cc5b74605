"""fp64 autograd references of the body-model backward (mhmr_body_backward / mhmr_smplx_backward): the raw smplx
body model (oracle/smplx_ref.lbs) and the placed SMPL-X layer (oracle/multihmr_ref.smpl_layer_forward), restated with
switches that plant the mistakes the GPU tests must detect, plus the inputs and the error bound shared by the tests."""
import math

import torch

from oracle import multihmr_ref, roma_ref, smplx_ref

U = 2.0 ** -24
# The gradient kernels' structure (smplx_lbs.cu), which the per-element bound below restates:
GTV = 80              # vertices per tile of body_grad_stream_kernel (kGTV)
GTC = 3 * GTV         # 240 PDX columns per tile (kGTC)
G_LANES = 8           # interleaved partial sums of each g_cf dot product over the tile's columns (s8), then a 3-level tree
G_SPLIT = 4           # interleaved partial sums of each per-tile vertex sum (s4, vertex v into v & 3), then a 2-level tree
GPB = 16              # persons per pass over a tile's PDX slab (kGPB), SMPL and SMPL-X
GROWS = 16            # PDX rows per staged chunk (kGRows)
GSTAGES = 3           # depth of the cp.async ring (kGStages)
KT_MAX = 512          # coefficient rows at most (kKTMax)
BETA_MAX = 32         # shape coefficients at most in the person kernel (beta[32])
TAYLOR_BELOW = 0.5    # rotvec_grad: A, B, A', B' from their 4-term Taylor series below this angle
TAYLOR_TRUNC = 1e-9   # ... whose truncation is below this at TAYLOR_BELOW (test_body_grad_bound_cpu checks it)
ROMA_FIRST_ORDER = 1e-6  # placed root: roma's first-order rotation I + K(r) below this angle
RODRIGUES_EPS = 1e-8  # smplx.batch_rodrigues: angle = ||r + 1e-8||


def _rodrigues(r, transpose_grad):
    R = smplx_ref.batch_rodrigues(r)
    if transpose_grad:  # same values, derivative of R^T
        Rt = R.transpose(1, 2)
        R = R.detach() + (Rt - Rt.detach())
    return R


def body(bm, full_pose, comps, dirs, *, no_posedirs=False, j_const=False, parent_swap=None, rod_t=False,
         no_scatter=False, last_tile=False, last_coef_row=False, lmk_corner=False, extra_last_vertex=False,
         leaf_parent=False):
    """smplx forward (no transl): vertices [P,V,3] and joints [P, NJ + 21 (+ 51), 3], dtype of the inputs.
    comps = [betas | expression], dirs = the matching [V,3,L] directions.  The switches plant mistakes of the
    backward (same values, wrong derivative unless noted):
      no_posedirs, j_const, rod_t, no_scatter: pose correctives dropped (values too), J(beta) constant, Rodrigues
        transposed, no vertex -> joint scatter;  parent_swap=j / leaf_parent: joint j (the last joint, a leaf) hangs
        from its grandparent (values too);
      last_tile: the vertices of the last GTV-vertex tile pass no gradient (to any output);
      last_coef_row: the last coefficient (last expression, or last beta without expressions) loses its blend-shape
        gradient and keeps its J(beta) part;
      lmk_corner: the first barycentric corner of landmark 0 is not scattered;
      extra_last_vertex: a vertex-picked joint on vertex V - 1 is not scattered."""
    dt, dev = comps.dtype, comps.device
    d = lambda k: torch.as_tensor(bm[k]).to(dev, dt)
    P = comps.shape[0]
    blend = lambda c: d("v_template") + torch.einsum("bl,mkl->bmk", c, dirs)
    v_shaped = blend(comps)
    Jr = d("J_regressor")
    J = torch.einsum("bik,ji->bjk", v_shaped.detach() if j_const else v_shaped, Jr)
    if last_coef_row:
        v_shaped = blend(torch.cat([comps[:, :-1], comps[:, -1:].detach()], 1))
    NJ = Jr.shape[0]
    rot = _rodrigues(full_pose.reshape(-1, 3), rod_t).view(P, NJ, 3, 3)
    pf = (rot[:, 1:] - torch.eye(3, dtype=dt, device=dev)).reshape(P, -1)
    v_posed = v_shaped if no_posedirs else v_shaped + (pf @ d("posedirs")).view(P, -1, 3)
    parents = torch.as_tensor(bm["parents"]).long().clone()
    if leaf_parent:
        parent_swap = NJ - 1
    if parent_swap is not None:
        parents[parent_swap] = parents[parents[parent_swap]]
    J_posed, A = smplx_ref.batch_rigid_transform(rot, J, parents)
    T = (d("lbs_weights") @ A.view(P, NJ, 16)).view(P, -1, 4, 4)
    homo = torch.cat([v_posed, torch.ones_like(v_posed[..., :1])], 2)
    verts = (T @ homo.unsqueeze(-1))[:, :, :3, 0]
    V = verts.shape[1]
    if last_tile:
        v0 = (V - 1) // GTV * GTV
        verts = torch.cat([verts[:, :v0], verts[:, v0:].detach()], 1)
    vs = verts.detach() if no_scatter else verts
    extra = torch.as_tensor(bm["extra_joints_idxs"]).long()
    picked = vs[:, extra]
    if extra_last_vertex:
        picked = torch.where((extra == V - 1).to(dev)[None, :, None], picked.detach(), picked)
    joints = [J_posed, picked]
    if "lmk_faces_idx" in bm and NJ == 55:
        tri = torch.as_tensor(bm["faces"]).long().to(dev)[torch.as_tensor(bm["lmk_faces_idx"]).long().to(dev)]
        bary = d("lmk_bary_coords")
        lmk = smplx_ref.vertices2landmarks(vs, torch.as_tensor(bm["faces"]).long().to(dev),
                                           torch.as_tensor(bm["lmk_faces_idx"]).long().to(dev), bary)
        if lmk_corner:
            c = bary[0, 0] * vs[:, tri[0, 0]]
            lmk = torch.cat([(lmk[:, 0] - c + c.detach()).unsqueeze(1), lmk[:, 1:]], 1)
        joints.append(lmk)
    return verts, torch.cat(joints, 1)


def edge_body(kind, nb, V=None):
    """body_forward_util.random_body (or exact_body's tables at V vertices) with vertex-picked joint 0 on vertex V - 1
    and (SMPL-X) landmark 0 on the face (V - 1, 0, 1): the shapes where the last tile's scatter entries matter."""
    import body_forward_util as bf

    bm = bf.random_body(kind, nb) if V is None else bf.exact_body(kind, V, nb)
    V = torch.as_tensor(bm["v_template"]).shape[0]
    ex = torch.as_tensor(bm["extra_joints_idxs"]).clone()
    ex[0] = V - 1
    bm["extra_joints_idxs"] = ex
    if kind == "smplx":
        faces = torch.as_tensor(bm["faces"]).clone()
        faces[int(torch.as_tensor(bm["lmk_faces_idx"])[0])] = torch.tensor([V - 1, 0, 1])
        bm["faces"] = faces
    return bm


def num_output_joints(kind):
    return (24 if kind == "smpl" else 55) + 21 + (51 if kind == "smplx" else 0)


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


# ------------------------------------------------------------------------------------------------ per-element bound
class Ev:
    """An fp64 intermediate of the backward: value v, sum of the magnitudes of its terms s (>= |v|) and a bound e on
    the error of the device's fp32 value."""
    __slots__ = ("v", "s", "e")

    def __init__(self, v, s=None, e=None):
        self.v = v
        self.s = v.abs() if s is None else s
        self.e = torch.zeros_like(v) if e is None else e.expand_as(v).clone()

    def __getitem__(self, i):
        return Ev(self.v[i], self.s[i], self.e[i])

    def __neg__(self):
        return Ev(-self.v, self.s, self.e)


def _dot(eq, a, b, n):
    """einsum(eq, a, b) as n-term fp32 dot products (n roundings on each term's running sum)."""
    es = lambda x, y: torch.einsum(eq, x, y)
    s = es(a.s, b.s)
    e = es(a.e, b.s + b.e) + es(a.s, b.e)
    return Ev(es(a.v, b.v), s, e + n * U * (s + e))


def _add(a, b, rounded=True):
    s, e = a.s + b.s, a.e + b.e
    return Ev(a.v + b.v, s, e + (U * (s + e) if rounded else 0.0))


def _seq(x, dim, start=None):
    """Sequential fp32 sum of the terms x along dim (fmaf of exact products, or plain sums), onto `start` if given.
    Every step rounds by at most u times its computed running value, which is within the partial sums' accumulated
    errors of the exact partial sum (Wilkinson's running error bound); n steps: the rounding total R satisfies
    R <= u sum_k (|s_k| + e_k) + n u R."""
    vr, er = x.v.cumsum(dim), x.e.cumsum(dim)
    v, s = vr.select(dim, -1), x.s.sum(dim)
    if start is not None:
        vr, er = vr + start.v.unsqueeze(dim), er + start.e.unsqueeze(dim)
        v, s = v + start.v, s + start.s
    n = x.v.shape[dim]
    rnd = U * (vr.abs() + er).sum(dim) / (1 - 2 * n * U)
    return Ev(v, s, er.select(dim, -1) + rnd)


def _proj_grad(o, do, K, g):
    """body_grad_joints_kernel / the stream kernel's proj_grad at the device's camera-space point o (error do per
    coordinate): d<g, K[:2] (o / o_z)>/do."""
    K = K.to(o.dtype)
    z = o[..., 2]
    den = z.abs() - do
    kk = lambda r, c: K[:, r, c].view(-1, *([1] * (g.dim() - 2)))
    gu = kk(0, 0) * g[..., 0] + kk(1, 0) * g[..., 1]
    gw = kk(0, 1) * g[..., 0] + kk(1, 1) * g[..., 1]
    gus = (kk(0, 0) * g[..., 0]).abs() + (kk(1, 0) * g[..., 1]).abs()
    gws = (kk(0, 1) * g[..., 0]).abs() + (kk(1, 1) * g[..., 1]).abs()
    num = gu * o[..., 0] + gw * o[..., 1]
    nums = gus * o[..., 0].abs() + gws * o[..., 1].abs()
    enum = 2 * U * (gus * o[..., 0].abs() + gws * o[..., 1].abs()) + (gus + gws) * do + 2 * U * nums
    v = torch.stack([gu / z, gw / z, -num / z ** 2], -1)
    s = torch.stack([gus / den, gws / den, nums / den ** 2], -1)
    exy = lambda a: 2 * U * a / den + a * do / (z.abs() * den) + 2 * U * a / den
    ez = enum / den ** 2 + nums * (2 * z.abs() * do + do ** 2) / (z ** 2 * den ** 2) + 3 * U * nums / den ** 2
    return Ev(v, s, torch.stack([exy(gus), exy(gws), ez], -1))


def _rot_coefs(a, taylor):
    """A, B, A', B' of rotvec_grad at the angle a: the 4-term series where `taylor`, else the closed forms."""
    a2 = a * a
    ser = (1 - a2 / 6 * (1 - a2 / 20 * (1 - a2 / 42 * (1 - a2 / 72))),
           0.5 * (1 - a2 / 12 * (1 - a2 / 30 * (1 - a2 / 56 * (1 - a2 / 90)))),
           -a / 3 * (1 - a2 / 10 * (1 - a2 / 28 * (1 - a2 / 54))),
           -a / 12 * (1 - a2 / 15 * (1 - a2 * (3 / 112) * (1 - a2 / 67.5))))
    ac = torch.where(taylor, torch.ones_like(a), a)
    s, c, omc = torch.sin(ac), torch.cos(ac), 2 * torch.sin(0.5 * ac) ** 2
    clo = (s / ac, omc / ac ** 2, (ac * c - s) / ac ** 2, (ac * s - 2 * omc) / ac ** 3)
    # rounding of the fp32 evaluation: the series 16 u of the value; the closed forms sinf / cosf within 2 ulp, and
    # a cos a - sin a, a sin a - 2 (1 - cos a) within 16 u of their terms (they cancel near a = 0.5)
    rc = (8 * U * s.abs() / ac, 16 * U * omc / ac ** 2, 16 * U * ((ac * c).abs() + s.abs()) / ac ** 2,
          16 * U * ((ac * s).abs() + 2 * omc) / ac ** 3)
    val = [torch.where(taylor, x, y) for x, y in zip(ser, clo)]
    err = [torch.where(taylor, 16 * U * x.abs() + TAYLOR_TRUNC * (2 * a) ** 8, y + 4 * U * z.abs())
           for x, y, z in zip(ser, rc, clo)]
    return val, err


def _rotvec_grad(r, g, eps, roma):
    """rotvec_grad: d<g, R(r)>/dr, r [...,3] (exact fp32 values), g Ev [...,3,3] (R's gradient)."""
    gv = g.v.flatten(-2)
    gs, ge_ = g.s.flatten(-2), g.e.flatten(-2)
    idx = ((7, 5), (2, 6), (3, 1))  # <g, K(e_k)> = g[i] - g[j]
    ge = Ev(torch.stack([gv[..., i] - gv[..., j] for i, j in idx], -1),
            torch.stack([gs[..., i] + gs[..., j] for i, j in idx], -1),
            torch.stack([ge_[..., i] + ge_[..., j] for i, j in idx], -1))
    ge.e = ge.e + U * (ge.s + ge.e)
    e = r + eps
    a = e.norm(dim=-1)
    da = (4 if eps else 3) * U * a + (U * e.abs().norm(dim=-1) if eps else 0.0)  # r + eps, the squares, sqrtf
    taylor = a < TAYLOR_BELOW
    (A, B, Ap, Bp), (eA, eB, eAp, eBp) = _rot_coefs(a, taylor)
    # the angle's error moves every coefficient by at most |coef'| da; |coef'| <= 1 for all four at any a
    eA, eB, eAp, eBp = (x + da for x in (eA, eB, eAp, eBp))
    z = torch.zeros_like(r[..., 0])
    Kr = torch.stack([z, -r[..., 2], r[..., 1], r[..., 2], z, -r[..., 0], -r[..., 1], r[..., 0], z], -1).view(
        *r.shape[:-1], 3, 3)
    KK = Kr @ Kr
    KKs = Kr.abs() @ Kr.abs()
    gK = Ev((gv * Kr.flatten(-2)).sum(-1), (gs * Kr.flatten(-2).abs()).sum(-1),
            (ge_ * Kr.flatten(-2).abs()).sum(-1))
    gK.e = gK.e + 9 * U * gK.s
    gKK = Ev((gv * KK.flatten(-2)).sum(-1), (gs * KKs.flatten(-2)).sum(-1), (ge_ * KKs.flatten(-2)).sum(-1))
    gKK.e = gKK.e + 12 * U * gKK.s
    E = torch.zeros(3, 3, 3, dtype=r.dtype, device=r.device)
    for k, (i, j) in enumerate(idx):
        E[k].view(-1)[i], E[k].view(-1)[j] = 1.0, -1.0
    M = torch.einsum("kmq,...qn->...kmn", E, Kr) + torch.einsum("...mq,kqn->...kmn", Kr, E)
    Ms = torch.einsum("kmq,...qn->...kmn", E.abs(), Kr.abs()) + torch.einsum("...mq,kqn->...kmn", Kr.abs(), E.abs())
    gM = Ev(torch.einsum("...mn,...kmn->...k", g.v, M), torch.einsum("...mn,...kmn->...k", g.s, Ms),
            torch.einsum("...mn,...kmn->...k", g.e, Ms))
    gM.e = gM.e + 10 * U * gM.s
    dadr = torch.where(a[..., None] > 0, e / a.clamp_min(1e-300)[..., None], torch.zeros_like(e))
    edadr = 5 * U * dadr.abs()
    t1 = Ap * gK.v + Bp * gKK.v
    t1s = Ap.abs() * gK.s + Bp.abs() * gKK.s
    t1e = Ap.abs() * gK.e + Bp.abs() * gKK.e + eAp * (gK.s + gK.e) + eBp * (gKK.s + gKK.e)
    v = dadr * t1[..., None] + A[..., None] * ge.v + B[..., None] * gM.v
    s = dadr.abs() * t1s[..., None] + A.abs()[..., None] * ge.s + B.abs()[..., None] * gM.s
    err = (dadr.abs() * t1e[..., None] + edadr * (t1s + t1e)[..., None] + A.abs()[..., None] * ge.e
           + eA[..., None] * (ge.s + ge.e) + B.abs()[..., None] * gM.e + eB[..., None] * (gM.s + gM.e))
    err = err + 5 * U * (s + err)
    if roma:  # first order below ROMA_FIRST_ORDER: <g, K(e_k)>
        small = (a < ROMA_FIRST_ORDER)[..., None]
        v, s, err = (torch.where(small, x, y) for x, y in ((ge.v, v), (ge.s, s), (ge.e, err)))
    return Ev(v, s, err)


def _pad_tiles(t, n, per_tile, dim=0):
    """t with dimension `dim` (n entries) zero-padded to whole tiles of `per_tile` and split into [tiles, per_tile]."""
    tiles = (n + per_tile - 1) // per_tile
    pad = tiles * per_tile - n
    if pad:
        shape = list(t.shape)
        shape[dim] = pad
        t = torch.cat([t, t.new_zeros(shape)], dim)
    return t.unflatten(dim, (tiles, per_tile))


def _tile_rounding(part):
    """Rounding of the person kernel's tile sum (from 0, in tile order) of the partials part [tiles, ...]."""
    return part.cumsum(0).abs().sum(0)


def _vertex_sum(W, x):
    """sum_v W[v, j] x[p, v, ...] as the stream kernel computes it: per tile G_SPLIT interleaved fmaf chains (vertex v
    into chain v & 3), a 2-level tree, then the person kernel's tile sum; every rounding bounded by u times the exact
    running value plus the errors carried in.  W [V, NW] exact, x Ev [P, V, ...] -> Ev [P, NW, ...]."""
    P, V = x.v.shape[:2]
    F = x.v[0, 0].numel()
    Wa = W.abs()
    v = torch.einsum("vj,pvf->pjf", W, x.v.reshape(P, V, F))
    s = torch.einsum("vj,pvf->pjf", Wa, x.s.reshape(P, V, F))
    e = torch.einsum("vj,pvf->pjf", Wa, x.e.reshape(P, V, F))
    tiles = (V + GTV - 1) // GTV
    rnd = torch.empty_like(v)
    for p in range(P):
        t = _pad_tiles(W[:, :, None] * x.v[p].reshape(V, 1, F), V, GTV)   # [tiles, GTV, NW, F]
        t = t.unflatten(1, (GTV // G_SPLIT, G_SPLIT))                      # [tiles, step, chain, NW, F]
        cs = t.cumsum(1)
        lane = cs[:, -1]
        tree = (lane[:, 0] + lane[:, 1]).abs() + (lane[:, 2] + lane[:, 3]).abs() + lane.sum(1).abs()
        rnd[p] = cs.abs().sum((0, 1, 2)) + tree.sum(0) + _tile_rounding(lane.sum(1))
    steps = GTV // G_SPLIT + 2 + tiles
    e = e + U * (rnd + steps * e) / (1 - 2 * steps * U)
    shape = x.v.shape[2:]
    return Ev(v.reshape(P, -1, *shape), s.reshape(P, -1, *shape), e.reshape(P, -1, *shape))


def _coef_grad(PDX, gvp):
    """g_cf = PDX . g_vposed as the stream kernel computes it: per (row, tile) G_LANES interleaved fmaf chains over the
    tile's GTC columns (column c into chain c % 8), a 3-level tree, then the tile sum.  PDX [KT, 3V] exact, gvp Ev
    [P, V, 3] -> Ev [P, KT]."""
    P = gvp.v.shape[0]
    KT, C = PDX.shape
    Pa = PDX.abs()
    flat = lambda t: t.reshape(P, C)
    v, s, e = flat(gvp.v) @ PDX.t(), flat(gvp.s) @ Pa.t(), flat(gvp.e) @ Pa.t()
    tiles = (C + GTC - 1) // GTC
    rnd = torch.empty_like(v)
    for p in range(P):
        t = _pad_tiles(PDX * flat(gvp.v)[p], C, GTC, 1).unflatten(2, (GTC // G_LANES, G_LANES))  # [KT, tile, step, lane]
        cs = t.cumsum(2)
        ln = cs[:, :, -1]
        a = ln[..., 0::2] + ln[..., 1::2]                                # (s0+s1), (s2+s3), (s4+s5), (s6+s7)
        b = a[..., 0::2] + a[..., 1::2]
        tree = a.abs().sum(-1) + b.abs().sum(-1) + b.sum(-1).abs()
        rnd[p] = cs.abs().sum((1, 2, 3)) + tree.sum(1) + _tile_rounding(ln.sum(-1).t())
    steps = GTC // G_LANES + 3 + tiles
    return Ev(v, s, e + U * (rnd + steps * e) / (1 - 2 * steps * U))


def _rodrigues_error(r, eps):
    """Entrywise bound of body_prep_kernel's fp32 Rodrigues (and the person kernel's identical restatement) at the
    exact fp32 rotation vectors r [..., 3]: e = r + eps (u), the angle (sqrtf of 3 squares: 4 u relative), the axis
    r / angle (5 u), sinf / cosf within 2 ulp plus the angle's error times |cos| / |sin|, KK = K K (3 terms, 13 u of
    |K| |K|) and R = I + s K + (1 - c) KK (3 u of its terms)."""
    e = r + eps
    ang = e.norm(dim=-1)
    dang = 4 * U * ang
    safe = torch.where(ang > 0, ang, torch.ones_like(ang))
    ax = torch.where(ang[..., None] > 0, r / safe[..., None], torch.zeros_like(r))
    s, c = torch.sin(ang), torch.cos(ang)
    c1 = 1 - c
    ds = 4 * U * s.abs() + dang * (c.abs() + dang)
    dc1 = 4 * U * c.abs() + dang * (s.abs() + dang) + U * c1.abs()
    z = torch.zeros_like(ax[..., 0])
    K = torch.stack([z, -ax[..., 2], ax[..., 1], ax[..., 2], z, -ax[..., 0], -ax[..., 1], ax[..., 0], z], -1)
    K = K.view(*r.shape[:-1], 3, 3).abs()
    KK = K @ K
    eye = torch.eye(3, dtype=r.dtype, device=r.device)
    s_, c1_ = s.abs()[..., None, None], c1.abs()[..., None, None]
    return (K * ds[..., None, None] + s_ * 5 * U * K + KK * dc1[..., None, None] + c1_ * 13 * U * KK
            + 3 * U * (eye + s_ * K + c1_ * KK))


def _chain_error(rot, eRm, J, dJ, par):
    """Bounds of body_prep_kernel's chain G_j = G_par [R_j | J_j - J_par], as forward_pieces derives them but with each
    joint's own rotation bound: the rotation part's error norm grows by ||dR_j||_F + 9 u per level (rotations have
    norm 1), the translation's by eG_par |t_j| + 2 sqrt(3) dJ + 4 u (sqrt(3) |t_j| + |G_t,par|), and A_j's translation
    G_t - G_R J_j adds eG_j |J_j| + sqrt(3) dJ + 4 u (|G_t,j| + sqrt(3) |J_j|).  Returns (G_R, G_t, eG, dGt, dAt): the
    values [P, NJ, 3, 3] / [P, NJ, 3] and the bounds [P, NJ] per entry / coordinate."""
    s3 = math.sqrt(3.0)
    lvl = eRm.flatten(-2).norm(dim=-1) + 9 * U                     # [P, NJ]
    GR, Gt, eG, dGt, dAt = [], [], [], [], []
    m = lambda t: t.abs().amax(-1)
    for j, p in enumerate(par):
        if p < 0:
            GR.append(rot[:, j]), Gt.append(J[:, j]), eG.append(lvl[:, j]), dGt.append(dJ)
        else:
            t = J[:, j] - J[:, p]
            tn = t.norm(dim=-1)
            GR.append(GR[p] @ rot[:, j])
            Gt.append((GR[p] @ t.unsqueeze(-1)).squeeze(-1) + Gt[p])
            eG.append(eG[p] * (1 + lvl[:, j]) + lvl[:, j])
            dGt.append(dGt[p] + eG[p] * tn + 2 * s3 * dJ + 4 * U * (s3 * tn + m(Gt[p])))
        Jn = J[:, j].norm(dim=-1)
        dAt.append(dGt[j] + eG[j] * Jn + s3 * dJ + 4 * U * (m(Gt[j]) + s3 * Jn))
    return tuple(torch.stack(x, 1) for x in (GR, Gt, eG, dGt, dAt))


def scatter_table(bm, NJ, J, V, dt, dev):
    """The vertex -> output-joint table of smplx_grad_init, dense: M [V, J] and the entries per vertex."""
    M = torch.zeros(V, J, dtype=dt, device=dev)
    cnt = torch.zeros(V, dtype=dt, device=dev)
    for e, v in enumerate(torch.as_tensor(bm["extra_joints_idxs"]).long().tolist()):
        M[v, NJ + e] += 1.0
        cnt[v] += 1
    if J > NJ + 21:
        tri = torch.as_tensor(bm["faces"]).long()[torch.as_tensor(bm["lmk_faces_idx"]).long()]
        bary = torch.as_tensor(bm["lmk_bary_coords"]).double()
        for l in range(tri.shape[0]):
            for f in range(3):
                M[int(tri[l, f]), NJ + 21 + l] += float(bary[l, f])
                cnt[int(tri[l, f])] += 1
    return M, cnt


def backward_bound(bm, args, up, placed=False, center=15):
    """Per-element bound of the fp32 backward (body_grad_joints_kernel, body_grad_stream_kernel,
    body_grad_person_kernel) against the fp64 gradients, by a running-error analysis in the kernels' structure.

    args: fp64 inputs on one device, raw (full_pose [P,NJ,3], betas, transl, K, expression or None) or placed
    (rotvec [P,53,3], shape, loc, dist, K, expression); up: the upstream gradients (fp32 values) by output name.
    Returns (grads, bounds): the restated fp64 gradients and their bounds, raw d_full_pose, d_betas[, d_expression],
    d_transl; placed d_rotvec, d_shape, d_expression, d_loc, d_dist.

    Every intermediate x carries (v, s, e): its value, the sum s of the magnitudes of its terms, and a bound e on the
    device value's error.  A product adds e_a (s_b + e_b) + s_a e_b; a short fp32 sum whose running value is rounded n
    times adds n u (s + e); every long sum (the stream kernel's lane and vertex chains, its trees, the tile sums, the
    KT-row v_posed chain, the transl / g_R_root / J(beta) sums) adds u times the sum of its exact running partial sums
    plus the errors carried in (Wilkinson's running error bound).  The forward quantities the kernels recompute enter
    with bounds at each person's own pose: the rotations entrywise at each angle (_rodrigues_error), the chain in
    body_forward_util.forward_pieces' norm form with each joint's own rotation bound (_chain_error), the skinning
    transforms T = sum_j w_j A_j from those (only non-zero weights round), the rest joints within forward_pieces' dJ
    and, when a 2-D upstream gradient makes the backward re-run the forward, the output points within its dv / dj.
    u = 2^-24.  The stages:

      1. gJ = g_j3d + proj^T g_j2d (+ g_transl_pelvis): proj_grad in a few roundings of its terms, and the point's
         error through 1/z and 1/z^2 (|z| - d in the denominators).
      2. g_o = g_v3d + proj^T g_v2d + sum_e w_e gJ_e over the vertex -> joint table: one fmaf per entry.
      3. g_x = R_root^T g_o (placed; raw: R = I, exact), 3 terms, R within eR.
      4. g_vposed = T_R^T g_x, 3 terms, T_R within dTR.
      5. g_cf_k = PDX_k . g_vposed per tile: G_LANES interleaved fmaf chains of GTC / G_LANES columns, then a 3-level
         tree (column c of a tile is rounded 30 - c // 8 + 3 times); the tile partials summed in tile order.
      6. v_posed (the stream's own) = v_template + sum_k cf_k PDX_k, one fmaf chain over the KT rows (row k rounded
         KT - k times), pose features R_j - I within eR + u.
      7. g_A_j = sum_i w_ij g_x_i [v_posed_i; 1]^T, sum_i g_o_i and sum_i g_o_i q_i^T (q = T [v_posed; 1], 4 terms):
         G_SPLIT interleaved fmaf chains per tile (vertex v rounded in the rest of its chain and the 2-level tree),
         then the tile sum.
      8. Placement: transl's gradient S = sum g_o + sum_j gJ_j (NJ more additions); placed: g_R_root = sum g_o q^T -
         (sum g_o) J_c^T + sum_j gJ_j (G_t,j - J_c)^T, g_centre = -R^T S, the cofactor inverse of K within 16 u of
         |K^-1|, loc / dist in 6 roundings of their terms.
      9. A -> (g_G, g_J): g_G_t = g_x + g_A_t, g_G_R = g_A_R - g_A_t J^T (one fmaf), g_J = -G_R^T g_A_t; the chain
         in reverse joint order: g_R_j = G_R,par^T g_G_R,j (3 terms), g_G_R,par += g_G_R,j R_j^T + g_G_t,j t_j^T
         (4 terms and the add), t_j = J_j - J_par, g_J_j / g_J_par -+= G_R,par^T g_G_t,j, g_G_t,par += g_G_t,j;
         pose features g_R_j += g_cf[9 (j - 1):9 j].
     10. rotvec_grad: <g, K(e_k)> and <g, K>, <g, K^2>, <g, E K + K E> in 1, 9, 12 and 10 roundings of their terms;
         A, B, A', B' within 16 u (series, below TAYLOR_BELOW, plus the truncation TAYLOR_TRUNC (2 a)^8) or, above,
         sinf / cosf within 2 ulp and the cancelling numerators a cos a - sin a, a sin a - 2 (1 - cos a) within 16 u of
         their terms; the angle within 4 u (r + 1e-8, squares, sqrtf) moves each coefficient by at most |coef'| da
         <= da; da / dr within 5 u; 5 roundings in the combination.  The placed root below ROMA_FIRST_ORDER:
         <g, K(e_k)> alone.
     11. g_beta_l = g_cf[PF + l] + sum_q Jdirs[q, l] g_J[q], one fmaf chain over the 3 NJ terms; Jdirs is folded at
         load time within (V / 256 + 14) u of sum_v |J_regressor| |dirs|.
    Second-order terms (an error times an error) are kept, so the bound holds for any device value within it of the
    true intermediates, not only to first order."""
    import body_forward_util as bf

    dt = torch.float64
    if placed:
        rotvec, betas, loc, dist, K, expr = args
        P = rotvec.shape[0]
        z = rotvec.new_zeros(P, 1, 3)
        pose = torch.cat([z, rotvec[:, 1:22], rotvec[:, 52:53], z, z, rotvec[:, 22:37], rotvec[:, 37:52]], 1)
        transl = multihmr_ref.inverse_perspective_projection(loc.unsqueeze(1), K, dist.reshape(P, 1, 1))[:, 0]
        Rroot = roma_ref.rotvec_to_rotmat(rotvec[:, 0])
        fw = bf.forward_pieces(bm, pose, torch.cat([betas, expr], -1), betas.shape[1], transl, K,
                               dict(R=Rroot, dtr=bf.transl_bound(loc, dist, K)), center)
    else:
        pose, betas, transl, K, expr = args
        P = pose.shape[0]
        comps = betas if expr is None else torch.cat([betas, expr], -1)
        fw = bf.forward_pieces(bm, pose, comps, betas.shape[1], transl, K)
    dev = pose.device
    d = lambda k: torch.as_tensor(bm[k]).to(dev, dt)
    nb = betas.shape[1]
    dirs = smplx_dirs(bm, nb, dt, dev)
    V, L = dirs.shape[0], dirs.shape[-1]
    NJ = fw["J"].shape[1]
    PF = 9 * (NJ - 1)
    KT = PF + L
    J = fw["j"].shape[1]
    par = [int(x) for x in torch.as_tensor(bm["parents"]).tolist()]
    eR = fw["eR"]
    g = {k: (None if v is None else v.to(dev, dt)) for k, v in up.items()}
    W = d("lbs_weights")
    # the prep kernel's rotations, chain and skinning transforms, entrywise at each angle
    eRm = _rodrigues_error(pose, RODRIGUES_EPS)
    GRv, Gtv, eG, dGt, dAt = _chain_error(fw["rot"], eRm, fw["J"], fw["dJ"], par)
    EG, EGt = eG[..., None, None].expand(P, NJ, 3, 3), dGt[..., None].expand(P, NJ, 3)
    EAt = dAt[..., None].expand(P, NJ, 3)
    Aabs = torch.cat([GRv.abs(), fw["A"][..., :3, 3:].abs()], -1)
    nnz = (W != 0).sum(1).double().view(1, V, 1, 1)  # fmaf(0, a, s) = s: only non-zero weights round
    dT = (torch.einsum("vj,pjrs->pvrs", W, torch.cat([EG, EAt.unsqueeze(-1)], -1))
          + U * nnz * torch.einsum("vj,pjrs->pvrs", W.abs(), Aabs))

    # 1. output joints
    gJ = Ev(g["j3d"] if g.get("j3d") is not None else torch.zeros(P, J, 3, dtype=dt, device=dev))
    if g.get("j2d") is not None:
        gJ = _add(gJ, _proj_grad(fw["j"], fw["dj"], K, g["j2d"]))
    if g.get("transl_pelvis") is not None:
        tp = torch.zeros(P, J, 3, dtype=dt, device=dev)
        tp[:, 0] = g["transl_pelvis"]
        gJ = _add(gJ, Ev(tp))
    # 2. vertex outputs and the scatter
    go = Ev(g["v3d"] if g.get("v3d") is not None else torch.zeros(P, V, 3, dtype=dt, device=dev))
    if g.get("v2d") is not None:
        go = _add(go, _proj_grad(fw["v"], fw["dv"], K, g["v2d"]))
    M, cnt = scatter_table(bm, NJ, J, V, dt, dev)
    sc = lambda x: torch.einsum("vj,pjc->pvc", M, x)
    s, e = go.s + sc(gJ.s), go.e + sc(gJ.e)
    go = Ev(go.v + sc(gJ.v), s, e + U * cnt[None, :, None] * (s + e))
    # 3. g_x
    if placed:
        # roma's formula: the Rodrigues bound with 4 u more for its separate products; exact below 1e-6 rad
        R = Ev(Rroot, Rroot.abs(), _rodrigues_error(rotvec[:, 0], 0.0) + 4 * U * Rroot.abs())
        gq = _dot("prc,pvr->pvc", R, go, 3)
    else:
        gq = go
    # 4. g_vposed
    T = fw["T"]
    TR = Ev(T[..., :3, :3], T[..., :3, :3].abs(), dT[..., :3])
    gvp = _dot("pvrc,pvr->pvc", TR, gq, 3)
    # 5. g_cf
    PDX = torch.cat([d("posedirs"), dirs.reshape(3 * V, L).t()], 0)  # [KT, 3V]
    Pa = PDX.abs()
    gcf = _coef_grad(PDX, gvp)
    # 6. the stream's v_posed
    pf = fw["pf"]
    cf = torch.cat([pf, betas] + ([] if expr is None else [expr]), 1)
    ecf = torch.cat([eRm[:, 1:].reshape(P, PF) + U * pf.abs(), torch.zeros_like(cf[:, PF:])], 1)
    vt = d("v_template")
    rnd = torch.stack([(cf[p, :, None] * PDX).cumsum(0).abs().sum(0) for p in range(P)]).view(P, V, 3)
    vpv = vt + (cf @ PDX).view(P, V, 3)
    e_prop = (ecf @ Pa).view(P, V, 3)
    e_vp = e_prop + U * (rnd + vpv.abs() + (KT + 1) * e_prop) / (1 - 2 * (KT + 1) * U)
    vp = Ev(vpv, vt.abs() + (cf.abs() @ Pa).view(P, V, 3), e_vp)
    # 7. g_A and the placement sums
    one = lambda x: torch.cat([x, torch.ones_like(x[..., :1])], -1)
    vp4 = Ev(one(vp.v), one(vp.s), torch.cat([vp.e, torch.zeros_like(vp.e[..., :1])], -1))
    outer = lambda a, b: Ev(a.v[..., :, None] * b.v[..., None, :], a.s[..., :, None] * b.s[..., None, :],
                            a.e[..., :, None] * (b.s + b.e)[..., None, :] + a.s[..., :, None] * b.e[..., None, :])
    Mv = outer(gq, vp4)
    gA = _vertex_sum(W, Mv)
    ones = torch.ones(V, 1, dtype=dt, device=dev)
    Sv = _vertex_sum(ones, go)[:, 0]
    # 8. placement
    gJk = gJ[:, :NJ]
    S = _seq(Ev(torch.cat([Sv.v[:, None], gJk.v], 1), torch.cat([Sv.s[:, None], gJk.s], 1),
                torch.cat([Sv.e[:, None], gJk.e], 1)), 1)
    Js = Ev(fw["J"], fw["J"].abs(), fw["dJ"].view(P, 1, 1).expand(P, NJ, 3))
    out = {}
    if placed:
        q = Ev((T[..., :3, :3] @ vp.v.unsqueeze(-1)).squeeze(-1) + T[..., :3, 3])
        q.s = (T[..., :3, :3].abs() @ vp.s.unsqueeze(-1)).squeeze(-1) + T[..., :3, 3].abs()
        q.e = ((dT[..., :3] @ (vp.s + vp.e).unsqueeze(-1)).squeeze(-1) + (T[..., :3, :3].abs() @ vp.e.unsqueeze(-1))
               .squeeze(-1) + dT[..., 3] + 4 * U * q.s)
        Mo = _vertex_sum(ones, outer(go, q))[:, 0]
        Gt = Ev(Gtv, Gtv.abs(), EGt)
        Jc = Gt[:, center]
        t0 = Mo.v - Sv.v[:, :, None] * Jc.v[:, None, :]
        t0 = Ev(t0, Mo.s + Sv.s[:, :, None] * Jc.s[:, None, :],
                Mo.e + Sv.e[:, :, None] * (Jc.s + Jc.e)[:, None, :] + Sv.s[:, :, None] * Jc.e[:, None, :])
        diff = Ev(Gt.v - Jc.v[:, None], Gt.s + Jc.s[:, None], Gt.e + Jc.e[:, None])
        diff.e = diff.e + U * (diff.s + diff.e)
        terms = outer(gJk, diff)  # [P, NJ, 3, 3]
        gRr = _seq(terms, 1, start=Ev(t0.v, t0.s, t0.e + U * (t0.s + t0.e)))
        root = _rotvec_grad(rotvec[:, 0], gRr, 0.0, True)
        gcen = -_dot("prc,pr->pc", R, S, 3)
        gt = S if g.get("transl") is None else _add(S, Ev(g["transl"]))
        Ki = torch.inverse(K)
        Kie = 16 * U * Ki.abs()
        Kv = Ev(Ki, Ki.abs(), Kie)
        lp = Ev(torch.cat([loc, torch.ones_like(loc[:, :1])], -1))
        row = _dot("pqc,pc->pq", Kv, lp, 3)  # K^-1 [loc; 1]
        dd = _dot("pq,pq->p", row, gt, 3)
        dd.e = dd.e + 2 * U * (dd.s + dd.e)
        dl = _dot("pqc,pq->pc", Kv, gt, 3)
        dl = _dot("pc,p->pc", dl, Ev(dist), 1)
        out.update(d_loc=dl[:, :2], d_dist=dd)
    else:
        out["d_transl"] = S
    # 9. A -> (g_G, g_J) and the chain
    gx = _dot("prc,pjr->pjc", R, gJk, 3) if placed else gJk
    if placed:
        cen = torch.zeros(P, NJ, 3, dtype=dt, device=dev)
        cen[:, center] = 1.0
        gx = _add(gx, Ev(cen * gcen.v[:, None], cen * gcen.s[:, None], cen * gcen.e[:, None]))
    gAR, gAt = gA[:, :, :, :3], gA[:, :, :, 3]
    gGt = _add(gx, gAt)
    gGR = _add(gAR, -outer(gAt, Js))
    GR = Ev(GRv, GRv.abs(), EG)
    gJl = -_dot("pjrc,pjr->pjc", GR, gAt, 3)
    rot = Ev(fw["rot"], fw["rot"].abs(), eRm)
    lst = lambda x: [x[:, j] for j in range(NJ)]
    gGR, gGt, gJl = lst(gGR), lst(gGt), lst(gJl)
    gR = [None] * NJ
    for j in range(NJ - 1, 0, -1):
        p_ = par[j]
        t = _add(Js[:, j], -Js[:, p_])
        Gp = GR[:, p_]
        gR[j] = _dot("pra,prb->pab", Gp, gGR[j], 3)
        inc = _add(_dot("prm,pcm->prc", gGR[j], rot[:, j], 4), outer(gGt[j], t), rounded=False)
        gGR[p_] = _add(gGR[p_], inc)
        uv = _dot("prc,pr->pc", Gp, gGt[j], 3)
        gJl[j] = _add(gJl[j], uv)
        gJl[p_] = _add(gJl[p_], -uv)
        gGt[p_] = _add(gGt[p_], gGt[j])
    gR[0] = gGR[0]
    gJl[0] = _add(gJl[0], gGt[0])
    for j in range(1, NJ):
        f = slice(9 * (j - 1), 9 * j)
        gR[j] = _add(gR[j], Ev(gcf.v[:, f].view(P, 3, 3), gcf.s[:, f].view(P, 3, 3), gcf.e[:, f].view(P, 3, 3)))
    gRs = Ev(torch.stack([x.v for x in gR], 1), torch.stack([x.s for x in gR], 1), torch.stack([x.e for x in gR], 1))
    rg = _rotvec_grad(pose, gRs, RODRIGUES_EPS, False)
    # 11. g_beta
    Jr = d("J_regressor")
    Jd = torch.einsum("jv,vcl->jcl", Jr, dirs).reshape(NJ * 3, L)
    eJd = (math.ceil(V / 256) + 14) * U * torch.einsum("jv,vcl->jcl", Jr.abs(), dirs.abs()).reshape(NJ * 3, L)
    gJq = Ev(torch.stack([x.v for x in gJl], 1).reshape(P, NJ * 3), torch.stack([x.s for x in gJl], 1).reshape(P, -1),
             torch.stack([x.e for x in gJl], 1).reshape(P, -1))
    terms = Ev(Jd[None] * gJq.v[..., None], Jd.abs()[None] * gJq.s[..., None],
               eJd[None] * (gJq.s + gJq.e)[..., None] + Jd.abs()[None] * gJq.e[..., None])
    gb = _seq(terms, 1, start=gcf[:, PF:])
    out_rot = rg
    if placed:
        src = [-1] + list(range(1, 22)) + [52, -1, -1] + list(range(22, 37)) + list(range(37, 52))
        v = torch.zeros(P, 53, 3, dtype=dt, device=dev)
        bnd = torch.zeros_like(v)
        for j, sj in enumerate(src):
            if sj >= 0:
                v[:, sj], bnd[:, sj] = rg.v[:, j], rg.e[:, j]
        v[:, 0], bnd[:, 0] = root.v, root.e
        out_rot = Ev(v, None, bnd)
    grads = {("d_rotvec" if placed else "d_full_pose"): out_rot.v, ("d_shape" if placed else "d_betas"): gb.v[:, :nb]}
    bounds = {("d_rotvec" if placed else "d_full_pose"): out_rot.e, ("d_shape" if placed else "d_betas"): gb.e[:, :nb]}
    if L > nb:
        grads["d_expression"], bounds["d_expression"] = gb.v[:, nb:], gb.e[:, nb:]
    for k, x in out.items():
        grads[k], bounds[k] = x.v, x.e
    return grads, bounds
