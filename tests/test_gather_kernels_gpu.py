"""Index-heavy kernels of the heads (head.cu) through their stage-level entry points, against plain fp64 torch
references: the camera rays of every token, the detection logit, the per-person gathers of the SMPL-X and Anny heads,
the inputs of the central-stream refinement, the value injection at the detected cells, the cls-row gather and the
placement of the Anny body.

Copies and single roundings are compared for exact equality.  Every other comparison states its tolerance next to it,
and every op has a sensitivity check: a reference with one plausible mistake (the (row, col) swap undone, the wrong
table index, the cls offset dropped, the neighbouring cell, ...) must fall outside that tolerance.  The person count is
a device int32 with count < max_persons, and rows at or past count must come back untouched."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # unit roundoff of fp32
SENTINEL = 12345.0
SENTINEL16 = -1234.0  # exact in fp16
PI32 = float(torch.tensor(math.pi, dtype=torch.float32))  # the reference multiplies fp32 rays by np.pi in fp32


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _count(dev, n):
    return torch.tensor([n], dtype=torch.int32, device=dev)


def _report(name, err, tol):
    r = (err / tol).max().item() if err.numel() else 0.0
    print(f"  {name}: worst err/tol {r:.3f} (max err {err.max().item() if err.numel() else 0.0:.2e})")
    return r


def _ulp16(v):
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def _cameras(B, S, g):
    """Asymmetric intrinsics: fx != fy, off-centre principal point with cx != cy."""
    K = torch.zeros(B, 3, 3)
    f = S / (2 * math.tan(math.radians(60) / 2))
    K[:, 0, 0] = f * (0.8 + 0.4 * torch.rand(B, generator=g))
    K[:, 1, 1] = f * (0.8 + 0.4 * torch.rand(B, generator=g))
    K[:, 0, 2] = S / 2 + 0.1 * S * torch.randn(B, generator=g)
    K[:, 1, 2] = S / 2 - 0.07 * S + 0.05 * S * torch.randn(B, generator=g)
    K[:, 2, 2] = 1.0
    return K


def _persons(B, res, n, g, corners=True):
    """n persons in (b, y, x) order over B images, the corner cells of the last image included."""
    cells = set()
    if corners and n >= 4:
        cells |= {(B - 1, 0, 0), (B - 1, 0, res - 1), (B - 1, res - 1, 0), (B - 1, res - 1, res - 1)}
    while len(cells) < n:
        cells.add((int(torch.randint(B, (1,), generator=g)), int(torch.randint(res, (1,), generator=g)),
                   int(torch.randint(res, (1,), generator=g))))
    return sorted(cells)


def _det(cells, Pm, dev):
    t = torch.full((3, max(Pm, 1)), -1, dtype=torch.int32)
    if cells:
        t[:, :len(cells)] = torch.tensor(cells, dtype=torch.int32).t()
    return [x.contiguous().to(dev) for x in t]


def _features(Kinv, gy, gx, freqs, transpose=False):
    """fp64 camera features (model.py:160-187) of cells (gy, gx) [n] with Kinv [n, 3, 3]: the (row, col) grid is fed to
    the un-projection as (x, y), i.e. px = row * 14 + 7.  Also returns the error bound of the fp32 kernel."""
    r, c = ((gx, gy) if transpose else (gy, gx))
    r, c = r.double(), c.double()
    p = torch.stack([r * 14.0 + 7, c * 14.0 + 7, torch.ones_like(r, dtype=torch.float64)], 1)
    ray = torch.einsum("nij,nj->ni", Kinv, p)
    arg = PI32 * ray[:, :, None] * freqs[None, None, :]                     # [n, 3, 16]
    feats = torch.cat([ray, torch.sin(arg).flatten(1), torch.cos(arg).flatten(1)], 1)
    # the ray: three fp32 products and two sums (4 u of sum|Kinv p|); the argument: two fp32 products (2 u) on top of
    # the ray error times pi f; sinf / cosf are within 2 ulp of the exact function (4 u absolute, |value| <= 1)
    dray = 4 * U * torch.einsum("nij,nj->ni", Kinv.abs(), p.abs())
    darg = PI32 * dray[:, :, None] * freqs[None, None, :] + 2 * U * arg.abs()
    tol = torch.cat([dray, (darg + 4 * U).flatten(1), (darg + 4 * U).flatten(1)], 1)
    return feats, tol


FREQS = torch.linspace(1, 32, 16)


# ------------------------------------------------------------------------------------------------------- camera ctx
@pytest.mark.parametrize("res,B", [(16, 2), (92, 2)])
def test_camera_ctx(cuda_device, res, B):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(res * 7 + B)
    K = _cameras(B, res * 14, g)
    col0, pad = 64, 128
    ld = col0 + pad + 8
    N = res * res
    ctx = torch.full((B * N + 1, ld), SENTINEL16, dtype=torch.float16, device=dev)
    kinv = ops.camera_ctx(K.to(dev), FREQS.to(dev), ctx[:B * N], res, col0, pad)
    # K^-1 by cofactors in fp32: componentwise within 32 u (|K^-1| |K| |K^-1|) (first-order perturbation of the inverse
    # for relative errors of a few u in each cofactor and the determinant)
    Kd = K.double()
    ref_inv = torch.linalg.inv(Kd)
    tol_inv = 32 * U * (ref_inv.abs() @ Kd.abs() @ ref_inv.abs())
    err_inv = (kinv.double().cpu() - ref_inv).abs()
    _report(f"invert_K res={res}", err_inv, tol_inv + 1e-30)
    assert torch.all(err_inv <= tol_inv)
    n = torch.arange(N)
    gy, gx = (n // res).repeat(B), (n % res).repeat(B)
    kb = kinv.double().cpu().repeat_interleave(N, 0)  # the kernel's own K^-1: the features are checked on their own
    ref, tol = _features(kb, gy, gx, FREQS.double())
    tol = tol + 0.5 * _ulp16(ref.abs() + tol)  # one fp16 rounding
    got = ctx[:B * N, col0:col0 + 99].double().cpu()
    err = (got - ref).abs()
    _report(f"camera_ctx res={res}", err, tol)
    assert torch.all(err <= tol)
    assert torch.all(ctx[:B * N, col0 + 99:col0 + pad] == 0)                   # pad columns exactly 0
    assert torch.all(ctx[:B * N, :col0] == SENTINEL16) and torch.all(ctx[:B * N, col0 + pad:] == SENTINEL16)
    assert torch.all(ctx[B * N] == SENTINEL16)
    # sensitivity: (row, col) not swapped
    wrong, _ = _features(kb, gy, gx, FREQS.double(), transpose=True)
    assert torch.any((got - wrong).abs() > tol)


# --------------------------------------------------------------------------------------------------- rowdot_sigmoid
# the kernel's clamp bounds: 1e-4f and 1.0f - 1e-4f in fp32
C_LO = float(torch.tensor(1e-4, dtype=torch.float32))
C_HI = float(torch.tensor(1.0) - torch.tensor(1e-4, dtype=torch.float32))


@pytest.mark.parametrize("clamp", [True, False])
@pytest.mark.parametrize("D", [384, 768, 1024])
def test_rowdot_sigmoid(cuda_device, D, clamp):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(D + clamp)
    M, ld = 1001, D + 8
    hid = torch.randn(M, ld, generator=g) * 0.5
    w = torch.randn(D, generator=g) / math.sqrt(D)
    b = torch.tensor([0.3])
    # rows scaled so that their logits reach +-30: the clamp binds there
    lg = hid[:, :D].double() @ w.double()
    target = torch.linspace(-30, 30, M, dtype=torch.float64)
    hid[:, :D] *= (target / lg).clamp(-60, 60).float()[:, None]
    hid = hid.half()
    scores = torch.full((M + 3,), SENTINEL, device=dev)
    logits = torch.full((M + 3,), SENTINEL, device=dev)
    ops.rowdot_sigmoid(hid.to(dev), D, w.to(dev), b.to(dev), scores[:M], logits=logits[:M], clamp=clamp)
    hd, wd = hid[:, :D].double(), w.double()
    l_ref = hd @ wd + float(b)
    # each lane chains 8 products per 256-column step, D/256 steps, then 5 butterfly levels and the bias:
    # depth <= D/32 + 6
    tol_l = (D / 32 + 8) * U * (hd.abs() @ wd.abs()) + U * l_ref.abs()
    err_l = (logits[:M].double().cpu() - l_ref).abs()
    _report(f"rowdot D={D} logits", err_l, tol_l)
    assert torch.all(err_l <= tol_l)
    s = torch.sigmoid(l_ref)
    ref = s.clamp(C_LO, C_HI) if clamp else s
    # sigmoid' = s (1 - s); expf and the division: 4 u relative
    tol = s * (1 - s) * tol_l + 4 * U * s + 1e-45
    got = scores[:M].double().cpu()
    err = (got - ref).abs()
    _report(f"rowdot D={D} clamp={clamp} scores", err, tol)
    assert torch.all(err <= tol)
    assert torch.all(scores[M:] == SENTINEL) and torch.all(logits[M:] == SENTINEL)
    # sensitivity: the clamp applied when it is off / missing when it is on
    wrong = s if clamp else s.clamp(C_LO, C_HI)
    assert torch.any((got - wrong).abs() > tol)


# ---------------------------------------------------------------------------------------------------- person_gather
def _ln_block_tol(xd, g, b, D):
    """LayerNorm of one row by 256 threads (person_gather / anny_gather): sums of depth D/256 + 5 (warp) + 8 (block);
    same structure as the backbone LayerNorm bound (test_backbone_kernels_gpu._ln_tol)."""
    d = D // 256 + 14
    mean = xd.mean(1, keepdim=True)
    var = ((xd - mean) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-6)
    xhat = (xd - mean) * rstd
    dm = d * U * xd.abs().mean(1, keepdim=True)
    return g.abs() * (xhat.abs() * (d + 8) * U + rstd * (dm + U * (xd - mean).abs())) + 3 * U * ((g * xhat).abs() + b.abs())


@pytest.mark.parametrize("refined", [False, True])
@pytest.mark.parametrize("D,P", [(384, 0), (384, 1), (384, 23), (768, 9)])
def test_person_gather(cuda_device, D, P, refined):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(D + P * 3 + refined)
    B, res = 3, 20
    N, C = res * res, D + 99
    ldq, Pm = C + 13, P + 3
    cells = _persons(B, res, P, g)
    det_b, det_y, det_x = _det(cells, Pm, dev)
    z32 = torch.randn(B * N, D, generator=g)
    K = _cameras(B, res * 14, g)
    kinv = torch.linalg.inv(K.double()).float().contiguous()  # linalg.inv returns column-major batches
    tabs = [torch.randn(res, C, generator=g) * 0.2 for _ in range(4)]  # cq_x, cq_y, cv_x, cv_y
    xr = norm = None
    if refined:
        xr = (2.0 + torch.randn(Pm, D, generator=g)).to(dev)
        norm = ((0.5 + torch.rand(D, generator=g)).to(dev), (0.2 * torch.randn(D, generator=g)).to(dev))
    zc = torch.full((Pm, D), SENTINEL, device=dev)
    query = torch.full((Pm, ldq), SENTINEL, device=dev)
    vals = torch.full((Pm, ldq), SENTINEL, device=dev)
    ops.person_gather(z32.to(dev), kinv.to(dev), FREQS.to(dev), *[t.to(dev) for t in tabs], det_b, det_y, det_x,
                      _count(dev, P), Pm, res, zc, query, vals, xr=xr, norm=norm or (None, None))
    for t in (zc, query, vals):
        assert torch.all(t[P:] == SENTINEL)
    assert torch.all(query[:P, C:] == 0) and torch.all(vals[:P, C:] == 0)   # pad columns exactly 0
    if P == 0:
        return
    cq_x, cq_y, cv_x, cv_y = tabs
    bi, yi, xi = (torch.tensor(v) for v in zip(*cells))
    cell = bi * N + yi * res + xi
    got_zc, got_q, got_v = zc[:P].cpu(), query[:P, :C].cpu(), vals[:P, :C].cpu()
    # values: one fp32 addition, as torch does it
    assert torch.equal(got_v, cv_x[yi] + cv_y[xi])
    feats, ftol = _features(kinv.double()[bi], yi, xi, FREQS.double())
    if refined:
        xd = xr[:P].double().cpu()
        gd, bd = (t.double().cpu() for t in norm)
        zref = F.layer_norm(xd, (D,), gd, bd, 1e-6)
        ztol = _ln_block_tol(xd, gd, bd, D)
        err = (got_zc.double() - zref).abs()
        _report(f"person_gather D={D} P={P} refined zc", err, ztol)
        assert torch.all(err <= ztol)
        base, btol = torch.cat([zref, feats], 1), torch.cat([ztol, ftol], 1)
    else:
        assert torch.equal(got_zc, z32[cell])                               # a copy of the cell's feature row
        # feature columns: the same two fp32 additions in the same order as torch
        assert torch.equal(got_q[:, :D], (z32[cell] + cq_x[yi, :D]) + cq_y[xi, :D])
        base, btol = torch.cat([z32[cell].double(), feats], 1), torch.cat([torch.zeros(P, D, dtype=torch.float64),
                                                                           ftol], 1)
    qref = base + cq_x[yi].double() + cq_y[xi].double()
    # the base value's error plus two fp32 additions
    qtol = btol + 2 * U * (base.abs() + cq_x[yi].double().abs() + cq_y[xi].double().abs()) + 1e-30
    err = (got_q.double() - qref).abs()
    _report(f"person_gather D={D} P={P} refined={refined} query", err, qtol)
    assert torch.all(err <= qtol)
    # sensitivity: cross_queries_x indexed by x (and cross_queries_y by y)
    wrong = base + cq_x[xi].double() + cq_y[yi].double()
    assert torch.any((got_q.double() - wrong).abs() > qtol)


def test_person_gather_zero_capacity(cuda_device):
    from multihmr_b200 import ops

    dev = cuda_device
    D, res = 384, 4
    C = D + 99
    det = _det([], 0, dev)
    empty = torch.empty(0, C + 1, device=dev)
    ops.person_gather(torch.zeros(res * res, D, device=dev), torch.eye(3, device=dev)[None], FREQS.to(dev),
                      *[torch.zeros(res, C, device=dev)] * 4, *det, _count(dev, 0), 0, res,
                      torch.empty(0, D, device=dev), empty, empty.clone())


# --------------------------------------------------------------------------------------------------- refine_prepare
@pytest.mark.parametrize("u8", [False, True])
@pytest.mark.parametrize("n_cls,P", [(0, 0), (0, 7), (3, 0), (3, 7)])
def test_refine_prepare(cuda_device, n_cls, P, u8):
    from multihmr_b200 import ops, preprocess

    dev = cuda_device
    g = _gen(n_cls * 10 + P + u8)
    B, S, D, ldp = 3, 280, 384, 596
    res = S // 14
    N, Pm = res * res, P + 2
    cells = _persons(B, res, P, g)
    det_b, det_y, det_x = _det(cells, Pm, dev)
    lut = None
    if u8:
        img = torch.randint(0, 256, (B, S, S, 3), generator=g, dtype=torch.uint8).to(dev)
        lut = torch.from_numpy(preprocess.normalize_rgb_table()).to(dev).contiguous()
        pix = lut[torch.arange(3, device=dev)[None, :, None, None], img.permute(0, 3, 1, 2).long()].cpu()
    else:
        img = torch.randn(B, 3, S, S, generator=g).to(dev)
        pix = img.cpu()
    rowadd = torch.randn(N, D, generator=g)
    cls_pos = torch.randn(D, generator=g)
    R = n_cls + Pm
    rowidx = torch.full((R,), -7, dtype=torch.int32, device=dev)
    patch = torch.full((R, ldp), SENTINEL, device=dev)
    xr = torch.full((R, D), SENTINEL, device=dev)
    rows_out = torch.full((1,), -7, dtype=torch.int32, device=dev)
    ops.refine_prepare(img, rowadd.to(dev), det_b, det_y, det_x, _count(dev, P), Pm, rowidx, patch, xr, lut=lut,
                       n_cls=n_cls, cls_pos=cls_pos.to(dev) if n_cls else None,
                       rows_out=rows_out if n_cls else None)
    rowidx, patch, xr = rowidx.cpu(), patch.cpu(), xr.cpu()
    if n_cls:
        assert rows_out.item() == n_cls + P
        assert torch.equal(rowidx[:n_cls], torch.arange(n_cls, dtype=torch.int32) * (N + 1))
        assert torch.all(patch[:n_cls] == 0) and torch.equal(xr[:n_cls], cls_pos.expand(n_cls, D))
    # untouched past count
    assert torch.all(rowidx[n_cls + P:] == -7) and torch.all(patch[n_cls + P:] == SENTINEL)
    assert torch.all(xr[n_cls + P:] == SENTINEL)
    if P == 0:
        return
    bi, yi, xi = (torch.tensor(v) for v in zip(*cells))
    n = yi * res + xi
    want_idx = (bi * (N + 1) + 1 + n).int()
    got_idx = rowidx[n_cls:n_cls + P]
    assert torch.equal(got_idx, want_idx)                                   # exact
    t = pix.reshape(B, 3, res, 14, res, 14).permute(0, 2, 4, 1, 3, 5).reshape(B, N, 588)
    assert torch.equal(patch[n_cls:n_cls + P, :588], t[bi, n])              # (c, ky, kx) order, exact
    assert torch.all(patch[n_cls:n_cls + P, 588:] == 0)
    assert torch.equal(xr[n_cls:n_cls + P], rowadd[n])
    # sensitivity: rowidx without the +1 cls offset
    assert not torch.equal(got_idx, (bi * (N + 1) + n).int())


# ------------------------------------------------------------------------------------------------------ kv_add_rows
def _kv_case(dev, g, B, res, cells, ncols, ldkv, Pm):
    N = res * res
    kv = torch.randn(B * N, ldkv, generator=g)
    dkv = torch.full((Pm, ncols), float("nan"))  # rows >= count must never be read
    table = {}
    for p, c in enumerate(cells):  # the values depend on the cell only: persons on one cell have equal rows
        if c not in table:
            table[c] = torch.randn(ncols, generator=g)
        dkv[p] = table[c]
    det_b, det_y, det_x = _det(cells, Pm, dev)
    return kv, dkv, table, (det_b, det_y, det_x)


def _kv_ref(kv, table, res, ncols, shift=0):
    ref = kv.clone()
    for (b, y, x), v in table.items():
        r = b * res * res + y * res + (x + shift) % res
        ref[r, :ncols] = kv[r, :ncols] + v  # one fp32 addition, once per distinct cell
    return ref


@pytest.mark.parametrize("dups", [False, True])
def test_kv_add_rows(cuda_device, dups):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(17 + dups)
    B, res, ncols, ldkv = 3, 20, 96, 104
    cells = _persons(B, res, 20, g)
    if dups:  # forced persons sharing cells: adjacent and far apart within an image
        cells = sorted(cells + [cells[3], cells[3], cells[10]])
        first = [c for c in cells if c[0] == cells[-1][0]][0]
        cells = cells + [first]  # the last person of the last image repeats that image's first cell
    P = len(cells)
    Pm = P + 5
    kv, dkv, table, det = _kv_case(dev, g, B, res, cells, ncols, ldkv, Pm)
    kv_d = kv.to(dev)
    ops.kv_add_rows(kv_d, dkv.to(dev), *det, _count(dev, P), Pm, res)
    got = kv_d.cpu()
    assert torch.equal(got, _kv_ref(kv, table, res, ncols))                 # exact; pitch columns and other rows kept
    # sensitivity: the neighbouring cell
    assert not torch.equal(got, _kv_ref(kv, table, res, ncols, shift=1))


def test_kv_add_rows_distant_duplicate(cuda_device):
    """Thousands of persons in one image, the first and the last on the same cell: their CTAs cannot run together, so
    an unguarded read-modify-write would add the values twice."""
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(23)
    B, res, ncols = 1, 92, 32
    order = torch.randperm(res * res, generator=g)[:6000]
    cells = [(0, int(c) // res, int(c) % res) for c in order]  # one image, caller's order within it
    cells.append(cells[0])
    P = len(cells)
    kv, dkv, table, det = _kv_case(dev, g, B, res, cells, ncols, ncols, P)
    kv_d = kv.to(dev)
    ops.kv_add_rows(kv_d, dkv.to(dev), *det, _count(dev, P), P, res)
    got = kv_d.cpu()
    assert torch.equal(got, _kv_ref(kv, table, res, ncols))
    r0 = cells[0][1] * res + cells[0][2]
    twice = kv[r0] + table[cells[0]] + table[cells[0]]
    assert not torch.equal(got[r0], twice)


def test_kv_add_rows_zero_capacity(cuda_device):
    from multihmr_b200 import ops

    dev = cuda_device
    kv = torch.randn(16, 8, device=dev)
    before = kv.clone()
    ops.kv_add_rows(kv, torch.empty(0, 8, device=dev), *_det([], 0, dev), _count(dev, 0), 0, 4)
    assert torch.equal(kv, before)


# ---------------------------------------------------------------------------------------- cls_gather / anny_gather
@pytest.mark.parametrize("split", [False, True])
def test_cls_gather(cuda_device, split):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(31 + split)
    B, T, D = 3, 401, 768
    x = 5.0 + torch.randn(B * T, D + 8, generator=g) * 2
    if split:
        hi, lo = x.half(), (x - x.half().float()).half()
        got = ops.cls_gather(hi.to(dev), T, B, D, xlo=lo.to(dev)).cpu()
        src = hi.float() + lo.float()  # one fp32 addition, as the kernel does it
    else:
        got = ops.cls_gather(x.to(dev), T, B, D).cpu()
        src = x
    rows = torch.arange(B) * T
    assert torch.equal(got, src[rows, :D])
    # sensitivity: row b T + 1
    assert not torch.equal(got, src[rows + 1, :D])


@pytest.mark.parametrize("refined", [False, True])
@pytest.mark.parametrize("P", [0, 1, 13])
def test_anny_gather(cuda_device, P, refined):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(41 + P + refined)
    B, res, D, dim = 2, 16, 384, 512
    N, Pm = res * res, P + 2
    cells = _persons(B, res, P, g)
    det = _det(cells, Pm, dev)
    z32 = torch.randn(B * N, D, generator=g)
    pos = torch.randn(N, dim, generator=g)
    xr = norm = None
    if refined:
        xr = (1.0 + torch.randn(Pm, D, generator=g) * 3).to(dev)
        norm = ((0.5 + torch.rand(D, generator=g)).to(dev), (0.2 * torch.randn(D, generator=g)).to(dev))
    zc = torch.full((Pm, D), SENTINEL, device=dev)
    xa = torch.full((Pm, dim), SENTINEL, device=dev)
    ops.anny_gather(z32.to(dev), pos.to(dev), *det, _count(dev, P), Pm, res, zc, xa, xr=xr, norm=norm or (None, None))
    assert torch.all(zc[P:] == SENTINEL) and torch.all(xa[P:] == SENTINEL)
    if P == 0:
        return
    bi, yi, xi = (torch.tensor(v) for v in zip(*cells))
    n = yi * res + xi
    got_xa = xa[:P].cpu()
    assert torch.equal(got_xa, pos[n])                                      # dec_pos_emb of the cell, exact
    if refined:
        xd = xr[:P].double().cpu()
        gd, bd = (t.double().cpu() for t in norm)
        ref, tol = F.layer_norm(xd, (D,), gd, bd, 1e-6), _ln_block_tol(xd, gd, bd, D)
        err = (zc[:P].double().cpu() - ref).abs()
        _report(f"anny_gather P={P} refined zc", err, tol)
        assert torch.all(err <= tol)
    else:
        assert torch.equal(zc[:P].cpu(), z32[bi * N + n])
    # sensitivity: the cell transposed (x * res + y)
    assert not torch.equal(got_xa, pos[xi * res + yi])


# ------------------------------------------------------------------------------------------------------- anny_place
@pytest.mark.parametrize("with_v2d", [False, True])
@pytest.mark.parametrize("P", [0, 1, 4])
def test_anny_place(cuda_device, P, with_v2d):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(51 + P + with_v2d)
    V, J, center = 300, 7, 2
    bones = torch.randn(max(P, 1), J, 4, 4, generator=g)[:P].contiguous()
    transl = torch.randn(P, 3, generator=g) * 0.5 + torch.tensor([0.0, 0.0, 4.0])
    K = _cameras(max(P, 1), 896, g)[:P].contiguous()
    v_in = torch.randn(P, V, 3, generator=g) * 0.4
    v3d = v_in.clone().to(dev)
    j3d = torch.full((P, J, 3), SENTINEL, device=dev)
    j2d = torch.full((P, J, 2), SENTINEL, device=dev)
    v2d = torch.full((P, V, 2), SENTINEL, device=dev) if with_v2d else None
    tp = torch.full((P, 3), SENTINEL, device=dev)
    ops.anny_place(bones.to(dev), transl.to(dev), K.to(dev), center, v3d, j3d, j2d, tp, v2d=v2d)
    if P == 0:
        return

    def ref_of(c):
        shift = (transl.double() - bones[:, c, :3, 3].double())[:, None]
        return v_in.double() + shift, bones[:, :, :3, 3].double() + shift

    def proj(p3):
        uvw = p3 / p3[..., 2:]
        return torch.einsum("pij,pnj->pni", K.double(), uvw)[..., :2]

    rv, rj = ref_of(center)
    cpt = bones[:, center, :3, 3].double().abs()[:, None]
    # (x - c) + t: two fp32 additions
    def tol3(x):
        return 2 * U * (x.abs() + cpt + transl.double().abs()[:, None]) + 1e-30

    def tol2(p3, t3):
        # u = x / z: the errors of x and z relative to z plus the division; then K [u, v, 1]: three products, two sums
        z = p3[..., 2:].abs()
        u = p3[..., :2] / p3[..., 2:]
        du = (t3[..., :2] + u.abs() * t3[..., 2:]) / z + U * u.abs()
        Kd = K.double()
        lin = torch.einsum("pij,pnj->pni", Kd[:, :2, :2].abs(), du)
        mag = torch.einsum("pij,pnj->pni", Kd[:, :2].abs(), torch.cat([u.abs(), torch.ones_like(z)], -1))
        return lin + 4 * U * mag

    got_v, got_j = v3d.double().cpu(), j3d.double().cpu()
    ev, ej = (got_v - rv).abs(), (got_j - rj).abs()
    tv, tj = tol3(rv), tol3(rj)
    _report(f"anny_place P={P} v3d", ev, tv)
    _report(f"anny_place P={P} j3d", ej, tj)
    assert torch.all(ev <= tv) and torch.all(ej <= tj)
    assert torch.equal(tp.cpu(), j3d[:, 0].cpu())                          # transl_pelvis = j3d[:, 0], exact
    tj2 = tol2(rj, tj)
    ej2 = (j2d.double().cpu() - proj(rj)).abs()
    _report(f"anny_place P={P} j2d", ej2, tj2)
    assert torch.all(ej2 <= tj2)
    if with_v2d:
        tv2 = tol2(rv, tv)
        ev2 = (v2d.double().cpu() - proj(rv)).abs()
        _report(f"anny_place P={P} v2d", ev2, tv2)
        assert torch.all(ev2 <= tv2)
    # sensitivity: the neighbouring bone as the centre
    wv, _ = ref_of(center + 1)
    assert torch.any((got_v - wv).abs() > tv)
