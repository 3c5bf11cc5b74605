"""fp64 autograd reference of the training loss and its gradient (mhmr_train_loss): the SMPL-X head's outputs from the
decoder rows (oracle person post-processing: Gram-Schmidt, rotmat_to_rotvec, the dist chain, loc), the placed SMPL-X
layer (body_grad_util.placed_outputs over oracle.smplx_ref) and the statement of reference loss.py, with switches that
plant the mistakes the GPU tests must detect; case builders and the error bound."""
import math

import torch

import body_grad_util as bg
from oracle import multihmr_ref, roma_ref

LO, HI = float(torch.tensor(1e-4, dtype=torch.float32)), float(torch.tensor(1 - 1e-4, dtype=torch.float32))
WEIGHTS = dict(bce=10.0, offset=1.0, rotmat=0.1, shape=1.0, dist=1.0, transl=1.0, j3d=100.0, v3d=100.0, j2d=1.0,
               v2d=1.0)
TERMS = ("bce", "offset", "rotmat", "shape", "dist", "transl", "j3d", "v3d", "j2d", "v2d")


def scores_from_logits(logit, clamp_grad=True):
    """The SMPL-X head's clamped sigmoid; a value on a bound counts as clamped (no gradient), as the engine sees it
    from the stored value.  clamp_grad=False plants the mistake of letting the gradient through the clamp."""
    s = torch.sigmoid(logit)
    c = s.detach().clamp(LO, HI)
    if not clamp_grad:
        return c + (s - s.detach())
    s32 = c.float()  # the stored value decides, as in the engine
    return torch.where((s32 > LO) & (s32 < HI), s, c)


def head_outputs(dec, offset, cells, K_det, nb, img_size, gs_t=False):
    """model.py:257-298 + SMPL_Layer from the decoder rows dec [P, 318 + nb + 13]: rotmat, rotvec, shape, expression,
    dist_pp, dist, loc.  cells [P, 2] = (x, y) patch indices.  gs_t plants a transposed Gram-Schmidt derivative."""
    P = dec.shape[0]
    R = multihmr_ref.rot6d_to_rotmat(dec[:, :318].reshape(P * 53, 6)).reshape(P, 53, 3, 3)
    if gs_t:
        Rt = R.transpose(-1, -2)
        R = R.detach() + (Rt - Rt.detach())
    rotvec = roma_ref.rotmat_to_rotvec(R.reshape(-1, 3, 3)).reshape(P, 53, 3)
    cam0 = dec[:, 318 + nb]
    fn = img_size / (2 * math.tan(math.radians(30)))
    dist = torch.clamp(torch.exp(cam0 * (K_det[:, 0, 0] / fn)) - 1e-10, 0, 50)
    loc = (cells.to(dec.dtype) + 0.5 + offset) * 14
    return dict(rotmat=R, rotvec=rotvec, shape=dec[:, 318:318 + nb], expression=dec[:, 321 + nb:331 + nb],
                dist_postprocessed=cam0, dist=dist, loc=loc, offset=offset)


def forward(bm, logit, dec, offset, cells, K_det, nb, img_size, gs_t=False, clamp_grad=True):
    o = head_outputs(dec, offset, cells, K_det, nb, img_size, gs_t)
    body = bg.placed_outputs(bm, o["rotvec"], o["shape"], o["loc"], o["dist"], K_det, o["expression"])
    o.update(body)
    o["scores"] = scores_from_logits(logit, clamp_grad)
    return o


def _nan_to_num(t):
    """nan_to_num of a scalar term: a replaced term is a constant 0 (no gradient)."""
    return t if torch.isfinite(t) else torch.zeros((), dtype=t.dtype, device=t.device)


def loss_terms(yh, y, img_size, no_pelvis=False, mask_per_person=False, no_inv_p=False):
    """loss.py:47-115 restated, term by term after nan_to_num; yh and y as head outputs and targets dicts."""
    s, gt = yh["scores"], (y["scores"] >= 1).to(yh["scores"].dtype)
    pos = torch.log(s + 1e-7) * (1 - s) ** 2 * gt
    neg = torch.log(1 - s + 1e-7) * s ** 2 * (1 - gt)
    npos = gt.sum()
    bce = -neg.sum() if npos == 0 else -(pos.sum() + neg.sum()) / npos
    mean0 = (lambda t: t.sum(0)) if no_inv_p else (lambda t: t.mean(0))
    t = dict(bce=bce)
    t["offset"] = mean0((yh["offset"] - y["offset"]).abs().sum(-1))
    t["rotmat"] = mean0((yh["rotmat"] - y["rotmat"]).abs().sum([1, 2, 3]))
    k = min(yh["shape"].shape[1], y["shape"].shape[1])
    t["shape"] = mean0((yh["shape"][:, :k] - y["shape"][:, :k]).abs().sum(-1))
    t["dist"] = mean0((yh["dist_postprocessed"] - y["dist_postprocessed"]).abs())
    t["transl"] = mean0((yh["transl"] - y["transl"]).abs().sum(-1))
    P = yh["j3d"].shape[0]
    ph, pg = yh["transl_pelvis"].reshape(P, 1, 3), y["transl_pelvis"].reshape(P, 1, 3)
    if no_pelvis:
        ph, pg = ph * 0, pg * 0
    for n in ("j3d", "v3d"):
        t[n] = ((y[n] - pg) - (yh[n] - ph)).abs().sum(-1).mean(-1).mean(0)
    for n in ("j2d", "v2d"):
        g = y[n]
        m = ((g > 0) & (g < img_size)).all(-1)
        d = (yh[n] - g).abs().sum(-1)
        if mask_per_person:
            t[n] = ((d * m).sum(1) / m.sum(1)).mean(0)
        else:
            t[n] = d[m].mean(0)
    return {k: _nan_to_num(v) for k, v in t.items()}


def total(terms, w, use_2d):
    return sum(w[k] * terms[k] for k in TERMS if use_2d or k not in ("j2d", "v2d"))


def reference(bm, case, use_2d=True, w=WEIGHTS, **mistake):
    """fp64 terms, total and the gradients (d_logits, d_offset, d_dec) plus the same gradients under |upstream| at
    the head's outputs (the magnitude the error bound scales with)."""
    fwd_m = {k: mistake.pop(k) for k in ("gs_t", "clamp_grad") if k in mistake}
    dev = case["dec"].device
    leaves = [case[k].to(dev, torch.float64).clone().requires_grad_() for k in ("logit", "dec", "offset")]
    K_det = case["K_det"].to(dev, torch.float64)
    yh = forward(bm, leaves[0], leaves[1], leaves[2], case["cells"].to(dev), K_det, case["nb"], case["img_size"],
                 **fwd_m)
    y = {k: v.to(dev, torch.float64) for k, v in case["targets"].items()}
    # the loss's own inputs as leaves: their gradients are the upstream of the chain (not totals through the graph)
    keys = ("scores", "offset", "rotmat", "shape", "dist_postprocessed", "transl", "transl_pelvis", "j3d", "v3d",
            "j2d", "v2d")
    yl = {k: yh[k].detach().requires_grad_() for k in keys}
    terms = loss_terms(yl, y, case["img_size"], **mistake)
    L = total(terms, w, use_2d)
    ups = torch.autograd.grad(L, [yl[k] for k in keys], allow_unused=True)
    up = {k: g for k, g in zip(keys, ups) if g is not None}
    ref = bg.vjp({k: yh[k] for k in up}, up, leaves)
    ref_abs = bg.vjp({k: yh[k] for k in up}, {k: g.abs() for k, g in up.items()}, leaves)
    return {k: float(v.detach()) for k, v in terms.items()}, float(L.detach()), ref, ref_abs, bce_coef(case, w)


def bce_coef(case, w=WEIGHTS):
    """d total / d (focal-loss sum): -alpha_bce / num_pos, or -alpha_bce without positives."""
    npos = float((case["targets"]["scores"] >= 1).sum())
    return -w["bce"] / npos if npos > 0 else -w["bce"]


def n_seq(V):
    """The body backward's accumulation depth (body_grad_util.n_seq) plus the loss's own chain: the upstream
    coefficient, the sign counts of the pelvis and the Gram-Schmidt / dist chains (16 roundings)."""
    return bg.n_seq(V, 55) + 16


def tolerance(ref, ref_abs, n):
    return bg.tolerance(ref, ref_abs, n)


def logit_tolerance(ref, logit, coef_bce):
    """d_logits is one fp32 expression per cell: both parts of each focal derivative share a sign, so 64 roundings
    relative, plus the absolute error of log(s + 1e-7) and log(1 - s + 1e-7) (rounding of the argument, u|log| of
    logf) carried by their factors 2(1 - s) and 2s, and of the two quotients."""
    s = torch.sigmoid(logit)
    q = 1 - s
    u = bg.U
    dlog = 2 * q * u * (2 + s.log().abs()) + 2 * s * u * (2 + q.log().abs()) + 3 * u * (q * q / s + s * s / q)
    return 64 * u * ref.abs() + 4 * abs(coef_bce) * s * q * dlog


def make_case(m, P, B, seed, nb_gt=11, edge=None):
    """Fixed head outputs of an engine `m` (decoder rows, offsets, clamped scores) and targets at a sign-safe
    distance from the fp64 outputs: every L1 difference is at least 1e-2 (1 px in 2-D) away from 0, so rounding
    cannot flip a sign.  edge: None, 'no_pos', 'no_2d', 'nan_shape', 'dist_clamp'."""
    from multihmr_b200 import synth

    g = torch.Generator().manual_seed(seed)
    res, S, nb, dev = m.res, m.img_size, m.num_betas, m.device
    N = res * res
    logit = torch.randn(B, res, res, generator=g, dtype=torch.float64) * 3
    logit.view(-1)[: N // 8] = -20.0  # on the lower clamp
    logit.view(-1)[N // 8: N // 8 + 5] = 20.0  # on the upper clamp
    s32 = torch.sigmoid(logit).float().double()  # the engine scores the stored fp32 value
    logit = torch.where((s32 > 0) & (s32 < 1), torch.logit(s32), logit)
    dec = torch.randn(P, 318 + nb + 13, generator=g, dtype=torch.float64) * 0.5
    dec[:, :318] += torch.tensor([1.0, 0, 0, 0, 1.0, 0], dtype=torch.float64).repeat(53)
    fn = S / (2 * math.tan(math.radians(30)))
    K = synth.make_cameras(B, S, jitter=True, seed=seed).to(torch.float64)
    b = torch.sort(torch.randint(0, B, (P,), generator=g)).values
    cells = torch.randint(2, res - 2, (P, 2), generator=g)
    K_det = K[b]
    z = 3.0 + 4.0 * torch.rand(P, generator=g, dtype=torch.float64)
    dec[:, 318 + nb] = torch.log(z) * fn / K_det[:, 0, 0]  # dist_pp giving depths 3..7 m
    if edge == "dist_clamp" and P >= 2:
        dec[0, 318 + nb] = -40.0 * fn / K_det[0, 0, 0]  # exp(-40) - 1e-10 < 0: clamped at 0
        dec[1, 318 + nb] = 5.0 * fn / K_det[1, 0, 0]  # e^5 > 50: clamped at 50
    offset = torch.rand(P, 2, generator=g, dtype=torch.float64) - 0.5
    with torch.no_grad():
        yh = forward(m._bm, logit, dec, offset, cells, K_det, nb, S)
    far = lambda t, lo, hi: (lo + (hi - lo) * torch.rand(t.shape, generator=g, dtype=torch.float64)) * (
        torch.randint(0, 2, t.shape, generator=g) * 2 - 1)
    tp = yh["transl_pelvis"] + 0.1 * torch.randn(P, 3, generator=g, dtype=torch.float64)
    shift = (tp - yh["transl_pelvis"]).unsqueeze(1)
    y = dict(
        scores=(torch.rand(B, res, res, generator=g) < 0.02).to(torch.float64) * (1 + torch.rand(B, res, res, generator=g)),
        offset=yh["offset"] + far(yh["offset"], 0.01, 0.05),
        rotmat=yh["rotmat"] + far(yh["rotmat"], 0.01, 0.05),
        shape=torch.cat([yh["shape"], torch.zeros(P, max(nb_gt - nb, 0), dtype=torch.float64)], 1)[:, :nb_gt],
        dist_postprocessed=yh["dist_postprocessed"] + far(yh["dist_postprocessed"], 0.01, 0.05),
        transl=yh["transl"] + far(yh["transl"], 0.01, 0.05), transl_pelvis=tp,
        j3d=yh["j3d"] + shift + far(yh["j3d"], 0.01, 0.05), v3d=yh["v3d"] + shift + far(yh["v3d"], 0.01, 0.05),
        j2d=yh["j2d"] + far(yh["j2d"], 1.0, 3.0), v2d=yh["v2d"] + far(yh["v2d"], 1.0, 3.0))
    y["shape"][:, :min(nb, nb_gt)] += far(y["shape"][:, :min(nb, nb_gt)], 0.01, 0.05)
    for n in ("j2d", "v2d"):  # points leaving the image, more for some persons than others
        out = torch.rand(y[n].shape[:2], generator=g) < torch.linspace(0.05, 0.6, P, dtype=torch.float64)[:, None]
        y[n][..., 0] = torch.where(out, -y[n][..., 0].abs() - 1, y[n][..., 0])
    if edge == "no_pos":
        y["scores"].zero_()
    if edge == "no_2d":
        y["j2d"][..., 1] = S + 5.0
        y["v2d"][..., 1] = -5.0
    if edge == "nan_shape":
        y["shape"][P // 2, 0] = float("nan")
    return dict(logit=logit, dec=dec, offset=offset, cells=cells, b=b, K=K, K_det=K_det, nb=nb, img_size=S,
                targets=y)


GOLDEN_SEED = 21  # oracle/make_golden_train.py: weights, body model and batch
GOLDEN_TARGETS = ("scores", "offset", "rotmat", "shape", "dist_postprocessed", "transl", "transl_pelvis", "j3d", "v3d",
                  "j2d", "v2d")


def golden_case(gold, nb=10, img_size=224):
    """A case of `reference` / the engine tests from tests/golden/train_loss_224_S.npz: the reference model's head
    outputs and the reference's targets."""
    t = lambda k: torch.as_tensor(gold[k])
    idx = t("gt_idx")
    K = t("K").to(torch.float64)
    return dict(logit=t("logits").to(torch.float64), dec=t("dec").to(torch.float64),
                offset=t("offset").to(torch.float64), cells=torch.stack([idx[2], idx[1]], 1), b=idx[0], K=K,
                K_det=K[idx[0]], nb=nb, img_size=img_size,
                targets={k: t("gt_" + k).to(torch.float64) for k in GOLDEN_TARGETS})
