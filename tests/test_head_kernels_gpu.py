"""Person-decoder kernels (head.cu, refine.cu) through their stage-level entry points, against plain fp64 torch
references written from the reference semantics: the skinny Linear, HPH self- and cross-attention, detection (NMS +
ordered compaction), the SMPL-X and Anny per-person post-processing and the fp32 central-stream refinement chain.

Every floating-point comparison states its tolerance next to it, and every op has a sensitivity check: a reference
with one plausible mistake (a dropped K element, the wrong image's keys, a missing sign flip, ...) must fall outside
that tolerance, so the tolerance is known to catch such slips.  The person count is a device int32 tensor with
count < max_persons where possible, and rows >= count must come back untouched."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # unit roundoff of fp32
SENTINEL = 12345.0


def _count(dev, n):
    return torch.tensor([n], dtype=torch.int32, device=dev)


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


# ------------------------------------------------------------------------------------------------------ skinny_linear
SKINNY = [
    # (K, ldx, Nout, P, max_persons, options)
    (4, 4, 1, 1, 1, ()),
    (4, 4, 11, 7, 8, ("ln", "bias")),
    (99, 100, 2, 8, 8, ("bias",)),                      # K % 4 != 0, padded pitch (NaN padding must not leak)
    (99, 101, 11, 9, 16, ("relu", "bias")),             # odd pitch: scalar loads
    (483, 483, 978, 17, 24, ("gelu",)),                 # odd pitch, ragged chunk
    (483, 488, 978, 17, 24, ("resid",)),
    (1123, 1124, 11, 64, 64, ("gelu", "bias")),         # > one 1024-wide K tile
    (1123, 1127, 4224, 5, 64, ("bias", "resid")),       # count << max_persons, unaligned pitch
    (2048, 2048, 4224, 9, 16, ("ln", "gelu", "bias", "resid")),
    (2048, 2048, 8192, 8, 8, ("ln",)),                  # SMPL-X to_kv width of an 8-layer 16-head HPH
    (512, 512, 512, 17, 24, ("ln", "relu", "bias", "inplace")),
    (512, 516, 512, 33, 40, ("bias", "inplace")),       # the engine's x += W . att + b
    (1024, 1024, 978, 64, 64, ("ln", "gelu", "bias", "resid")),
]


def _skinny_ref(x, K, w, bias, ln, act, resid, drop_last=False):
    xin = x[:, :K].double()
    if ln is not None:
        g, b, eps = ln
        xin = F.layer_norm(xin, (K,), g.double(), b.double(), eps)
    wd = w[:, :K].double()
    if drop_last:
        xin = xin.clone()
        xin[:, -1] = 0.0
    y = xin @ wd.t()
    if bias is not None:
        y = y + bias.double()
    if act == 1:
        y = torch.relu(y)
    elif act == 2:
        y = F.gelu(y)
    if resid is not None:
        y = y + resid.double()
    return y


@pytest.mark.parametrize("cols", [16, 32])
@pytest.mark.parametrize("K,ldx,Nout,P,Pm,opts", SKINNY)
def test_skinny_linear(cuda_device, K, ldx, Nout, P, Pm, opts, cols):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(K * 131 + Nout * 7 + P)
    Kp = (K + 3) & ~3
    x = torch.randn(Pm, ldx, generator=g) + 0.3
    x[:, K:] = float("nan")                      # pitch padding: must never contribute
    x[P:] = float("nan")                         # rows >= count must not be read into anything
    ldw = Kp + 4
    w = torch.randn(Nout, ldw, generator=g) / math.sqrt(K)
    w[:, K:] = 1e30                              # W padding is multiplied by zeros (finite by contract)
    bias = torch.randn(Nout, generator=g) * 0.5 if "bias" in opts else None
    ln = None
    if "ln" in opts:
        ln = ((torch.rand(K, generator=g) + 0.5).to(dev), (torch.randn(K, generator=g) * 0.2).to(dev), 1e-5)
    act = 1 if "relu" in opts else 2 if "gelu" in opts else 0
    ldo = Nout + 3
    resid = None
    if "resid" in opts or "inplace" in opts:
        resid = torch.randn(Pm, ldo, generator=g).to(dev)
    x, w = x.to(dev), w.to(dev)
    bias = bias.to(dev) if bias is not None else None
    if "inplace" in opts:
        out = resid                               # out == resid, as the engine's residual updates call it
        before = resid.clone()
    else:
        out = torch.full((Pm, ldo), SENTINEL, device=dev)
        before = out.clone()
    resid_ref = None if resid is None else resid[:P, :Nout].clone()
    ops.skinny_linear(x, _count(dev, P), Pm, K, w, out, bias=bias, ln=ln, act=act, resid=resid, cols=cols)
    torch.cuda.synchronize()
    got = out[:P, :Nout].double().cpu()
    ref = _skinny_ref(x[:P], K, w, bias, ln, act, resid_ref).cpu()
    # Tolerance: an fp32 dot product of K terms is within ~sqrt(K) u sum|w x| of the exact one for random signs
    # (Higham's probabilistic bound, c = 8 covers the 4-term partial sums and the butterfly); LayerNorm adds a few u
    # of |x_hat g| + |beta| per input (inside |xin|), ReLU/GELU are 1.13-Lipschitz, and the bias and residual
    # additions round once each.
    xin = x[:P, :K].double()
    if ln is not None:
        xin = F.layer_norm(xin, (K,), None, None, ln[2]).abs() * ln[0].double() + ln[1].double().abs()
    mag = xin.abs() @ w[:, :K].double().abs().t()
    if bias is not None:
        mag = mag + bias.double().abs()
    tol = 8 * math.sqrt(K) * U * mag * 1.13 + 2 * U * ref.abs().to(mag.device)
    tol = tol.cpu() + 1e-30
    err = (got - ref).abs()
    print(f"  skinny K={K} N={Nout} P={P} cols={cols} {opts}: worst err/tol {(err / tol).max().item():.3f}"
          f" (max err {err.max().item():.2e})")
    assert torch.isfinite(got).all()
    assert (err <= tol).all(), (err / tol).max().item()
    # untouched: rows >= count and the pitch columns beyond Nout
    assert torch.equal(out[P:], before[P:])
    assert torch.equal(out[:, Nout:], before[:, Nout:])
    # sensitivity: the same reference with the last K element dropped must fall outside the tolerance
    bad = _skinny_ref(x[:P], K, w, bias, ln, act, resid_ref, drop_last=True).cpu()
    assert ((got - bad).abs() > tol).any()


def test_skinny_linear_cols_zero_matches_an_explicit_variant(cuda_device):
    """cols = 0 (the engine's choice) computes the same thing bit for bit as the variant it picks."""
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(3)
    x = torch.randn(9, 512, generator=g).to(dev)
    w = (torch.randn(40, 512, generator=g) / 20).to(dev)
    outs = []
    for cols in (0, 16, 32):
        o = torch.zeros(9, 40, device=dev)
        ops.skinny_linear(x, _count(dev, 9), 9, 512, w, o, cols=cols)
        outs.append(o)
    assert torch.equal(outs[0], outs[1]) or torch.equal(outs[0], outs[2])


def test_skinny_linear_rejects_bad_arguments(cuda_device):
    from multihmr_b200 import ops

    dev = cuda_device
    x = torch.zeros(8, 64, device=dev)
    w = torch.zeros(8, 64, device=dev)
    out = torch.zeros(8, 8, device=dev)
    with pytest.raises(AssertionError):
        ops.skinny_linear(x, _count(dev, 1), 8, 64, w, out, cols=8)
    with pytest.raises(AssertionError):
        ops.skinny_linear(torch.zeros(8, 30, device=dev), _count(dev, 1), 8, 64, w, out)   # K beyond the rows
    with pytest.raises(AssertionError):
        ops.skinny_linear(x, _count(dev, 1), 8, 64, w, out, act=3)


# ------------------------------------------------------------------------------------------------- HPH attention
def _layout(counts):
    det_b = torch.cat([torch.full((c,), b, dtype=torch.int32) for b, c in enumerate(counts)])
    img_off = torch.tensor([0] + list(torch.tensor(counts).cumsum(0).tolist()), dtype=torch.int32)
    return det_b, img_off


def _attend(q, k, v, heads):
    """softmax(q k^T 32^-0.5) v per head in fp64; q [n, h*32], k, v [m, h*32]."""
    n, m = q.shape[0], k.shape[0]
    qh, kh, vh = (t.double().reshape(t.shape[0], heads, 32).transpose(0, 1) for t in (q, k, v))
    a = torch.softmax(qh @ kh.transpose(-1, -2) * 32 ** -0.5, dim=-1)
    return (a @ vh).transpose(0, 1).reshape(n, heads * 32)


def _attn_tol(q, k, v, heads):
    """Per (person, head): the logit error of an fp32 32-term dot product is within ~5 u |q_h| |k_h| (tree sum,
    log2(32) levels), a softmax weight moves by at most twice the largest logit error, and the running sums over the
    m keys add ~sqrt(m) u; all relative to the largest |v| of that head."""
    n, m = q.shape[0], k.shape[0]
    qn = q.double().reshape(n, heads, 32).norm(dim=-1)
    kn = k.double().reshape(m, heads, 32).norm(dim=-1).max(dim=0).values
    vmax = v.double().reshape(m, heads, 32).abs().amax(dim=(0, 2))
    delta = qn * kn * 32 ** -0.5
    tol = U * vmax * (16 * delta + 8 * math.sqrt(m) + 8)
    return tol[:, :, None].expand(n, heads, 32).reshape(n, heads * 32)


@pytest.mark.parametrize("heads", [8, 16])
@pytest.mark.parametrize("counts,peaky", [([0, 1, 2, 40, 0], False), ([2, 0, 1, 40], True), ([3], False),
                                          ([1, 1, 1, 1, 1, 1, 1, 1, 1, 1], True)])
def test_hph_self_attn(cuda_device, heads, counts, peaky):
    from multihmr_b200 import ops

    dev = cuda_device
    inner = heads * 32
    P, Pm = sum(counts), sum(counts) + 5
    g = _gen(P * 10 + heads)
    ld = 3 * inner + 4
    qkv = torch.randn(Pm, ld, generator=g) * (20.0 if peaky else 1.0) ** 0.5
    det_b, img_off = _layout(counts)
    det_b = torch.cat([det_b, torch.zeros(Pm - P, dtype=torch.int32)])
    out = torch.full((Pm, inner), SENTINEL, device=dev)
    ops.hph_self_attn(qkv.to(dev), det_b.to(dev), img_off.to(dev), _count(dev, P), Pm, heads, out)
    got = out.cpu().double()
    assert (got[P:] == SENTINEL).all()
    q, k, v = qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:3 * inner]
    ref = torch.zeros(P, inner, dtype=torch.float64)
    tol = torch.zeros(P, inner, dtype=torch.float64)
    bad = torch.zeros(P, inner, dtype=torch.float64)
    nonempty = [b for b, c in enumerate(counts) if c > 0]
    for i, b in enumerate(nonempty):
        s, e = int(img_off[b]), int(img_off[b + 1])
        ref[s:e] = _attend(q[s:e], k[s:e], v[s:e], heads)
        tol[s:e] = _attn_tol(q[s:e], k[s:e], v[s:e], heads)
        # mistake: the persons of image b paired with the next non-empty image's keys and values
        b2 = nonempty[(i + 1) % len(nonempty)]
        s2, e2 = int(img_off[b2]), int(img_off[b2 + 1])
        bad[s:e] = _attend(q[s:e], k[s2:e2], v[s2:e2], heads)
    err = (got[:P] - ref).abs()
    print(f"  self-attn heads={heads} counts={counts}: worst err/tol {(err / tol).max().item():.3f}")
    assert (err <= tol).all(), (err / tol).max().item()
    if len(nonempty) > 1:
        assert ((got[:P] - bad).abs() > tol).any()


@pytest.mark.parametrize("N", [16, 255, 256, 257, 400, 2304, 8464])
@pytest.mark.parametrize("heads", [8, 16])
def test_hph_cross_attn(cuda_device, N, heads):
    from multihmr_b200 import ops

    dev = cuda_device
    inner = heads * 32
    counts = [0, 1, 2, 40] if N <= 2304 else [2, 0, 7]
    B, P = len(counts), sum(counts)
    Pm = P + 3
    layer, depth = 1, 2                              # keys / values of a later layer: k_col = l * 2 * inner
    ldkv = depth * 2 * inner
    k_col, v_col = layer * 2 * inner, layer * 2 * inner + inner
    g = torch.Generator(device=dev).manual_seed(N * 3 + heads)
    KV = torch.randn(B * N, ldkv, device=dev, generator=g)
    KV[:, :k_col] = float("nan")                     # layer 0's columns must not be read
    q = torch.randn(Pm, inner + 4, device=dev, generator=g)
    q[: P // 2] *= 20.0                               # logits x20 (a peaky softmax) for half of the persons
    KV[:, k_col:k_col + 32] = KV[0:1, k_col:k_col + 32]   # head 0: all keys equal -> uniform weights
    det_b, _ = _layout(counts)
    det_b = torch.cat([det_b, torch.zeros(Pm - P, dtype=torch.int32)]).to(dev)
    out = torch.full((Pm, inner), SENTINEL, device=dev)
    ops.hph_cross_attn(q, KV, k_col, v_col, det_b, _count(dev, P), Pm, heads, N, out)
    torch.cuda.synchronize()
    got = out.double()
    assert (got[P:] == SENTINEL).all()
    ref = torch.zeros(P, inner, dtype=torch.float64, device=dev)
    tol = torch.zeros_like(ref)
    bad = torch.zeros_like(ref)
    for p in range(P):
        b = int(det_b[p])
        rows = KV[b * N:(b + 1) * N]
        k, v = rows[:, k_col:k_col + inner], rows[:, v_col:v_col + inner]
        ref[p] = _attend(q[p:p + 1, :inner], k, v, heads)[0]
        tol[p] = _attn_tol(q[p:p + 1, :inner], k, v, heads)[0]
        b2 = (b + 1) % B                             # mistake: image b + 1's keys and values
        rows2 = KV[b2 * N:(b2 + 1) * N]
        bad[p] = _attend(q[p:p + 1, :inner], rows2[:, k_col:k_col + inner], rows2[:, v_col:v_col + inner], heads)[0]
    err = (got[:P] - ref).abs()
    print(f"  cross-attn N={N} heads={heads}: worst err/tol {(err / tol).max().item():.3f}")
    assert (err <= tol).all(), (err / tol).max().item()
    assert ((got[:P] - bad).abs() > tol).any()


# --------------------------------------------------------------------------------------------------------- detect
def _detect_ref(scores, k, thresh, Pm, strict=False):
    from oracle import multihmr_ref

    heat = scores[:, None]
    if k > 1:
        heat = multihmr_ref.nms(heat, k)
    heat = heat[:, 0]
    b, y, x = torch.where(heat > thresh if strict else heat >= thresh)
    P = b.shape[0]
    Pc = min(P, Pm)
    img_off = torch.tensor([int((b[:Pc] < i).sum()) for i in range(scores.shape[0] + 1)], dtype=torch.int32)
    return dict(scores_out=heat, det_b=b[:Pc].int(), det_y=y[:Pc].int(), det_x=x[:Pc].int(),
                det_score=heat[b[:Pc], y[:Pc], x[:Pc]], count=P, count_clamped=Pc, img_off=img_off)


def _score_map(kind, B, res, thresh, g):
    if kind == "random":
        s = torch.rand(B, res, res, generator=g)
    else:  # plateaus of equal values (the SMPL-X clamp at 1 - 1e-4 makes them common), straddling window borders
        lv = torch.tensor([0.05, thresh, 0.5, 1 - 1e-4], dtype=torch.float32)
        s = lv[torch.randint(0, 4, (B, (res + 1) // 2, (res + 1) // 2), generator=g)]
        s = s.repeat_interleave(2, 1).repeat_interleave(2, 2)[:, :res, :res].contiguous()
        s[:, 1::3, :] = torch.roll(s[:, 1::3, :], 1, dims=2)      # ties across 2x2 block borders
    s = s.float()
    s.view(-1)[:: 7] = thresh                                     # values exactly at the threshold
    if B >= 5:
        s[0] = 0.01                                               # empty first, middle and last images
        s[B // 2] = 0.01
        s[-1] = 0.01
    elif B == 3:
        s[1] = 0.01
    return s


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 7])
@pytest.mark.parametrize("B,res", [(1, 16), (41, 5), (3, 64), (5, 32)])
@pytest.mark.parametrize("kind", ["random", "plateau"])
def test_detect_exact(cuda_device, k, B, res, kind):
    """Pure comparison and compaction: the map, indices, score, counts and img_off must match exactly."""
    from multihmr_b200 import ops

    thresh = float(torch.tensor(0.3, dtype=torch.float32))
    g = _gen(k * 100 + B * res + (kind == "plateau"))
    s = _score_map(kind, B, res, thresh, g)
    for Pm in (1024, 7):                              # capacity, then overflow: the first 7 in order, true count kept
        o = ops.detect(s.to(cuda_device), k, thresh, Pm)
        r = _detect_ref(s, k, thresh, Pm)
        Pc = r["count_clamped"]
        assert torch.equal(o["scores_out"].cpu(), r["scores_out"])
        assert int(o["count"]) == r["count"] and int(o["count_clamped"]) == Pc
        for key in ("det_b", "det_y", "det_x", "det_score"):
            assert torch.equal(o[key][:Pc].cpu(), r[key]), key
        assert torch.equal(o["img_off"].cpu(), r["img_off"])
        if Pm == 7 and kind == "plateau":
            assert r["count"] > Pm


@pytest.mark.parametrize("k", [2, 3])
def test_detect_sensitivity(cuda_device, k):
    """The exact comparison rejects a strict threshold (a plateau of cells at the threshold) and, for the even
    kernel, a window anchored at (y, x) instead of ending there."""
    from multihmr_b200 import ops

    thresh = float(torch.tensor(0.3, dtype=torch.float32))
    s = torch.zeros(2, 8, 8)
    s[0, 2:4, 3:5] = thresh                          # a 2x2 plateau exactly at the threshold: all four are kept
    s[1, 5, 5], s[1, 5, 6] = 0.9, 0.8
    o = ops.detect(s.to(cuda_device), k, thresh, 16)
    r = _detect_ref(s, k, thresh, 16)
    assert int(o["count"]) == r["count"] and torch.equal(o["scores_out"].cpu(), r["scores_out"])
    assert _detect_ref(s, k, thresh, 16, strict=True)["count"] != int(o["count"])
    if k == 2:
        heat = s[:, None]
        hmax = F.max_pool2d(F.pad(heat, (0, 1, 0, 1), value=-math.inf), 2, 1)
        wrong = (heat * (hmax == heat).float())[:, 0]
        assert not torch.equal(wrong, o["scores_out"].cpu())


def test_detect_all_empty(cuda_device):
    from multihmr_b200 import ops

    s = torch.zeros(4, 8, 8)
    o = ops.detect(s.to(cuda_device), 3, 0.3, 16)
    assert int(o["count"]) == 0 and int(o["count_clamped"]) == 0
    assert o["img_off"].cpu().tolist() == [0] * 5


# ---------------------------------------------------------------------------------------------- person post-processing
def _axis_angle(axis, angle):
    a = torch.tensor(axis, dtype=torch.float64)
    return a / a.norm() * angle


def _rotation_cases():
    """Rotation vectors whose matrices reach every quaternion branch and the series / sign edges."""
    rv = [_axis_angle([0.3, -0.5, 0.8], a) for a in (0.0, 1e-4, 1e-3 - 1e-5, 1e-3 + 1e-5, 0.3, 1.5)]   # trace largest
    for i in range(3):                                   # diagonal element i largest: near-pi turns about ~e_i
        ax = [0.1, -0.15, 0.2]
        ax[i] = 1.0
        rv += [_axis_angle(ax, a) for a in (2.5, math.pi - 1e-3, math.pi - 1e-6)]
        ax[(i + 1) % 3] = -0.4
        rv.append(_axis_angle(ax, 2.9))
    rv += [_axis_angle([-0.6, 0.2, -0.7], a) for a in (2.0, 3.0)]                                         # w < 0 on entry
    return torch.stack(rv)


def _six_d(R, g, parallel):
    """Two columns of R, scaled, with a multiple of the first added to the second (Gram-Schmidt removes it).  With
    `parallel` the second column is 1e-3 R[:,1] + R[:,0]: condition number ~1e3."""
    n = R.shape[0]
    s1 = torch.rand(n, 1, generator=g, dtype=torch.float64) + 0.5
    s2 = torch.rand(n, 1, generator=g, dtype=torch.float64) + 0.5
    t = torch.randn(n, 1, generator=g, dtype=torch.float64)
    a = R[:, :, 0] * s1
    b = R[:, :, 1] * s2 + t * R[:, :, 0]
    if parallel:
        b = R[:, :, 1] * 1e-3 + R[:, :, 0]
    return a, b


def _quat_to_rotvec_without_flip(q):
    half = torch.atan2(torch.norm(q[:, :3], dim=1), q[:, 3])
    angle = 2 * half
    return (angle / torch.sin(half))[:, None] * q[:, :3]


def _rot_checks(got_R, got_rv, a, b, u=None):
    """fp64 Gram-Schmidt and rotvec of the fp32 inputs (roma semantics).  Tolerances: both columns are normalised in
    fp32 (a few u), the second after removing its component along the first, which amplifies the rounding by the
    condition number kappa = |a||b| / |a x b|: |dR| <= 16 u kappa.  The quaternion branch is the well-conditioned one
    (largest of trace / diagonal), and atan2 and the scale factor are smooth up to the angle, so |d rotvec| <= 64 u
    kappa (1 + angle).  Within max(1e-5, that tolerance) of pi an angle error can cross pi, where the rotation vector
    and its antipode describe the same rotation, so there rotvec_to_rotmat(rotvec) is compared with R instead."""
    from oracle import roma_ref

    M = torch.stack([a, b], dim=-1)
    R = roma_ref.special_gramschmidt(M)
    if u is not None:
        R = u[:, None, None] * R + (1 - u[:, None, None]) * torch.eye(3, dtype=torch.float64)
    rv = roma_ref.rotmat_to_rotvec(R)
    kappa = a.norm(dim=1) * b.norm(dim=1) / torch.cross(a, b, dim=1).norm(dim=1)
    if u is not None:                                  # the blend of a rotation with I is no longer orthogonal
        kappa = kappa / torch.clamp(u + (1 - u) * 0.1, max=1.0)
    tol_R = 16 * U * kappa
    eR = (got_R.double() - R).abs().amax(dim=(1, 2))
    assert (eR <= tol_R).all(), (eR / tol_R).max().item()
    angle = rv.norm(dim=1)
    tol_rv = 64 * U * kappa * (1 + angle)
    near_pi = (math.pi - angle) < torch.clamp(tol_rv, min=1e-5)
    erv = (got_rv.double() - rv).abs().amax(dim=1)
    erv_pi = (roma_ref.rotvec_to_rotmat(got_rv.double()) - R).abs().amax(dim=(1, 2))
    erv = torch.where(near_pi, erv_pi, erv)
    assert (erv <= tol_rv).all(), (erv / tol_rv).max().item()
    # sensitivity: without the shortest-arc sign flip (w >= 0) the rotation vectors of w < 0 inputs are wrong
    q = roma_ref.rotmat_to_unitquat(R)
    bad = _quat_to_rotvec_without_flip(q)
    assert ((got_rv.double() - bad).abs().amax(dim=1) > tol_rv)[~near_pi].any()
    return (eR / tol_R).max().item(), (erv / tol_rv).max().item()


@pytest.mark.parametrize("num_betas", [10, 11])
def test_person_post_smplx(cuda_device, num_betas):
    from oracle import multihmr_ref, roma_ref

    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(num_betas)
    cases = _rotation_cases()                                     # [n, 3]
    n = cases.shape[0]
    P, Pm, B, S = 6, 8, 3, 448
    # joint j of person p uses rotation case (p * 53 + j) % n; every third person has nearly parallel columns
    idx = torch.arange(P * 53) % n
    R_true = roma_ref.rotvec_to_rotmat(cases[idx])
    a, b = _six_d(R_true, g, parallel=False)
    par = (torch.arange(P * 53) // 53) % 3 == 2
    a_p, b_p = _six_d(R_true, g, parallel=True)
    a, b = torch.where(par[:, None], a_p, a), torch.where(par[:, None], b_p, b)
    a, b = a.float(), b.float()
    ld = 318 + num_betas + 13 + 3
    dec = torch.randn(Pm, ld, generator=g)
    dec[:P, :318] = torch.cat([a, b], 1).reshape(P, 53 * 6)
    cam0 = torch.tensor([-30.0, 10.0, 0.7, -0.2, 1.3, 0.05, 0.0, 0.0])   # low clamp, high clamp, in between
    dec[:, 318 + num_betas] = cam0
    offset = torch.rand(Pm, 2, generator=g) - 0.5
    K = torch.zeros(B, 3, 3)
    K[:, 0, 0] = K[:, 1, 1] = torch.tensor([400.0, 650.0, 900.0])
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 224.0, 230.0, 1.0
    det_b = torch.tensor([0, 0, 1, 2, 2, 2, 0, 0], dtype=torch.int32)
    det_y = torch.randint(0, S // 14, (Pm,), generator=g, dtype=torch.int32)
    det_x = torch.randint(0, S // 14, (Pm,), generator=g, dtype=torch.int32)
    focal_norm = float(torch.tensor(S / (2 * math.tan(math.radians(30))), dtype=torch.float32))
    o = ops.person_post(dec.to(dev), num_betas, offset.to(dev), K.to(dev), det_b.to(dev), det_y.to(dev), det_x.to(dev),
                        _count(dev, P), Pm, focal_norm)
    o = {k: v.cpu() for k, v in o.items()}
    for k in o:
        assert (o[k][P:] == 0).all(), k                           # rows >= count untouched
    rR, rrv = _rot_checks(o["rotmat"][:P].reshape(-1, 3, 3), o["rotvec"][:P].reshape(-1, 3), a.double(), b.double())
    # copies and the scalar chain, fp64 (model.py:189-203, :272-275, blocks/smpl_layer.py:123)
    assert torch.equal(o["shape"][:P], dec[:P, 318:318 + num_betas])
    assert torch.equal(o["expression"][:P], dec[:P, 318 + num_betas + 3:318 + num_betas + 13])
    assert torch.equal(o["dist_pp"][:P], cam0[:P])
    Kd = K.double()[det_b[:P].long()]
    arg = cam0[:P].double() * Kd[:, 0, 0] / multihmr_ref.focal_from_fov(60, S)
    dist = torch.clamp(torch.exp(arg) - 1e-10, 0, 50)
    # exp of an fp32 argument: relative error (2 + |arg|) u plus the two products of the argument
    tol_d = 8 * U * (2 + arg.abs()) * dist + 1e-30
    ed = (o["dist"][:P].double() - dist).abs()
    assert (ed <= tol_d).all(), (ed / tol_d).max().item()
    assert o["dist"][0] == 0.0 and o["dist"][1] == 50.0
    loc = (torch.stack([det_x[:P], det_y[:P]], 1).double() + 0.5 + offset[:P].double()) * 14
    assert ((o["loc"][:P].double() - loc).abs() <= 4 * U * loc.abs()).all()
    transl = torch.einsum("pij,pj->pi", torch.inverse(Kd), torch.cat([loc, torch.ones(P, 1, dtype=torch.float64)], 1))
    transl = transl * dist[:, None]
    # K^-1 in fp32 by cofactors (|K^-1| |K| ~ focal / 1 terms): 32 u of |K^-1| |[loc, 1]| dist per component
    tol_t = 32 * U * (torch.inverse(Kd).abs() @ torch.cat([loc, torch.ones(P, 1, dtype=torch.float64)], 1)[..., None])[..., 0]
    tol_t = tol_t * dist[:, None] + 1e-30
    et = (o["transl"][:P].double() - transl).abs()
    assert (et <= tol_t).all(), (et / tol_t).max().item()
    assert torch.equal(o["K_det"][:P], K[det_b[:P].long()])
    print(f"  person_post nb={num_betas}: rotmat err/tol {rR:.3f}, rotvec err/tol {rrv:.3f},"
          f" dist {(ed / tol_d).max().item():.3f}, transl {(et / tol_t).max().item():.3f}")


@pytest.mark.parametrize("with_K", [True, False])
def test_anny_person_post(cuda_device, with_K):
    from oracle import roma_ref

    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(7 + with_K)
    J, nb, P, Pm, B, S, D = 163, 11, 5, 8, 3, 448, 384
    cases = _rotation_cases()
    idx = torch.arange(P * J) % cases.shape[0]
    R_true = roma_ref.rotvec_to_rotmat(cases[idx])
    a, b = _six_d(R_true, g, parallel=False)
    par = (torch.arange(P * J) % 5) == 4
    a_p, b_p = _six_d(R_true, g, parallel=True)
    a, b = torch.where(par[:, None], a_p, a).float(), torch.where(par[:, None], b_p, b).float()
    ld6 = (6 * J + 3) & ~3
    rot6d = torch.randn(Pm, ld6, generator=g)
    # rot6d.reshape(3, 2): columns (x0, x2, x4) and (x1, x3, x5)
    rot6d[:P, :6 * J] = torch.stack([a, b], -1).reshape(P, J * 6)
    useful = torch.tensor([0.0, 0.3, 1.0])[torch.arange(J) % 3]
    hid = torch.randn(B, D, generator=g)
    w2 = torch.randn(D, generator=g) / math.sqrt(D)
    b2 = torch.tensor([0.1])
    fov_max = torch.tensor([2.2])
    K = torch.zeros(B, 3, 3)
    K[:, 0, 0] = K[:, 1, 1] = torch.tensor([400.0, 650.0, 900.0])
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 224.0, 230.0, 1.0
    shape_in = torch.randn(Pm, nb, generator=g) * 3
    offset = torch.rand(Pm, 2, generator=g) - 0.5
    dist_pp = torch.tensor([-12.0, -15.0, -2.0, 0.3, 1.1, 0.0, 0.0, 0.0])   # the 1e-5 clamp is active for <= -11.5
    det_b = torch.tensor([0, 1, 1, 2, 2, 0, 0, 0], dtype=torch.int32)
    det_y = torch.randint(0, S // 14, (Pm,), generator=g, dtype=torch.int32)
    det_x = torch.randint(0, S // 14, (Pm,), generator=g, dtype=torch.int32)
    shape_dev = shape_in.to(dev)
    o = ops.anny_person_post(hid.to(dev), w2.to(dev), b2.to(dev), fov_max.to(dev), K.to(dev) if with_K else None, S,
                             rot6d.to(dev), J, useful.to(dev), shape_dev, offset.to(dev), dist_pp.to(dev),
                             det_b.to(dev), det_y.to(dev), det_x.to(dev), _count(dev, P), Pm)
    o = {k: v.cpu() for k, v in o.items()}
    for k in ("rotmat", "rotmat_homo", "rotvec", "dist", "loc", "transl", "K_det"):
        assert (o[k][P:] == 0).all(), k
    assert torch.equal(o["shape"][P:], shape_in[P:])
    # camera (encoder.py:50-56): a D-term fp32 dot product (sqrt(D) u), then sigmoid, tan: relative 1e-6 is ~16 u
    fov = fov_max.double() * torch.sigmoid(hid.double() @ w2.double() + b2.double())
    f = (S / 2) / torch.tan(fov / 2)
    K_reg = torch.zeros(B, 3, 3, dtype=torch.float64)
    K_reg[:, 0, 0] = K_reg[:, 1, 1] = f
    K_reg[:, 0, 2] = K_reg[:, 1, 2] = S / 2
    K_reg[:, 2, 2] = 1
    dot_mag = hid.double().abs() @ w2.double().abs()
    tol_fov = 8 * math.sqrt(D) * U * dot_mag * fov_max.double() * 0.25 + 8 * U * fov
    assert ((o["fov"].double() - fov).abs() <= tol_fov).all()
    tol_f = f * (tol_fov / torch.sin(fov) + 8 * U)               # d/dfov of (S/2) / tan(fov/2) = f / sin(fov)
    assert ((o["K_regressed"].double() - K_reg).abs().amax(dim=(1, 2)) <= tol_f).all()
    K_use = K.double() if with_K else K_reg
    if with_K:
        assert torch.equal(o["K_use"], K)
    # rotations with the useful_rotmat blend
    u = useful.double()[torch.arange(P * J) % J]
    rR, rrv = _rot_checks(o["rotmat"][:P].reshape(-1, 3, 3), o["rotvec"][:P].reshape(-1, 3), a.double(), b.double(), u)
    H = o["rotmat_homo"][:P]
    assert torch.equal(H[..., :3, :3], o["rotmat"][:P])
    assert (H[..., 3, :3] == 0).all() and (H[..., :3, 3] == 0).all() and (H[..., 3, 3] == 1).all()
    # sigmoid(shape), dist with the clamp, loc, transl (multi_hmr.py:133-141)
    assert ((o["shape"][:P].double() - torch.sigmoid(shape_in[:P].double())).abs() <= 4 * U).all()
    Kd = K_use[det_b[:P].long()]
    Kd_dev = o["K_use"].double()[det_b[:P].long()]               # the kernel's own K (regressed: within tol_f)
    dist = Kd_dev[:, 0, 0] / torch.clamp(torch.exp(dist_pp[:P].double()), min=1e-5)
    tol_d = 8 * U * (2 + dist_pp[:P].double().abs()) * dist
    ed = (o["dist"][:P].double() - dist).abs()
    assert (ed <= tol_d).all(), (ed / tol_d).max().item()
    # sensitivity: without the clamp the two persons at dist_pp <= -12 fall outside the tolerance
    unclamped = Kd_dev[:, 0, 0] / torch.exp(dist_pp[:P].double())
    assert ((o["dist"][:P].double() - unclamped).abs() > tol_d).sum() == 2
    loc = (torch.stack([det_x[:P], det_y[:P]], 1).double() + 0.5 + offset[:P].double()) * 14
    assert ((o["loc"][:P].double() - loc).abs() <= 4 * U * loc.abs()).all()
    hom = torch.cat([loc, torch.ones(P, 1, dtype=torch.float64)], 1)
    transl = torch.einsum("pij,pj->pi", torch.inverse(Kd_dev), hom) * dist[:, None]
    tol_t = 32 * U * (torch.inverse(Kd_dev).abs() @ hom[..., None])[..., 0] * dist[:, None]
    et = (o["transl"][:P].double() - transl).abs()
    assert (et <= tol_t).all(), (et / tol_t).max().item()
    assert torch.equal(o["K_det"][:P], o["K_use"][det_b[:P].long()])
    assert (Kd - Kd_dev).abs().max() <= tol_f.max()
    print(f"  anny_person_post K={with_K}: rotmat err/tol {rR:.3f}, rotvec err/tol {rrv:.3f},"
          f" dist {(ed / tol_d).max().item():.3f}, transl {(et / tol_t).max().item():.3f}")


# ------------------------------------------------------------------------------------------------------ refine chain
def _refine_layers(D, depth, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    r = lambda *s: torch.randn(*s, device=dev, generator=g)
    return {"Wproj": r(depth, D, D) / math.sqrt(D), "bproj": r(depth, D) * 0.1,
            "ls1": torch.rand(depth, D, device=dev, generator=g) * 0.5 + 0.1,
            "ln2_g": torch.rand(depth, D, device=dev, generator=g) + 0.5, "ln2_b": r(depth, D) * 0.2,
            "Wfc1": r(depth, 4 * D, D) / math.sqrt(D), "bfc1": r(depth, 4 * D) * 0.1,
            "Wfc2": r(depth, D, 4 * D) / math.sqrt(4 * D), "bfc2": r(depth, D) * 0.1,
            "ls2": torch.rand(depth, D, device=dev, generator=g) * 0.5 + 0.1}


def _refine_ref(L, o16, rowidx, x, dtype):
    """dinov2 Block.forward's arithmetic for one row (layers/block.py): x += ls1 (proj(attn) + b);
    x += ls2 (fc2(gelu(fc1(norm2(x)))) + b), LayerNorm eps 1e-6, erf GELU."""
    x = x.to(dtype)
    c = {k: v.to(dtype) for k, v in L.items()}
    for l in range(o16.shape[0]):
        o = o16[l][rowidx.long()].to(dtype)
        x = x + c["ls1"][l] * (o @ c["Wproj"][l].t() + c["bproj"][l])
        y = F.layer_norm(x, (x.shape[1],), c["ln2_g"][l], c["ln2_b"][l], 1e-6)
        h = F.gelu(y @ c["Wfc1"][l].t() + c["bfc1"][l])
        x = x + c["ls2"][l] * (h @ c["Wfc2"][l].t() + c["bfc2"][l])
    return x


@pytest.mark.parametrize("D,depth", [(384, 1), (384, 4), (768, 1), (768, 4), (1024, 1), (1024, 4), (100, 2)])
def test_refine_chain(cuda_device, D, depth):
    """fp32 chain (persistent cooperative kernel, grid barrier, bulk copies) vs fp64.  Tolerance: no worse than 4x
    the error of torch fp32 (TF32 off) on the same inputs, plus 8 u of the row's largest |x|.  D = 100 (not a
    multiple of 32) covers the per-warp K slices of the chain."""
    from multihmr_b200 import ops

    dev = cuda_device
    L = _refine_layers(D, depth, dev, D * 10 + depth)
    R = 300
    g = torch.Generator(device=dev).manual_seed(D + depth)
    o16 = torch.randn(depth, R, D, device=dev, generator=g).half()
    for P in (0, 1, 8, 9, 17, 33):
        Pm = P + 3
        rowidx = torch.randperm(R, device=dev, generator=g)[:Pm].int()          # not monotonic
        x0 = torch.randn(Pm, D, device=dev, generator=g) * 1.5 + 0.7
        x0[:, 5] += 60.0                                                      # a massive channel, as in DINOv2
        if P > 2:
            x0[2, 17] -= 35.0
        x = x0.clone()
        ops.refine_chain(L, o16, rowidx, _count(dev, P), x)
        x2 = x0.clone()
        ops.refine_chain(L, o16, rowidx, _count(dev, P), x2)
        assert torch.equal(x, x2), "the chain must be bit-reproducible"
        assert torch.equal(x[P:], x0[P:]), "rows >= count must be untouched"
        if P == 0:
            continue
        ref = _refine_ref(L, o16, rowidx[:P], x0[:P], torch.float64)
        ref32 = _refine_ref(L, o16, rowidx[:P], x0[:P], torch.float32).double()
        err = (x[:P].double() - ref).abs().max().item()
        err32 = (ref32 - ref).abs().max().item()
        tol = 4 * err32 + 8 * U * ref.abs().max().item()
        print(f"  refine D={D} depth={depth} P={P}: err {err:.3e} (torch fp32 {err32:.3e}, tol {tol:.3e})")
        assert err <= tol, (err, tol)
        if P >= 2:   # sensitivity: every person paired with its neighbour's attention row
            bad = _refine_ref(L, o16, torch.roll(rowidx[:P], 1), x0[:P], torch.float64)
            assert (x[:P].double() - bad).abs().max().item() > tol
