"""Backbone-entry and folded-LayerNorm kernels (vit_misc.cu, the internal GEMM epilogues of gemm_tc.cu) through their
stage-level entry points, against plain fp64 torch references: the patch gathers of the fp32 and uint8 loaders, the
split of the residual stream with its row statistics, LayerNorm (fp32 and split sources, cls row dropped), the load-time
folding of a LayerNorm into the next Linear, and GEMM epilogue kinds 6-9.

Copies and single roundings are compared for exact equality.  Every other comparison states its tolerance next to it,
and every op has a sensitivity check: a reference with one plausible mistake must fall outside that tolerance.
Rows past M and columns past the written width are pre-filled with a sentinel and must come back untouched."""
import pytest
import torch
import torch.nn.functional as F

from fp64_util import SENTINEL, SENTINEL16, U, _acc_tol, _gelu_tol, _report, _ulp16

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _outliers(x, g, n=4, mag=150.0):
    """DINOv2-like massive-activation channels: a few columns of O(100) in every row."""
    cols = torch.randperm(x.shape[1], generator=g)[:n]
    x[:, cols] = mag * torch.sign(torch.randn(n, generator=g)) * (1 + torch.rand(x.shape[0], n, generator=g))
    return x


# ------------------------------------------------------------------------------------------------------------ im2col
def _im2col_ref(img, transpose=False):
    B, C, S, _ = img.shape
    h = S // 14
    t = img.reshape(B, C, h, 14, h, 14)  # b, c, gy, ky, gx, kx
    t = t.permute(0, 2, 4, 1, 5, 3) if transpose else t.permute(0, 2, 4, 1, 3, 5)
    return t.reshape(B * h * h, C * 196)


@pytest.mark.parametrize("S,B", [(224, 3), (280, 2), (896, 1), (1288, 2)])
def test_im2col_patch14(cuda_device, S, B):
    from multihmr_b200 import ops, preprocess

    dev = cuda_device
    g = _gen(S + B)
    M, ldA = B * (S // 14) ** 2, 592
    img = (torch.randn(B, 3, S, S, generator=g) * 1.3).to(dev)
    A = torch.full((M + 1, ldA), SENTINEL16, dtype=torch.float16, device=dev)
    ops.im2col_patch14(img, A[:M])
    ref = _im2col_ref(img).half()
    # a copy with one fp16 rounding: bit-exact, the last row / column of the grid included
    assert torch.equal(A[:M, :588], ref)
    assert torch.all(A[:M, 588:] == SENTINEL16) and torch.all(A[M] == SENTINEL16)
    # sensitivity: (kx, ky) transposed inside the patch
    assert not torch.equal(A[:M, :588], _im2col_ref(img, transpose=True).half())

    # uint8 HWC loader: the fp32 path applied to normalize_u8's output, bit for bit
    img8 = torch.randint(0, 256, (B, S, S, 3), generator=g, dtype=torch.uint8).to(dev)
    lut = torch.from_numpy(preprocess.normalize_rgb_table()).to(dev).contiguous()
    A8 = torch.full((M + 1, ldA), SENTINEL16, dtype=torch.float16, device=dev)
    ops.im2col_patch14(img8, A8[:M], lut=lut)
    via_f32 = torch.full_like(A8, SENTINEL16)
    ops.im2col_patch14(ops.normalize_u8(img8, lut), via_f32[:M])
    host = lut[torch.arange(3, device=dev)[None, :, None, None], img8.permute(0, 3, 1, 2).long()]
    assert torch.equal(A8, via_f32)
    assert torch.equal(A8[:M, :588], _im2col_ref(host).half())
    assert torch.all(A8[:M, 588:] == SENTINEL16) and torch.all(A8[M] == SENTINEL16)
    assert not torch.equal(A8[:M, :588], _im2col_ref(host, transpose=True).half())


# ---------------------------------------------------------------------------------------------------- split_rowstats
def _rows(M, D, g, mean=40.0, std=0.5, outliers=True):
    x = mean + std * torch.randn(M, D, generator=g)
    return _outliers(x, g) if outliers else x


@pytest.mark.parametrize("slots", [2, 4, 8])
@pytest.mark.parametrize("D", [384, 640, 768, 1024])
def test_split_rowstats(cuda_device, D, slots):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(D * 10 + slots)
    M, ld = 37, D + 64  # ragged against 8 rows per CTA; plane pitch > D
    x = _rows(M, D, g).to(dev)
    hi = torch.full((M + 2, ld), SENTINEL16, dtype=torch.float16, device=dev)
    lo = hi.clone()
    stats = torch.full((M + 2, slots, 2), SENTINEL, device=dev)
    ops.split_rowstats(x, hi[:M], lo[:M], stats[:M])
    # the split is two single roundings: exact
    assert torch.equal(hi[:M, :D], x.half())
    assert torch.equal(lo[:M, :D], (x - x.half().float()).half())
    for t in (hi, lo):
        assert torch.all(t[:M, D:] == SENTINEL16) and torch.all(t[M:] == SENTINEL16)
    assert torch.all(stats[:M, 1:] == 0.0) and torch.all(stats[M:] == SENTINEL)
    got = stats[:M, 0].double().cpu()
    xd = x.double().cpu()
    ref = torch.stack([xd.sum(1), (xd * xd).sum(1)], 1)
    # fp32 summation: each lane adds D/128 float4 pair sums in sequence, then 5 butterfly levels: depth <= D/128 + 7,
    # so |err| <= (D/128 + 8) u sum|x| (sum) and one more u for the squares (sum of squares)
    d = D // 128 + 8
    tol = torch.stack([d * U * xd.abs().sum(1), (d + 1) * U * (xd * xd).sum(1)], 1)
    err = (got - ref).abs()
    _report(f"split_rowstats D={D} slots={slots}", err, tol)
    assert torch.all(err <= tol)
    # sensitivity: the centred sum of squares (rows here have mean >> std)
    wrong = ((xd - xd.mean(1, keepdim=True)) ** 2).sum(1)
    assert torch.any((got[:, 1] - wrong).abs() > tol[:, 1])


# -------------------------------------------------------------------------------------------------------- layernorm
def _ln_tol(xd, g, b, D):
    """Two-pass fp32 LayerNorm bound (the kernel: mean, centred sum of squares, rsqrtf, (x - mean) rstd g + b).
    Sums have depth d = D/128 + 7 (see split_rowstats), so the mean is off by dm <= d u mean|x|, the variance by
    (d + 3) u relative (squares, sum, division, + eps) and rsqrtf adds 2 ulp: rstd is within (d/2 + 4) u relative,
    doubled for margin.  The output then carries |g| (|xhat| eps_r + rstd (dm + u |x - mean|)) plus 3 u of |g xhat| + |b|
    for the two products and the addition."""
    d = D // 128 + 7
    mean = xd.mean(1, keepdim=True)
    var = ((xd - mean) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-6)
    xhat = (xd - mean) * rstd
    dm = d * U * xd.abs().mean(1, keepdim=True)
    eps_r = (d + 8) * U
    return g.abs() * (xhat.abs() * eps_r + rstd * (dm + U * (xd - mean).abs())) + 3 * U * ((g * xhat).abs() + b.abs())


LN_CASES = [(v * 128, ri) for v in range(1, 9) for ri in (0, 17)]


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("D,rows_in", LN_CASES)
def test_layernorm(cuda_device, D, rows_in, split):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(D * 3 + rows_in + split)
    B = 3
    M = B * rows_in if rows_in else 41
    skip = 1 if rows_in else 0
    Mo = M - B * skip
    x = _rows(M, D, g, mean=3.0, std=1.0).to(dev)
    gamma = (0.5 + torch.rand(D, generator=g)).to(dev)
    beta = (0.3 * torch.randn(D, generator=g)).to(dev)
    out16 = torch.full((Mo + 2, D + 8), SENTINEL16, dtype=torch.float16, device=dev)
    out32 = torch.full((Mo + 2, D + 4), SENTINEL, device=dev)
    if split:
        hi = x.half()
        lo = (x - hi.float()).half()
        ops.layernorm(hi, gamma, beta, out16=out16[:Mo], out32=out32[:Mo], rows_in=rows_in, skip=skip, xlo=lo)
        xd = hi.double() + lo.double()
    else:
        ops.layernorm(x, gamma, beta, out16=out16[:Mo], out32=out32[:Mo], rows_in=rows_in, skip=skip)
        xd = x.double()
    xd, gd, bd = xd.cpu(), gamma.double().cpu(), beta.double().cpu()
    keep = torch.ones(M, dtype=torch.bool)
    if rows_in:
        keep[torch.arange(M) % rows_in < skip] = False
    ref = F.layer_norm(xd[keep], (D,), gd, bd, 1e-6)
    tol32 = _ln_tol(xd[keep], gd, bd, D)
    got32 = out32[:Mo, :D].double().cpu()
    err32 = (got32 - ref).abs()
    _report(f"layernorm D={D} rows_in={rows_in} split={split} fp32", err32, tol32)
    assert torch.all(err32 <= tol32)
    # fp16 output: the fp32 value rounded once more (half an fp16 ulp)
    tol16 = tol32 + 0.5 * _ulp16(ref.abs() + tol32)
    err16 = (out16[:Mo, :D].double().cpu() - ref).abs()
    _report(f"layernorm D={D} rows_in={rows_in} split={split} fp16", err16, tol16)
    assert torch.all(err16 <= tol16)
    assert torch.all(out32[:Mo, D:] == SENTINEL) and torch.all(out32[Mo:] == SENTINEL)
    assert torch.all(out16[:Mo, D:] == SENTINEL16) and torch.all(out16[Mo:] == SENTINEL16)
    # sensitivity: the cls row kept (skip 0) / the unbiased variance
    if rows_in:
        wrong = F.layer_norm(xd, (D,), gd, bd, 1e-6)[:Mo]
    else:
        xc = xd - xd.mean(1, keepdim=True)
        wrong = xc / torch.sqrt((xc * xc).sum(1, keepdim=True) / (D - 1) + 1e-6) * gd + bd
    assert torch.any((got32 - wrong).abs() > tol32)


# --------------------------------------------------------------------------------------------------- fold_ln_linear
@pytest.mark.parametrize("N,K", [(1152, 384), (1536, 384), (2304, 768), (3072, 768), (3072, 1024), (4096, 1024)])
def test_fold_ln_linear(cuda_device, N, K):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(N + K)
    w = (torch.randn(N, K, generator=g) * 0.05 + 0.01).to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    ln_g = (0.5 + torch.rand(K, generator=g)).to(dev)
    ln_b = (0.2 * torch.randn(K, generator=g)).to(dev)
    w16, b2 = ops.fold_ln_linear(w, bias, ln_g, ln_b)
    wd, gd = w.double().cpu(), ln_g.double().cpu()
    c = wd * gd
    mean = c.mean(1, keepdim=True)
    ref = c - mean
    # W16: fp32 w*g (1 u) and a row mean summed by 32 lanes in sequence (K/32 terms) plus 5 butterfly levels:
    # dm <= (K/32 + 6) u mean|c|; the difference rounds once in fp32, then once to fp16 (half an fp16 ulp)
    dm = (K // 32 + 6) * U * c.abs().mean(1, keepdim=True)
    pre = 2 * U * c.abs() + dm + U * ref.abs()
    tol = 0.5 * _ulp16(ref.abs() + pre) + pre
    got = w16.double().cpu()
    err = (got - ref).abs()
    _report(f"fold_ln_linear N={N} K={K} W16", err, tol)
    assert torch.all(err <= tol)
    # bias2 = bias + sum_k ln_b[k] W[n,k]: fp32 products and the same summation depth
    terms = ln_b.double().cpu() * wd
    bref = bias.double().cpu() + terms.sum(1)
    btol = (K // 32 + 7) * U * terms.abs().sum(1) + 2 * U * bref.abs()
    berr = (b2.double().cpu() - bref).abs()
    _report(f"fold_ln_linear N={N} K={K} bias2", berr, btol)
    assert torch.all(berr <= btol)
    # sensitivity: rows not centred
    assert torch.any((got - c).abs() > tol)


# ---------------------------------------------------------------------------------------------------- GEMM kinds 6-9
@pytest.mark.parametrize("bn,N,M", [(128, 384, 300), (512, 768, 300), (512, 1024, 77)])
def test_gemm_split_residual_and_stats(cuda_device, bn, N, M):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(bn + N + M)
    K = 384
    a = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    bias = torch.randn(N, generator=g)
    gamma = 0.1 + torch.rand(N, generator=g)
    x = 2.0 + torch.randn(M, N, generator=g)
    x = _outliers(x, g, mag=60.0)
    ld = N + 64
    hi = torch.full((M + 3, ld), SENTINEL16, dtype=torch.float16)
    lo = hi.clone()
    hi[:M, :N] = x.half()
    lo[:M, :N] = (x - x.half().float()).half()
    tile = 128 if bn == 128 else 256
    slots = 2 * ((N + tile - 1) // tile)
    stats = torch.full((M + 3, slots, 2), SENTINEL)
    hi, lo, stats = hi.to(dev), lo.to(dev), stats.to(dev)
    x_in = hi[:M, :N].double().cpu() + lo[:M, :N].double().cpu()
    ops.gemm_internal(a.to(dev), w.to(dev), ops.EPI_LS_RESID_SPLIT, bn, bias=bias.to(dev), gamma=gamma.to(dev),
                      hi=hi[:M], lo=lo[:M], stats=stats[:M])
    ad, wd = a.double(), w.double()
    gd, bd = gamma.double(), bias.double()
    ref = x_in + gd * (ad @ wd.t() + bd)
    # the fp32 value: gamma (acc + b) + x as one fma after the acc + b rounding, then split into 22 bits (hi + lo is
    # within 2^-22 of it, 2^-25 absolute where lo is subnormal)
    e_a = gd * (_acc_tol(ad, wd) + U * (ad @ wd.t() + bd).abs()) + U * ref.abs()
    tol = e_a + 2.0 ** -22 * ref.abs() + 2.0 ** -25
    got = hi[:M, :N].double().cpu() + lo[:M, :N].double().cpu()
    err = (got - ref).abs()
    _report(f"gemm kind 6 bn={bn} N={N} x", err, tol)
    assert torch.all(err <= tol)
    assert torch.all(hi[:M, N:] == SENTINEL16) and torch.all(hi[M:] == SENTINEL16)
    assert torch.all(lo[:M, N:] == SENTINEL16) and torch.all(lo[M:] == SENTINEL16)
    assert torch.all(stats[M:] == SENTINEL)
    # every slot holds the partial sums of its own N/slots columns: slot 2 n_blk + half covers tile/2 columns
    wcols = N // slots
    parts = ref.reshape(M, slots, wcols)
    eparts = e_a.reshape(M, slots, wcols)
    s_ref = parts.sum(2)
    q_ref = (parts * parts).sum(2)
    # a lane adds 8 columns per 32-column chunk in sequence, over wcols/32 chunks, then 2 shuffle levels:
    # depth <= wcols/4 + 3
    d = wcols // 4 + 4
    s_tol = eparts.sum(2) + d * U * parts.abs().sum(2)
    q_tol = (2 * parts.abs() * eparts).sum(2) + (d + 1) * U * (parts * parts).sum(2)
    gs = stats[:M].double().cpu()
    es, eq = (gs[..., 0] - s_ref).abs(), (gs[..., 1] - q_ref).abs()
    _report(f"gemm kind 6 bn={bn} N={N} stats", torch.cat([es, eq]), torch.cat([s_tol, q_tol]))
    assert torch.all(es <= s_tol) and torch.all(eq <= q_tol)
    # sensitivity: stats written to the other half's slot
    swapped = s_ref.reshape(M, slots // 2, 2).flip(2).reshape(M, slots)
    assert torch.any((gs[..., 0] - swapped).abs() > s_tol)


@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("slots,spread", [(2, 2), (4, 4), (6, 6), (8, 8), (8, 1)])
def test_gemm_folded_ln_consumer(cuda_device, slots, spread, gelu):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(slots * 10 + spread + gelu)
    M, K, N = 300, 384, 512
    a = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    bias = torch.randn(N, generator=g)
    # statistics of rows with mean 0.5 and std 0.2 .. 2, split into `spread` random parts over the last slots
    xr = 0.5 + torch.randn(M, K, generator=g) * (0.2 + 1.8 * torch.rand(M, 1, generator=g))
    tot = torch.stack([xr.double().sum(1), (xr.double() ** 2).sum(1)], 1)
    frac = torch.rand(M, spread, generator=g, dtype=torch.float64)
    frac = frac / frac.sum(1, keepdim=True)
    stats = torch.zeros(M, slots, 2)
    stats[:, slots - spread:] = (frac[:, :, None] * tot[:, None, :]).float()
    out = torch.full((M + 2, N + 8), SENTINEL16, dtype=torch.float16, device=dev)
    kind = ops.EPI_LN_GELU_F16 if gelu else ops.EPI_LN_BIAS_F16
    ops.gemm_internal(a.to(dev), w.to(dev), kind, 256, out=out[:M], bias=bias.to(dev), stats=stats.to(dev))
    ad, wd, bd = a.double(), w.double(), bias.double()
    sd = stats.double()

    def ref_of(st):
        s, q = st[..., 0].sum(1, keepdim=True), st[..., 1].sum(1, keepdim=True)
        mean = s / K
        rstd = 1.0 / torch.sqrt((q / K - mean * mean).clamp_min(0.0) + 1e-6)
        return rstd, rstd * (ad @ wd.t()) + bd

    rstd, pre = ref_of(sd)
    # rstd: <= 8 positive slot values summed in fp32 (7 u), q/K - mean^2 cancels by q/(K var) (rows here: <= 7.3),
    # so the variance is within ~80 u and rstd (rsqrtf: 2 ulp) within ~42 u relative: 128 u leaves margin; then
    # rstd acc + b' as one fma
    acc = ad @ wd.t()
    e_pre = rstd * (_acc_tol(ad, wd) + 128 * U * acc.abs()) + U * pre.abs()
    ref = F.gelu(pre) if gelu else pre
    tol = e_pre * 1.13 + (_gelu_tol(pre) if gelu else 0.0)
    tol = tol + 0.5 * _ulp16(ref.abs() + tol)  # one fp16 rounding of the output
    got = out[:M, :N].double().cpu()
    err = (got - ref).abs()
    _report(f"gemm kind {kind} slots={slots} spread={spread}", err, tol)
    assert torch.all(err <= tol)
    assert torch.all(out[:M, N:] == SENTINEL16) and torch.all(out[M:] == SENTINEL16)
    # sensitivity: reading one slot fewer
    _, pre_w = ref_of(sd[:, :-1])
    wrong = F.gelu(pre_w) if gelu else pre_w
    assert torch.any((got - wrong).abs() > tol)


@pytest.mark.parametrize("M,rows_in,bn", [(300, 97, 128), (4096 + 5, 2304, 256), (513, 256, 512)])
def test_gemm_rowadd_f16(cuda_device, M, rows_in, bn):
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(M + rows_in + bn)
    K, N = 384, 512
    a = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    table = torch.randn(rows_in, N, generator=g)
    out = torch.full((M + 2, N + 8), SENTINEL16, dtype=torch.float16, device=dev)
    ops.gemm_internal(a.to(dev), w.to(dev), ops.EPI_ROWADD_F16, bn, out=out[:M], rowadd=table.to(dev), rows_in=rows_in)
    ad, wd = a.double(), w.double()
    rows = torch.arange(M) % rows_in
    ref = ad @ wd.t() + table.double()[rows]
    # accumulation, one fp32 addition, one fp16 rounding
    tol = _acc_tol(ad, wd) + U * ref.abs()
    tol = tol + 0.5 * _ulp16(ref.abs() + tol)
    got = out[:M, :N].double().cpu()
    err = (got - ref).abs()
    _report(f"gemm kind 9 M={M} rows_in={rows_in} bn={bn}", err, tol)
    assert torch.all(err <= tol)
    assert torch.all(out[:M, N:] == SENTINEL16) and torch.all(out[M:] == SENTINEL16)
    # sensitivity: row m of a longer table instead of m % rows_in
    longer = torch.cat([table.double(), torch.randn(M, N, generator=g, dtype=torch.float64)])
    wrong = ad @ wd.t() + longer[torch.arange(M)]
    assert torch.any((got - wrong).abs() > tol)
