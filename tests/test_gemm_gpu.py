"""wgmma GEMM family (gemm_tc.cu, public epilogues 0-5) against plain fp64 references on the same fp16 operands.

Two kinds of check:
  * exact products: A and W in {-1, 0, 1} with small integer bias, table and residual and gamma = 0.5 make every
    partial sum an integer below 2^11, so the result does not depend on the summation order and must EQUAL the fp64
    reference.  These run the tile-schedule sweep (tiles per CTA, k blocks against the stage ring), the M / N / K
    edges and the row remap, each into a sentinel canvas whose guard band must come back untouched.
  * random data: a per-element bound from the rounding points (fp64_util._acc_tol for the fp32 accumulation, one
    rounding per epilogue operation, _gelu_tol, half an fp16 ulp for fp16 outputs), with a sensitivity check: a
    reference with one plausible mistake must fall outside it.
Plus pitched operands with NaN pads, batch-size invariance, determinism, and a plan built for more rows than it runs
(how the engine runs its maximum-batch plans)."""
import pytest
import torch

from fp64_util import SENTINEL, SENTINEL16, U, _acc_tol, _gelu_tol, _report, _ulp16

pytestmark = pytest.mark.gpu

STAGES = {128: 5, 256: 3, 512: 3}  # smem ring depth of gemm_tc.cu per block_n
F16_KINDS = (0, 1, 2)  # EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_RELU_F16


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _ref_linear(a16, w16):
    return a16.double() @ w16.double().t()


def _canvas(M, N, dtype, dev, fill=None, rows=2, cols=8):
    """A [M + rows, N + cols] sentinel canvas; the call writes into its [:M, :N] view."""
    if fill is None:
        fill = SENTINEL16 if dtype == torch.float16 else SENTINEL
    return torch.full((M + rows, N + cols), fill, dtype=dtype, device=dev)


def _guard_ok(c, M, N, fill):
    return bool(torch.all(c[:M, N:] == fill)) and bool(torch.all(c[M:] == fill))


# ------------------------------------------------------------------------------------------------ exact products
def _tern(*shape, g):
    return torch.randint(-1, 2, shape, generator=g).half()


def _ints(*shape, g, lo=-4, hi=5):
    return torch.randint(lo, hi, shape, generator=g).float()


def _exact_case(kind, M, N, K, g, dev, lda=None):
    """Operands, arguments and the fp64 result of one exact-product call of `kind`; the output canvas is
    pre-filled (the residual rows for kind 3, the sentinel elsewhere)."""
    a, w = _tern(M, K, g=g), _tern(N, K, g=g)
    acc = _ref_linear(a, w)
    kw, f16 = {}, kind in F16_KINDS
    fill = SENTINEL16 if f16 else SENTINEL
    canvas = _canvas(M, N, torch.float16 if f16 else torch.float32, dev)
    if kind in (0, 1, 2, 3, 5):
        bias = _ints(N, g=g)
        kw["bias"] = bias.to(dev)
        pre = acc + bias.double()
    if kind == 5 and N % 64 == 32:  # the null-bias form of EPI_BIAS_F32 (HPH to_kv)
        kw.pop("bias")
        pre = acc
    if kind == 0:
        ref = pre
    elif kind == 2:
        ref = pre.clamp_min(0)
    elif kind == 1:
        ref = None  # GELU is not exact: covered by the per-element test
    elif kind == 3:
        x0 = _ints(M, N, g=g, lo=-64, hi=65)
        canvas[:M, :N] = x0.to(dev)
        kw["gamma"] = torch.full((N,), 0.5, device=dev)
        ref = x0.double() + 0.5 * pre
    elif kind == 4:
        table = _ints(M, N, g=g)
        kw.update(rowadd=table.to(dev), rows_in=M, rows_out=M, row_off=0)
        ref = acc + table.double()
    else:
        ref = pre
    return a.to(dev), w.to(dev), kw, canvas, fill, ref


def _pitched(t):
    """t as a column view of a buffer with a pitch of a multiple of 8 (TMA) and NaN pad columns, when K needs one."""
    K = t.shape[1]
    if K % 8 == 0:
        return t
    big = torch.full((t.shape[0], (K + 7) // 8 * 8), float("nan"), dtype=t.dtype, device=t.device)
    big[:, :K] = t
    return big[:, :K]


def _run_exact(kind, M, N, K, bn, seed, dev):
    from multihmr_b200 import ops

    a, w, kw, canvas, fill, ref = _exact_case(kind, M, N, K, _gen(seed), dev)
    ops.gemm_f16(_pitched(a), _pitched(w), kind, canvas[:M, :N], block_n=bn, **kw)
    got = canvas[:M, :N].double()
    assert torch.equal(got, ref.to(dev)), (kind, M, N, K, bn, (got - ref.to(dev)).abs().max().item())
    assert _guard_ok(canvas, M, N, fill), (kind, M, N, K, bn)


@pytest.mark.parametrize("bn", [128, 256, 512])
@pytest.mark.parametrize("kind", [0, 2, 3, 4, 5])
@pytest.mark.parametrize("M,N,K", [(385, 800, 200), (300, 832, 16), (129, 288, 40), (257, 544, 588),
                                   (200, 1056, 1152)])
def test_gemm_exact_products(cuda_device, kind, bn, M, N, K):
    """Integer-valued operands: zero tolerance, so a misplaced k block, tile, column half or 32-column chunk shows.
    N = 800 / 288 / 544 / 1056 end in a partial tile (and an odd 32-column chunk count: the null-bias form of
    EPI_BIAS_F32); K = 16 / 40 / 200 / 588 end in a partial k block."""
    _run_exact(kind, M, N, K, bn, kind * 1000 + bn + M + N + K, cuda_device)


def _sweep_shape(bn, tiles):
    """(M, N) with exactly `tiles` output tiles (128 x bn, or 256 x 256 for the CTA pair), the last M block partial."""
    tm = 256 if bn == 512 else 128
    tn = 256 if bn == 512 else bn
    n_blk = 2 if tiles % 2 == 0 else 1
    m_blk = tiles // n_blk
    return tm * (m_blk - 1) + tm - 37, tn * n_blk


@pytest.mark.parametrize("bn", [128, 256, 512])
@pytest.mark.parametrize("which", ["1", "sms-1", "sms", "sms+1", "2sms+1"])
def test_gemm_tile_schedule_sweep(cuda_device, bn, which):
    """Persistent schedule: 0, 1 or 2 extra tiles per CTA (CTA pair: per pair of SMs), each at k-block counts of
    1, stages - 1, stages and stages + 1, where the stage / phase state carries across tiles and wraps."""
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    units = sms // 2 if bn == 512 else sms
    tiles = {"1": 1, "sms-1": units - 1, "sms": units, "sms+1": units + 1, "2sms+1": 2 * units + 1}[which]
    M, N = _sweep_shape(bn, tiles)
    st = STAGES[bn]
    for i, nkb in enumerate(sorted({1, st - 1, st, st + 1})):
        K = 64 * nkb - (24 if i % 2 else 0)  # every other count with a partial last k block
        kind = (0, 3, 5, 2)[i]
        _run_exact(kind, M, N, K, bn, tiles * 10 + nkb, cuda_device)


@pytest.mark.parametrize("M", [1, 127, 128, 129, 255, 256, 257, 385])
def test_gemm_edges_rows_pair(cuda_device, M):
    """bn 512: M rows give an empty or partial rank-1 half of the CTA pair."""
    for kind in (0, 3, 4):
        _run_exact(kind, M, 512, 128, 512, M * 7 + kind, cuda_device)


@pytest.mark.parametrize("bn", [256, 512])
@pytest.mark.parametrize("N", [32, 96, 160, 288])
def test_gemm_edges_columns(cuda_device, bn, N):
    """N smaller than a consumer half (empty second consumer) and partial last 32-column chunks."""
    for kind in (0, 2, 3, 5):
        _run_exact(kind, 300, N, 192, bn, N * 3 + bn + kind, cuda_device)


@pytest.mark.parametrize("bn,D", [(128, 384), (512, 1024)])
def test_gemm_rowadd_guard_rows(cuda_device, bn, D):
    """Patch-embed scatter (ViT-S at bn 128, ViT-B/L at bn 512): image b's rows land at b * rows_out + 1 + n; the
    cls rows, the gap rows before the next image and the rows after the last image keep the sentinel."""
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(bn + D)
    B, rows_in, K = 3, 197, 588
    rows_out = rows_in + 3
    M = B * rows_in
    a, w = _tern(M, K, g=g), _tern(D, K, g=g)
    table = _ints(rows_in, D, g=g)
    out = torch.full((B * rows_out + 2, D + 8), SENTINEL, device=dev)
    ops.gemm_f16(_pitched(a.to(dev)), _pitched(w.to(dev)), ops.EPI_ROWADD_F32, out[:B * rows_out, :D], rowadd=table.to(dev),
                 rows_in=rows_in, rows_out=rows_out, row_off=1, block_n=bn)
    ref = (_ref_linear(a, w).view(B, rows_in, D) + table.double()).to(dev)
    got = out[:B * rows_out].view(B, rows_out, D + 8).double()
    assert torch.equal(got[:, 1:1 + rows_in, :D], ref)
    written = torch.zeros(B * rows_out + 2, D + 8, dtype=torch.bool, device=dev)
    written[:B * rows_out].view(B, rows_out, D + 8)[:, 1:1 + rows_in, :D] = True
    assert torch.all(out[~written] == SENTINEL)


def test_gemm_pitched_operands(cuda_device):
    """A and W as column views of wider buffers with fp16 NaN in the pad columns and NaN rows after M in A's
    allocation (the engine's ctx16 with lda = D + 128 > K): bitwise the contiguous result."""
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(7)
    for (M, N, K, lda, bn, kind) in [(300, 384, 384, 512, 128, 2), (1000, 1024, 1024, 1152, 512, 2),
                                     (257, 768, 768, 896, 256, 0), (129, 512, 40, 64, 512, 5)]:
        a = torch.randn(M, K, generator=g).half().to(dev)
        w = (torch.randn(N, K, generator=g) * 0.05).half().to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        dt = torch.float16 if kind in F16_KINDS else torch.float32
        want = torch.empty(M, N, dtype=dt, device=dev)
        ops.gemm_f16(a, w, kind, want, bias=bias, block_n=bn)
        abig = torch.full((M + 5, lda), float("nan"), dtype=torch.float16, device=dev)
        abig[:M, :K] = a
        wbig = torch.full((N, lda + 8), float("nan"), dtype=torch.float16, device=dev)
        wbig[:, :K] = w
        got = torch.empty_like(want)
        ops.gemm_f16(abig[:M, :K], wbig[:, :K], kind, got, bias=bias, block_n=bn)
        assert torch.equal(got, want), (M, N, K, lda, bn)


# ------------------------------------------------------------------------------------------- fp64 per-element bounds
SHAPES = [
    # (M, N, K): multiples, M tails, K tails (588 -> padded 592), ViT-S dims, big
    (128, 256, 64),
    (256, 256, 128),
    (300, 1024, 1024),
    (4097, 3072, 1024),
    (2305, 384, 1536),
    (1000, 1152, 384),
    (513, 1024, 592),
    (4096, 1024, 1152),
    (64, 32, 1024),
]


def _neighbour_chunk(v):
    """The vector with each 32-column chunk replaced by its neighbour's (chunks swapped in pairs, N >= 64)."""
    n = v.shape[-1] // 64 * 64
    out = v.clone()
    out[..., :n] = v[..., :n].reshape(*v.shape[:-1], -1, 2, 32).flip(-2).reshape(*v.shape[:-1], n)
    return out


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("bn", [128, 256, 512])
def test_gemm_bias_f16(cuda_device, M, N, K, bn):
    from multihmr_b200 import ops

    dev = cuda_device
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = (torch.randn(M, K, generator=g) * 1.0).to(dev).half()
    w = (torch.randn(N, K, generator=g) * 0.05).to(dev).half()
    bias = torch.randn(N, generator=g).to(dev)
    canvas = _canvas(M, N, torch.float16, dev)
    ops.gemm_f16(a, w, ops.EPI_BIAS_F16, canvas[:M, :N], bias=bias, block_n=bn)
    acc = _ref_linear(a, w)
    ref = acc + bias.double()
    # fp32 accumulation, the bias add (one rounding), one fp16 rounding of the output
    tol = _acc_tol(a.double(), w.double()) + U * ref.abs()
    tol = tol + 0.5 * _ulp16(ref.abs() + tol)
    got = canvas[:M, :N].double()
    err = (got - ref).abs()
    _report(f"gemm bias_f16 M={M} N={N} K={K} bn={bn}", err, tol)
    assert torch.all(err <= tol)
    assert _guard_ok(canvas, M, N, SENTINEL16)
    # sensitivity: the bias of the neighbouring 32-column chunk; the last 16 K columns dropped
    if N >= 64:
        assert torch.any((got - (acc + _neighbour_chunk(bias).double())).abs() > tol)
    if K == 592:
        assert torch.any((got - (_ref_linear(a[:, :576], w[:, :576]) + bias.double())).abs() > tol)


@pytest.mark.parametrize("bn", [128, 256, 512])
@pytest.mark.parametrize("epi", ["gelu", "relu"])
def test_gemm_act_f16(cuda_device, epi, bn):
    from multihmr_b200 import ops

    dev = cuda_device
    M, N, K = 1537, 4096, 1024
    g = torch.Generator(device="cpu").manual_seed(5)
    a = torch.randn(M, K, generator=g).to(dev).half()
    w = (torch.randn(N, K, generator=g) * 0.03).to(dev).half()
    bias = torch.randn(N, generator=g).to(dev)
    canvas = _canvas(M, N, torch.float16, dev)
    kind = ops.EPI_BIAS_GELU_F16 if epi == "gelu" else ops.EPI_BIAS_RELU_F16
    ops.gemm_f16(a, w, kind, canvas[:M, :N], bias=bias, block_n=bn)
    pre = _ref_linear(a, w) + bias.double()
    e_pre = _acc_tol(a.double(), w.double()) + U * pre.abs()
    if epi == "gelu":
        ref = torch.nn.functional.gelu(pre)
        tol = 1.13 * e_pre + _gelu_tol(pre)  # |gelu'| <= 1.13
    else:
        ref, tol = pre.clamp_min(0), e_pre
    tol = tol + 0.5 * _ulp16(ref.abs() + tol)
    got = canvas[:M, :N].double()
    err = (got - ref).abs()
    _report(f"gemm {epi}_f16 bn={bn}", err, tol)
    assert torch.all(err <= tol)
    assert _guard_ok(canvas, M, N, SENTINEL16)
    # sensitivity: the bias of the neighbouring chunk
    act = torch.nn.functional.gelu if epi == "gelu" else (lambda y: y.clamp_min(0))
    wrong = act(_ref_linear(a, w) + _neighbour_chunk(bias).double())
    assert torch.any((got - wrong).abs() > tol)


@pytest.mark.parametrize("bn", [128, 256, 512])
def test_gemm_layerscale_residual_f32(cuda_device, bn):
    from multihmr_b200 import ops

    dev = cuda_device
    M, N, K = 4097 * 2, 1024, 4096
    g = torch.Generator(device="cpu").manual_seed(11)
    a = torch.randn(M, K, generator=g).to(dev).half()
    w = (torch.randn(N, K, generator=g) * 0.02).to(dev).half()
    bias = torch.randn(N, generator=g).to(dev)
    gamma = torch.rand(N, generator=g).to(dev)
    x0 = torch.randn(M, N, generator=g).to(dev)
    canvas = _canvas(M, N, torch.float32, dev)
    canvas[:M, :N] = x0
    ops.gemm_f16(a, w, ops.EPI_LS_RESID_F32, canvas[:M, :N], bias=bias, gamma=gamma, block_n=bn)
    acc = _ref_linear(a, w)
    gd, bd = gamma.double(), bias.double()
    ref = x0.double() + gd * (acc + bd)
    # acc + b (one rounding), times gamma (one rounding, or none in an fma), plus x (one rounding)
    tol = gd * (_acc_tol(a.double(), w.double()) + 2 * U * (acc + bd).abs()) + U * ref.abs()
    got = canvas[:M, :N].double()
    err = (got - ref).abs()
    _report(f"gemm ls_resid_f32 bn={bn}", err, tol)
    assert torch.all(err <= tol)
    assert _guard_ok(canvas, M, N, SENTINEL)
    # sensitivity: the layer scale applied after the bias instead of to (acc + bias)
    assert torch.any((got - (x0.double() + gd * acc + bd)).abs() > tol)


def test_gemm_rowadd_remap_f32(cuda_device):
    """Patch-embed shape: rows of image b land at b*T + 1 + n, with a per-n additive table; ViT-S (D = 384) at
    bn 128 and ViT-L (D = 1024) at bn 512, as the engine runs them."""
    from multihmr_b200 import ops

    dev = cuda_device
    for bn, D in ((128, 384), (512, 1024)):
        B, Np, K = 3, 2304, 592
        T = Np + 1
        g = torch.Generator(device="cpu").manual_seed(13)
        a = torch.randn(B * Np, K, generator=g).to(dev).half()
        w = (torch.randn(D, K, generator=g) * 0.05).to(dev).half()
        table = torch.randn(Np, D, generator=g).to(dev)
        out = _canvas(B * T, D, torch.float32, dev, fill=7.0)
        ops.gemm_f16(a, w, ops.EPI_ROWADD_F32, out[:B * T, :D], rowadd=table, rows_in=Np, rows_out=T, row_off=1,
                     block_n=bn)
        ref = _ref_linear(a, w).view(B, Np, D) + table.double()
        got = out[:B * T].view(B, T, D + 8)
        assert torch.all(got[:, 0] == 7.0) and torch.all(got[:, :, D:] == 7.0) and torch.all(out[B * T:] == 7.0)
        g64 = got[:, 1:, :D].double()
        # accumulation and one fp32 addition
        tol = _acc_tol(a.double(), w.double()).view(B, Np, D) + U * ref.abs()
        err = (g64 - ref).abs()
        _report(f"gemm rowadd_f32 bn={bn}", err, tol)
        assert torch.all(err <= tol)
        # sensitivity: the last 16 K columns dropped
        wrong = _ref_linear(a[:, :576], w[:, :576]).view(B, Np, D) + table.double()
        assert torch.any((g64 - wrong).abs() > tol)


@pytest.mark.parametrize("bn", [128, 256, 512])
def test_gemm_bias_f32_nobias(cuda_device, bn):
    from multihmr_b200 import ops

    dev = cuda_device
    M, N, K = 2304, 1024, 1152
    g = torch.Generator(device="cpu").manual_seed(17)
    a = torch.randn(M, K, generator=g).to(dev).half()
    w = (torch.randn(N, K, generator=g) * 0.05).to(dev).half()
    bias = torch.randn(N, generator=g).to(dev)
    for b in (None, bias):
        canvas = _canvas(M, N, torch.float32, dev)
        ops.gemm_f16(a, w, ops.EPI_BIAS_F32, canvas[:M, :N], bias=b, block_n=bn)
        acc = _ref_linear(a, w)
        ref = acc if b is None else acc + b.double()
        tol = _acc_tol(a.double(), w.double()) + U * ref.abs()
        got = canvas[:M, :N].double()
        err = (got - ref).abs()
        _report(f"gemm bias_f32 bn={bn} bias={b is not None}", err, tol)
        assert torch.all(err <= tol)
        assert _guard_ok(canvas, M, N, SENTINEL)
        # sensitivity: the last 16 K columns dropped (K = 1152 = 18 k blocks)
        wrong = _ref_linear(a[:, :K - 16], w[:, :K - 16]) + (0 if b is None else b.double())
        assert torch.any((got - wrong).abs() > tol)


# ------------------------------------------------------------------------------------ invariance and plan reuse
@pytest.mark.parametrize("bn", [128, 256, 512])
def test_gemm_row_count_invariance(cuda_device, bn):
    """Rows [0, m) of a call on M rows equal a call on the first m rows bit for bit; two identical calls are equal."""
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(bn)
    M, N, K = 1300, 1024, 768
    a = torch.randn(M, K, generator=g).half().to(dev)
    w = (torch.randn(N, K, generator=g) * 0.05).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    full = torch.empty(M, N, dtype=torch.float16, device=dev)
    ops.gemm_f16(a, w, ops.EPI_BIAS_GELU_F16, full, bias=bias, block_n=bn)
    again = torch.empty_like(full)
    ops.gemm_f16(a, w, ops.EPI_BIAS_GELU_F16, again, bias=bias, block_n=bn)
    assert torch.equal(full, again)
    for m in (1, 129, 257, 1000):
        part = torch.empty(m, N, dtype=torch.float16, device=dev)
        ops.gemm_f16(a[:m], w, ops.EPI_BIAS_GELU_F16, part, bias=bias, block_n=bn)
        assert torch.equal(part, full[:m]), m


@pytest.mark.parametrize("bn", [128, 256, 512])
@pytest.mark.parametrize("kind", [0, 3, 6, 9])
def test_gemm_plan_reuse_smaller_m(cuda_device, kind, bn):
    """A plan built for M_plan rows run on M_run < M_plan (the engine's maximum-batch plans at a smaller batch), with
    NaN in A's rows M_run .. M_plan: rows below M_run equal a fresh M_run-row call bit for bit (output, split planes
    and statistics), and nothing from row M_run on is written."""
    from multihmr_b200 import ops

    dev = cuda_device
    g = _gen(kind * 10 + bn)
    M_plan, N, K = 1031, 512, 384
    a = torch.randn(M_plan, K, generator=g).half().to(dev)
    w = (torch.randn(N, K, generator=g) * 0.05).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    gamma = (0.1 + torch.rand(N, generator=g)).to(dev)
    x0 = torch.randn(M_plan, N, generator=g).to(dev)
    table = torch.randn(97, N, generator=g).to(dev)
    tile = 128 if bn == 128 else 256
    slots = 2 * (N // tile)

    def run(rows, a_in, m_run=None):
        """Fresh buffers sized for `rows`; returns every tensor the call may write."""
        kw, bufs = dict(bias=bias), {}
        if kind == 0:
            bufs["out"] = _canvas(rows, N, torch.float16, dev)
            kw["out"] = bufs["out"][:rows, :N]
        elif kind == 3:
            bufs["out"] = _canvas(rows, N, torch.float32, dev)
            bufs["out"][:rows, :N] = x0[:rows]
            kw.update(out=bufs["out"][:rows, :N], gamma=gamma)
        elif kind == 6:
            hi = _canvas(rows, N, torch.float16, dev)
            lo = hi.clone()
            hi[:rows, :N] = x0[:rows].half()
            lo[:rows, :N] = (x0[:rows] - x0[:rows].half().float()).half()
            stats = torch.full((rows + 2, slots, 2), SENTINEL, device=dev)
            bufs.update(hi=hi, lo=lo, stats=stats)
            kw.update(gamma=gamma, hi=hi[:rows, :N], lo=lo[:rows, :N], stats=stats[:rows])
        else:
            bufs["out"] = _canvas(rows, N, torch.float16, dev)
            kw = dict(out=bufs["out"][:rows, :N], rowadd=table, rows_in=97)
        ops.gemm_internal(a_in, w, kind, bn, m_run=m_run, **kw)
        return bufs

    for M_run in (1, 200, 513, 1030):
        a_nan = a.clone()
        a_nan[M_run:] = float("nan")
        got = run(M_plan, a_nan, m_run=M_run)
        want = run(M_run, a[:M_run].clone())
        for name, t in got.items():
            assert torch.equal(t[:M_run], want[name][:M_run]), (name, M_run)
            if name == "stats":
                assert torch.all(t[M_run:] == SENTINEL), (name, M_run)
            else:
                fill = SENTINEL16 if t.dtype == torch.float16 else SENTINEL
                ref_rest = t.new_full(t[M_run:].shape, fill)
                if kind == 3:
                    ref_rest[:M_plan - M_run, :N] = x0[M_run:]
                if kind == 6:
                    src = x0[M_run:]
                    ref_rest[:M_plan - M_run, :N] = src.half() if name == "hi" else (src - src.half().float()).half()
                assert torch.equal(t[M_run:], ref_rest), (name, M_run)


def test_gemm_rejects_bad_args(cuda_device):
    from multihmr_b200 import ops

    a = torch.zeros(16, 64, device=cuda_device, dtype=torch.float16)
    w = torch.zeros(48, 64, device=cuda_device, dtype=torch.float16)  # N not multiple of 32
    out = torch.zeros(16, 48, device=cuda_device, dtype=torch.float16)
    with pytest.raises(AssertionError):
        ops.gemm_f16(a, w, ops.EPI_BIAS_F16, out, bias=torch.zeros(48, device=cuda_device))
    # a plan runs at most the rows it was built for
    w = torch.zeros(64, 64, device=cuda_device, dtype=torch.float16)
    out = torch.zeros(16, 64, device=cuda_device, dtype=torch.float16)
    with pytest.raises(AssertionError):
        ops.gemm_internal(a, w, ops.EPI_BIAS_F16, 128, out=out, bias=torch.zeros(64, device=cuda_device), m_run=17)


@pytest.mark.parametrize("D,N,Ka,M,gelu", [
    (1024, 4096, 1024, 4097 * 2 + 3, True),    # ViT-L norm2 -> fc1 (CTA pairs on both sides), ragged M
    (1024, 3072, 4096, 2305, False),           # ViT-L fc2 -> next block's norm1 -> qkv
    (768, 2304, 768, 1000, False),             # ViT-B
    (384, 1536, 384, 1370, True),              # ViT-S: single-CTA producer (N = 384), CTA-pair consumer
    (384, 1152, 1536, 257, False),             # ViT-S qkv: single-CTA kernels on both sides
])
def test_folded_layernorm_seam(cuda_device, D, N, Ka, M, gelu):
    """proj / fc2 epilogue emits the raw fp16 rows + row statistics, the next GEMM normalises in its epilogue:
    compared with the unfused fp32 chain (residual update -> LayerNorm -> Linear -> GELU) of the reference block
    (dinov2 layers/block.py), on a stream with a non-zero mean and a few massive channels."""
    from multihmr_b200 import ops

    g = torch.Generator(device="cpu").manual_seed(D + N + M)
    a = torch.randn(M, Ka, generator=g).to(cuda_device).half()
    wp = (torch.randn(D, Ka, generator=g) * (1.0 / Ka ** 0.5)).to(cuda_device).half()
    bp = (torch.randn(D, generator=g) * 0.1).to(cuda_device)
    ls = (torch.rand(D, generator=g) * 0.5 + 0.1).to(cuda_device)
    x0 = torch.randn(M, D, generator=g) * 1.5 + 0.7               # row mean about half a sigma
    x0[:, 5] += 60.0                                              # massive channels (DINOv2-like outliers)
    x0[: M // 3, 77] -= 35.0
    x0 = x0.to(cuda_device)
    ln_g = (torch.rand(D, generator=g) + 0.5).to(cuda_device)
    ln_b = (torch.randn(D, generator=g) * 0.2).to(cuda_device)
    w = (torch.randn(N, D, generator=g) * (1.0 / D ** 0.5)).to(cuda_device)
    b = (torch.randn(N, generator=g) * 0.1).to(cuda_device)

    x = x0.clone()
    out = ops.resid_ln_linear_f16(a, wp, bp, ls, x, ln_g, ln_b, w, b, gelu=gelu)
    x_ref = x0 + ls * (a.float() @ wp.float().t() + bp)
    assert (x - x_ref).abs().max().item() <= 2e-4
    # fp64 reference of the normalised Linear on the reference stream
    xr = x_ref.double()
    y = torch.nn.functional.layer_norm(xr, (D,), ln_g.double(), ln_b.double(), eps=1e-6) @ w.double().t() + b.double()
    if gelu:
        y = torch.nn.functional.gelu(y)
    err = (out.double() - y).abs()
    # what the unfused fp16 path gives on the same data: fp16(LN(x)) @ fp16(W) -- the folded path must be no worse
    # than 1.5x of it (same rounding points: one fp16 rounding per activation and per weight)
    ln16 = torch.nn.functional.layer_norm(x_ref, (D,), ln_g, ln_b, eps=1e-6).half()
    y16 = ln16.float() @ w.half().float().t() + b
    if gelu:
        y16 = torch.nn.functional.gelu(y16)
    err16 = (y16.half().double() - y).abs()
    assert err.max().item() <= 1.5 * err16.max().item() + 1e-3, (err.max().item(), err16.max().item())
    assert err.pow(2).mean().sqrt().item() <= 1.25 * err16.pow(2).mean().sqrt().item() + 1e-5


def test_public_gemm_rejects_internal_epilogues(cuda_device):
    from multihmr_b200 import ops

    a = torch.zeros(128, 64, device=cuda_device, dtype=torch.float16)
    w = torch.zeros(128, 64, device=cuda_device, dtype=torch.float16)
    out = torch.zeros(128, 128, device=cuda_device, dtype=torch.float16)
    with pytest.raises(AssertionError):
        ops.gemm_f16(a, w, 7, out, bias=torch.zeros(128, device=cuda_device), block_n=128)
