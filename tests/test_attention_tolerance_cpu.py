"""The per-element bound of the attention tests (fp64_util.attn_head_ref), checked without a GPU: a torch emulation of
the kernel's rounding points (attn_tc.cu) must land inside it, and references with one plausible mistake outside it.

Emulated: 128-key tiles, S in fp32, the exp2 argument s * scale_log2 - m rounded once (the fma), exp2 in fp32, the
running max and alpha rescale of O and l, l summed over the fp32 p, P rounded to fp16 before PV, O accumulated in
fp32, the output rounded to fp16."""
import math

import pytest
import torch

from fp64_util import _report, attn_head_ref, needle_positions, needle_qkv

SCALE_LOG2 = torch.tensor(0.125 * 1.4426950408889634, dtype=torch.float32)


def emulate(q16, k16, v16, T):
    """The kernel on one head of one image: q16 [Tq, 64], k16 / v16 [>= T, 64] fp16 (rows >= T are never used)."""
    q = q16.float()
    Tq = q.shape[0]
    n_kv = (T + 127) // 128
    m = torch.full((Tq, 1), -math.inf)
    l = torch.zeros(Tq, 1)
    o = torch.zeros(Tq, 64)
    c = SCALE_LOG2
    for j in range(n_kv):
        kt = torch.zeros(128, 64)
        vt = torch.zeros(128, 64)
        n = min(128, T - 128 * j)
        kt[:n] = k16[128 * j:128 * j + n].float()
        vt[:n] = v16[128 * j:128 * j + n].float()
        s = q @ kt.t()
        s[:, n:] = -math.inf
        m_new = torch.maximum(m, s.amax(1, keepdim=True) * c)
        alpha = torch.exp2(m - m_new)
        p = torch.exp2((s.double() * c.double() - m_new.double()).float())  # one fma rounding, then exp2
        l = l * alpha + p.sum(1, keepdim=True)
        o = o * alpha + p.half().float() @ vt
        m = m_new
    return (o * (1.0 / l)).half()


def _heads(qkv, B, T, D, b, h):
    x = qkv[b * T:(b + 1) * T].view(T, 3, D)
    return x[:, 0, h * 64:(h + 1) * 64], x[:, 1, h * 64:(h + 1) * 64], x[:, 2, h * 64:(h + 1) * 64]


@pytest.mark.parametrize("T,scale", [(1, 1.0), (17, 1.0), (128, 1.0), (129, 1.0), (300, 4.0), (401, 1.0),
                                     (2 * 128 + 32, 8.0), (513, 1.0)])
def test_emulation_inside_bound(T, scale):
    g = torch.Generator().manual_seed(T)
    D = 128
    qkv = (torch.randn(T, 3 * D, generator=g) * scale).half()
    worst = 0.0
    for h in range(D // 64):
        q, k, v = _heads(qkv, 1, T, D, 0, h)
        ref, tol = attn_head_ref(q, k, v)
        err = (emulate(q, k, v, T).double() - ref).abs()
        worst = max(worst, _report(f"emulation T={T} scale={scale} head {h}", err, tol))
        assert torch.all(err <= tol)
    # a bound that the emulated rounding does not come near would catch nothing (T = 1 is exact: o = v)
    assert worst > 1e-2 or T == 1, worst


@pytest.mark.parametrize("T", [129, 128 + 17, 2 * 128 + 32, 2 * 128 + 33, 4 * 128 + 127])
def test_needles_separate_right_and_wrong_references(T):
    g = torch.Generator().manual_seed(T + 1)
    B, D = 2, 64
    qkv = needle_qkv(B, T, D, g).half()
    q, k, v = _heads(qkv, B, T, D, 0, 0)
    emu = emulate(q, k, v, T).double()
    ref, tol = attn_head_ref(q, k, v)
    _report(f"needles T={T}", (emu - ref).abs(), tol)
    assert torch.all((emu - ref).abs() <= tol)
    # each needle holds > 0.9 of its query's softmax mass
    s = q.double() @ k.double().t() / 8.0
    w = torch.softmax(s, dim=1)
    for p in needle_positions(T):
        assert w[p, p] > 0.9, (p, w[p, p].item())
    # key T - 1 dropped / key T (row 0 of the next image, same direction as key T - 1) admitted
    drop, _ = attn_head_ref(q, k[:T - 1], v[:T - 1])
    kn = qkv[:T + 1].view(T + 1, 3, D)
    admit, _ = attn_head_ref(q, kn[:, 1], kn[:, 2])
    for wrong in (drop, admit):
        assert torch.any((emu - wrong).abs() > tol)
