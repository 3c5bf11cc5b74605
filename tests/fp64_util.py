"""Shared pieces of the kernel tests that compare against plain fp64 references: sentinels for guard bands, fp16 /
fp32 rounding units, the tensor-core accumulation and erf-GELU error bounds, and the worst err/tol report."""
import torch

U = 2.0 ** -24  # unit roundoff of fp32
SENTINEL = 12345.0
SENTINEL16 = -1234.0  # exact in fp16


def _report(name, err, tol):
    r = (err / tol).max().item() if err.numel() else 0.0
    print(f"  {name}: worst err/tol {r:.3f} (max err {err.max().item() if err.numel() else 0.0:.2e})")
    return r


def _ulp16(v):
    """fp16 ulp of |v| (subnormal spacing 2^-24 below 2^-14)."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def _acc_tol(a, w):
    """fp32 tensor-core accumulation of exact fp16 products: one fp32 accumulation per 16-deep k step, each within
    2 u of the running sum, plus the alignment inside a step: (K/4 + 16) u sum|a w| covers both with margin."""
    K = a.shape[1]
    return (K / 4 + 16) * U * (a.abs() @ w.abs().t())


def _gelu_tol(y):
    # Abramowitz-Stegun erf (|error| <= 1.5e-7) and ~8 fp32 operations on the way
    return 0.5 * y.abs() * (1.5e-7 + 8 * U) + 4 * U * y.abs()


def attn_head_ref(q, k, v, n_kv=None, chunk=1024):
    """softmax(q k^T / 8) v of one head in fp64 (q [Tq, 64], k and v [Tk, 64]; any float dtype, promoted), and the
    per-element bound of the flash-attention kernel (attn_tc.cu) against it.  With w_j the exact softmax weights and
    n_kv the number of 128-key tiles the kernel runs:

      * P is rounded to fp16 before the PV product while l sums the fp32 p: 2^-11 sum_j w_j |v_jd| (relative fp16
        rounding), plus 2^-25 sum_j |v_jd| for p in the fp16 subnormal range (absolute half spacing; p <= 1 at the
        running max and l >= 1, and a later rescale by alpha <= 1 only shrinks it).  The dominant term.
      * S = q.k in fp32 on the tensor cores (the _acc_tol of K = 64: 32 u sum_k |q_k k_jk|), scaled by the rounded
        scale_log2 and shifted by the running max in one fma, then ex2.approx.ftz (<= 8 u relative).  In the exp2
        domain times ln 2 these give p_j a relative error eps_j = 4 u sum_k |q_k k_jk| + 2 u (s_max - s_j) / 8 + 8 u;
        the error of the max itself is common to every p and cancels in o = sum p v / sum p.  A relative error in
        p_j moves o_d by w_j eps_j (|v_jd| + |o_d|).
      * O accumulates the fp16 products exactly in fp32 over T keys (depth T/16 k-steps, bound (T/4 + 16) u as
        _acc_tol) with up to n_kv rescales by alpha (one rounding each, alpha itself is shared with l and cancels);
        l sums 32 values per lane per tile plus one add per tile and 2 quad levels, then 1/l and O / l: together
        (T/4 + 16 + 4 n_kv + 40) u sum_j w_j |v_jd|.
      * One fp16 rounding of the output: half an fp16 ulp.

    Returns (o, tol), fp64 [Tq, 64]."""
    q, k, v = q.double(), k.double(), v.double()
    Tk = k.shape[0]
    if n_kv is None:
        n_kv = (Tk + 127) // 128
    va = v.abs()
    floor = 2.0 ** -25 * va.sum(0, keepdim=True)
    lin = 2.0 ** -11 + (Tk / 4 + 16 + 4 * n_kv + 40) * U
    os, tols = [], []
    for i0 in range(0, q.shape[0], chunk):
        qi = q[i0:i0 + chunk]
        s = qi @ k.t()
        w = torch.softmax(s / 8.0, dim=1)
        o = w @ v
        eps = 4 * U * (qi.abs() @ k.abs().t()) + 2 * U * (s.amax(1, keepdim=True) - s) / 8.0 + 8 * U
        we = w * eps
        t = lin * (w @ va) + we @ va + we.sum(1, keepdim=True) * o.abs() + floor
        os.append(o)
        tols.append(t + 0.5 * _ulp16(o.abs() + t))
    return torch.cat(os), torch.cat(tols)


def needle_positions(T):
    return sorted({p for p in (0, 127, 128, T - 2, T - 1) if 0 <= p < T})


def needle_qkv(B, T, D, g):
    """fp32 [B*T, 3D] q | k | v (heads of 64) with needle keys: for the i-th position p of needle_positions(T),
    key p and query p of every head and image are 4 on dims 8i .. 8i+7 and 0 elsewhere, so q_p . k_p / 8 = 16 and
    the needle holds > 0.99 of query p's softmax mass (other scores are ~0.4 at T = 8465).  Row 0 of every image
    after the first also carries the last needle's direction: a kernel that admits key T of image b gives it the
    same score as key T - 1."""
    qkv = torch.randn(B * T, 3 * D, generator=g) * 0.3
    qkv[:, 2 * D:] = torch.randn(B * T, D, generator=g)
    pos = needle_positions(T)
    last = len(pos) - 1
    for b in range(B):
        for h in range(D // 64):
            for i, p in enumerate(pos):
                r = b * T + p
                for c0 in (h * 64, D + h * 64):
                    qkv[r, c0:c0 + 64] = 0.0
                    qkv[r, c0 + 8 * i:c0 + 8 * i + 8] = 4.0
            if b > 0:
                c0 = D + h * 64
                qkv[b * T, c0 + 8 * last:c0 + 8 * last + 8] = 4.0
    return qkv
