"""CPU emulation of the folded-LayerNorm bulk pass vs the separate-LayerNorm bulk pass (DESIGN.md §5).

Both variants round where the engine rounds (fp16 operands / workspaces, fp32 accumulate and residual); the script
reports (a) the row statistics of the residual stream that decide how much the fold costs (|mean| / sigma),
(b) the error of the bulk features and (c) of the fp32-refined rows fed with each bulk pass's attention outputs.
DIAGNOSTIC TOOL, never on the product path.   python tools/ln_fold_study.py [case]
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import parity_util as pu  # noqa: E402
from oracle import dinov2_ref  # noqa: E402

EPS = 1e-6


def r16(t):
    """fp16 rounding of t, kept in t's dtype (the study runs in fp32 on the CPU and in fp64 in the tests)"""
    return t.to(torch.float16).to(t.dtype)


def split16(t):
    """two-term fp16 representation (hi + lo) of the residual stream in the folded engine"""
    hi = r16(t)
    return hi + r16(t - hi)


def ln_linear(x, g, b, w, bias, mode, shift=None, qa=None, qw=None):
    """Linear(LayerNorm(x)) with the engine's rounding points.  mode: 'exact' | 'sep' | 'fold' | 'fold_shift'.
    qa / qw round the folded GEMM's operands (fp16 by default: r16 as it is when called)."""
    D = x.shape[-1]
    qa, qw = qa or r16, qw or r16
    if mode == "exact":
        return F.linear(F.layer_norm(x, (D,), g, b, EPS), w, bias)
    if mode == "sep":
        return F.linear(r16(F.layer_norm(x, (D,), g, b, EPS)), r16(w), bias)
    wf = w * g
    wf = qw(wf - wf.mean(1, keepdim=True))   # W' = W diag(gamma) with centred rows, rounded
    b2 = bias + w @ b
    mean = x.mean(-1, keepdim=True)
    var = (x * x).mean(-1, keepdim=True) - mean * mean
    rstd = torch.rsqrt(var.clamp_min(0) + EPS)
    if mode == "fold":
        return rstd * F.linear(qa(x), wf) + b2
    # fold_shift: the fp16 copy holds x - shift (shift = the row mean one residual update earlier)
    return rstd * F.linear(r16(x - shift), wf) + b2


def attention(q, k, v):
    s = torch.matmul(q, k.transpose(-1, -2)) * (q.shape[-1] ** -0.5)
    m = s.amax(dim=-1, keepdim=True)
    p = torch.exp(s - m)
    return torch.matmul(r16(p), v) / p.sum(dim=-1, keepdim=True)


def forward(x_img, sd, name, pre, mode, o_in=None, mlp8=None, keep_cls=False, attn=None, taps=None):
    """mode 'sep' / 'fold' / 'fold_shift': bulk pass, returns (z, [O16 per layer], stats).  mode 'refine': fp32
    stream fed with the given attention outputs.  mlp8 = (fc1 A, fc1 W, fc2 A, fc2 W): the 'fold' bulk pass rounds
    the operands of fc1 (raw stream, folded W') and fc2 (GELU output, W2) with these functions instead of fp16
    (tools/precision_study.py --fp8).
    keep_cls: z keeps the final-normed cls row in front.  attn: attention(q, k, v) in place of `attention` (the same
    arithmetic in another loop order).  taps: {layers: None} is filled with the residual stream [B, T, D] after the
    patch embedding (layers = 0) and after each listed number of blocks."""
    cfg = dinov2_ref.ARCHS[name]
    H = cfg["num_heads"]
    if mode == "refine" or mode == "exact":
        x = dinov2_ref.prepare_tokens(x_img, sd, pre)
    else:
        w = sd[pre + "patch_embed.proj.weight"]
        xp = F.conv2d(r16(x_img), r16(w), sd[pre + "patch_embed.proj.bias"], stride=14).flatten(2).transpose(1, 2)
        x = torch.cat((sd[pre + "cls_token"].expand(x_img.shape[0], -1, -1), xp), 1)
        x = x + dinov2_ref.interpolate_pos_encoding(sd[pre + "pos_embed"], x_img.shape[-1], x_img.shape[-2])
    B, T, D = x.shape
    outs, ratios = [], []
    if mode.startswith("fold"):
        x = split16(x)
    if taps is not None and 0 in taps:
        taps[0] = x
    shift = x.mean(-1, keepdim=True)
    for i in range(cfg["depth"]):
        p = f"{pre}blocks.{i}."
        if mode in ("refine",):
            o = o_in[i]
        else:
            ratios.append((x.mean(-1).abs() / x.std(-1)).max().item())
            lm = "exact" if mode == "exact" else mode
            qkv = ln_linear(x, sd[p + "norm1.weight"], sd[p + "norm1.bias"], sd[p + "attn.qkv.weight"],
                            sd[p + "attn.qkv.bias"], lm, shift)
            if mode != "exact":
                qkv = r16(qkv)
            qkv = qkv.reshape(B, T, 3, H, D // H).permute(2, 0, 3, 1, 4)
            if mode == "exact":
                o = F.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2])
            else:
                o = r16((attn or attention)(qkv[0], qkv[1], qkv[2]))
            o = o.transpose(1, 2).reshape(B, T, D)
            outs.append(o)
        full = mode in ("refine", "exact")
        wp = sd[p + "attn.proj.weight"]
        shift = x.mean(-1, keepdim=True)
        x = x + sd[p + "ls1.gamma"] * F.linear(o, wp if full else r16(wp), sd[p + "attn.proj.bias"])
        if mode.startswith("fold"):
            x = split16(x)
        qa1, qw1, qa2, qw2 = (None, None, r16, r16) if mlp8 is None else mlp8
        h = ln_linear(x, sd[p + "norm2.weight"], sd[p + "norm2.bias"], sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"],
                      "exact" if full else mode, shift, qa1, qw1)
        h = F.gelu(h)
        w2 = sd[p + "mlp.fc2.weight"]
        shift = x.mean(-1, keepdim=True)
        x = x + sd[p + "ls2.gamma"] * F.linear(h if full else qa2(h), w2 if full else qw2(w2), sd[p + "mlp.fc2.bias"])
        if mode.startswith("fold"):
            x = split16(x)
        if taps is not None and i + 1 in taps:
            taps[i + 1] = x
    z = F.layer_norm(x, (D,), sd[pre + "norm.weight"], sd[pre + "norm.bias"], EPS)
    z = z if keep_cls else z[:, 1:]
    return z, outs, ratios


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "s_280_L_forced"
    torch.set_num_threads(min(16, os.cpu_count()))
    case, sd, bm, x, K, idx = pu.build_inputs(name)
    pre = "backbone.encoder."
    with torch.no_grad():
        z_ref, _, ratios = forward(x, sd, case["backbone"], pre, "exact")
        print("max over rows of |mean|/sigma of the residual stream, per layer (entering norm1):")
        print("  ", " ".join(f"{r:.2f}" for r in ratios))
        for mode in ("sep", "fold", "fold_shift"):
            z, outs, _ = forward(x, sd, case["backbone"], pre, mode)
            zr, _, _ = forward(x, sd, case["backbone"], pre, "refine", o_in=outs)
            e_b = (z - z_ref)
            e_r = (zr - z_ref)
            print(f"{mode:11s} bulk z: max {e_b.abs().max():.3e} rms {e_b.pow(2).mean().sqrt():.3e} | refined rows: max "
                  f"{e_r.abs().max():.3e} rms {e_r.pow(2).mean().sqrt():.3e}")


if __name__ == "__main__":
    main()
