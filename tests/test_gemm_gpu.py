"""wgmma GEMM family vs plain torch fp32 on the same fp16-rounded operands (floating-point kernel:
torch fp32 reference, see task ③).  Tolerances are stated per test."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref_linear(a16, w16):
    return a16.float() @ w16.float().t()


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


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("bn", [128, 256, 512])
def test_gemm_bias_f16(cuda_device, M, N, K, bn):
    from multihmr_b200 import ops

    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = (torch.randn(M, K, generator=g) * 1.0).to(cuda_device).half()
    w = (torch.randn(N, K, generator=g) * 0.05).to(cuda_device).half()
    bias = torch.randn(N, generator=g).to(cuda_device)
    out = torch.empty(M, N, device=cuda_device, dtype=torch.float16)
    ops.gemm_f16(a, w, ops.EPI_BIAS_F16, out, bias=bias, block_n=bn)
    ref = _ref_linear(a, w) + bias
    err = (out.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    # fp32 accumulate of exact fp16 products, then one fp16 rounding of the output: 2^-11 relative
    assert err <= 1e-3 * max(scale, 1.0) + 1e-3, (err, scale)


@pytest.mark.parametrize("bn", [256, 512])
@pytest.mark.parametrize("epi", ["gelu", "relu"])
def test_gemm_act_f16(cuda_device, epi, bn):
    from multihmr_b200 import ops

    M, N, K = 1537, 4096, 1024
    g = torch.Generator(device="cpu").manual_seed(5)
    a = torch.randn(M, K, generator=g).to(cuda_device).half()
    w = (torch.randn(N, K, generator=g) * 0.03).to(cuda_device).half()
    bias = torch.randn(N, generator=g).to(cuda_device)
    out = torch.empty(M, N, device=cuda_device, dtype=torch.float16)
    kind = ops.EPI_BIAS_GELU_F16 if epi == "gelu" else ops.EPI_BIAS_RELU_F16
    ops.gemm_f16(a, w, kind, out, bias=bias, block_n=bn)
    pre = _ref_linear(a, w) + bias
    ref = torch.nn.functional.gelu(pre) if epi == "gelu" else torch.relu(pre)
    err = (out.float() - ref).abs().max().item()
    assert err <= 2e-3 * max(ref.abs().max().item(), 1.0), err


@pytest.mark.parametrize("bn", [256, 512])
def test_gemm_layerscale_residual_f32(cuda_device, bn):
    from multihmr_b200 import ops

    M, N, K = 4097 * 2, 1024, 4096
    g = torch.Generator(device="cpu").manual_seed(11)
    a = torch.randn(M, K, generator=g).to(cuda_device).half()
    w = (torch.randn(N, K, generator=g) * 0.02).to(cuda_device).half()
    bias = torch.randn(N, generator=g).to(cuda_device)
    gamma = torch.rand(N, generator=g).to(cuda_device)
    x0 = torch.randn(M, N, generator=g).to(cuda_device)
    x = x0.clone()
    ops.gemm_f16(a, w, ops.EPI_LS_RESID_F32, x, bias=bias, gamma=gamma, block_n=bn)
    ref = x0 + gamma * (_ref_linear(a, w) + bias)
    err = (x - ref).abs().max().item()
    # fp32 everywhere after the exact fp16 products: only summation-order noise
    assert err <= 2e-4, err


def test_gemm_rowadd_remap_f32(cuda_device):
    """Patch-embed shape: rows of image b land at b*T + 1 + n, with a per-n additive table."""
    from multihmr_b200 import ops

    B, Np, D, K = 3, 2304, 384, 592
    T = Np + 1
    g = torch.Generator(device="cpu").manual_seed(13)
    a = torch.randn(B * Np, K, generator=g).to(cuda_device).half()
    w = (torch.randn(D, K, generator=g) * 0.05).to(cuda_device).half()
    table = torch.randn(Np, D, generator=g).to(cuda_device)
    out = torch.full((B * T, D), 7.0, device=cuda_device)
    ops.gemm_f16(a, w, ops.EPI_ROWADD_F32, out, rowadd=table, rows_in=Np, rows_out=T, row_off=1, block_n=128)
    ref = (_ref_linear(a, w).view(B, Np, D) + table).reshape(B, Np, D)
    got = out.view(B, T, D)
    assert torch.all(got[:, 0] == 7.0)  # cls rows untouched
    err = (got[:, 1:] - ref).abs().max().item()
    assert err <= 2e-4, err


@pytest.mark.parametrize("bn", [256, 512])
def test_gemm_bias_f32_nobias(cuda_device, bn):
    from multihmr_b200 import ops

    M, N, K = 2304, 1024, 1152
    g = torch.Generator(device="cpu").manual_seed(17)
    a = torch.randn(M, K, generator=g).to(cuda_device).half()
    w = (torch.randn(N, K, generator=g) * 0.05).to(cuda_device).half()
    out = torch.empty(M, N, device=cuda_device)
    ops.gemm_f16(a, w, ops.EPI_BIAS_F32, out, block_n=bn)
    err = (out - _ref_linear(a, w)).abs().max().item()
    assert err <= 2e-4, err


def test_gemm_rejects_bad_args(cuda_device):
    from multihmr_b200 import ops

    a = torch.zeros(16, 64, device=cuda_device, dtype=torch.float16)
    w = torch.zeros(48, 64, device=cuda_device, dtype=torch.float16)  # N not multiple of 32
    out = torch.zeros(16, 48, device=cuda_device, dtype=torch.float16)
    with pytest.raises(AssertionError):
        ops.gemm_f16(a, w, ops.EPI_BIAS_F16, out, bias=torch.zeros(48, device=cuda_device))


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
    x_ref = x0 + ls * (_ref_linear(a, wp) + bp)
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
