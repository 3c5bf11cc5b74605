"""wgmma flash attention vs torch fp32 softmax attention on the same fp16-rounded q, k, v."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(qkv, B, T, D):
    H = D // 64
    q, k, v = qkv.float().view(B, T, 3, H, 64).permute(2, 0, 3, 1, 4)
    o = torch.nn.functional.scaled_dot_product_attention(q, k, v)
    return o.transpose(1, 2).reshape(B * T, D)


@pytest.mark.parametrize("B,T,D,scale", [
    (1, 128, 64, 1.0),      # one full tile
    (1, 1, 64, 1.0),        # single token
    (1, 130, 128, 1.0),     # ragged tail of 2
    (2, 257, 384, 1.0),     # ViT-S heads, tail of 1, two images
    (1, 2305, 384, 1.0),    # 672 / 14 grid + cls (ViT-S)
    (2, 4097, 1024, 1.0),   # 896 / 14 grid + cls (ViT-L)
    (1, 1000, 128, 4.0),    # peaky softmax: exercises the lazy-rescale path
    (1, 128 + 17, 64, 1.0), # tail of 17 keys: two 16-column groups, one 32-column chunk
    (1, 256 + 40, 64, 1.0), # tail of 40 keys: 48 columns, two chunks
    (1, 384 + 100, 64, 1.0),# tail of 100 keys: 112 columns, four chunks
    (1, 33, 64, 1.0),       # one short tile, query warps 2..3 have no rows
    (1, 130, 64, 1.0),      # second query tile with 2 rows: three of its warps only keep the protocol alive
    (3, 600, 128, 1.0),     # odd number of query tiles: the last CTA of an image holds a single tile
    (1, 2 * 128 + 1, 64, 8.0),  # peaky softmax across three key tiles + single-row last query tile
    (1, 2 * 256 + 17, 128, 1.0),  # 17 query rows beyond the last full pair of query tiles
    (3, 513, 64, 1.0),      # one query row beyond two full pairs, three images
])
def test_attention_matches_fp32(cuda_device, B, T, D, scale):
    from multihmr_b200 import ops

    g = torch.Generator(device="cpu").manual_seed(B * 1000 + T + D)
    qkv = (torch.randn(B * T, 3 * D, generator=g) * scale).to(cuda_device).half()
    out = ops.attention(qkv, B, T, D)
    ref = _ref(qkv, B, T, D)
    err = (out.float() - ref).abs().max().item()
    # P is rounded to fp16 (2^-11 relative) before the PV product and the output is fp16
    tol = 4e-3 * max(ref.abs().max().item(), 1.0)
    assert err <= tol, (err, tol)


def test_attention_images_independent(cuda_device):
    """Rows of image 1 must not leak into image 0 (the last KV tile of an image crosses into the next)."""
    from multihmr_b200 import ops

    g = torch.Generator(device="cpu").manual_seed(3)
    B, T, D = 2, 200, 128
    qkv = torch.randn(B * T, 3 * D, generator=g).to(cuda_device).half()
    out_a = ops.attention(qkv, B, T, D)
    qkv2 = qkv.clone()
    qkv2[T:] = 1e4  # poison image 1 with huge finite values
    out_b = ops.attention(qkv2, B, T, D)
    assert torch.equal(out_a[:T], out_b[:T])

