"""wgmma flash attention (attn_tc.cu) against softmax(q k^T / 8) v in fp64 on the same fp16 q, k, v, per element.

The bound of every comparison is fp64_util.attn_head_ref (derived in its docstring from the kernel's rounding points,
and checked against a CPU emulation of them in test_attention_tolerance_cpu.py).  Needle keys at the tile edges make
an off-by-one in the key mask fall far outside it; sentinel canvases and NaN pads catch stores and loads outside the
[B*T, D] / [B*T, 3D] views; the batch tests hold each image to its own rows bit for bit."""
import pytest
import torch

from fp64_util import SENTINEL16, _report, attn_head_ref, needle_positions, needle_qkv

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _ref(qkv, B, T, D):
    """(o, tol) fp64 [B*T, D] on qkv's device."""
    o = torch.empty(B * T, D, dtype=torch.float64, device=qkv.device)
    tol = torch.empty_like(o)
    x = qkv.view(B, T, 3, D)
    for b in range(B):
        for h in range(D // 64):
            c = slice(h * 64, (h + 1) * 64)
            o[b * T:(b + 1) * T, c], tol[b * T:(b + 1) * T, c] = attn_head_ref(x[b, :, 0, c], x[b, :, 1, c],
                                                                              x[b, :, 2, c])
    return o, tol


@pytest.mark.parametrize("B,T,D,scale", [
    (1, 128, 64, 1.0),      # one full tile
    (1, 1, 64, 1.0),        # single token
    (1, 130, 128, 1.0),     # ragged tail of 2
    (2, 257, 384, 1.0),     # ViT-S heads, tail of 1, two images (224 px)
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
    (2, 401, 768, 1.0),     # ViT-B (12 heads) at 280 px: narrow last tile of 17 keys
    (2, 1025, 768, 1.0),    # ViT-B at 448 px
    (2, 1025, 1024, 1.0),   # ViT-L at 448 px
    (4, 2305, 1024, 1.0),   # ViT-L at 672 px, the batch of the 672 px workload
    (1, 8465, 1024, 1.0),   # ViT-L at 1288 px: 67 key tiles, last one 17 keys
])
def test_attention_matches_fp32(cuda_device, B, T, D, scale):
    from multihmr_b200 import ops

    g = _gen(B * 1000 + T + D)
    qkv = (torch.randn(B * T, 3 * D, generator=g) * scale).to(cuda_device).half()
    out = ops.attention(qkv, B, T, D)
    ref, tol = _ref(qkv, B, T, D)
    err = (out.double() - ref).abs()
    # per element: fp16 P in PV (dominant), fp32 S / exp2 / O / l, one fp16 output rounding (attn_head_ref)
    _report(f"attention B={B} T={T} D={D} scale={scale}", err, tol)
    assert torch.all(err <= tol)


# (last-tile width, key tiles): widths 1..32 take the narrow attn_fwd_kernel<32> path when there are >= 2 tiles,
# 33 is the first that does not; the tile counts give odd and even numbers of query tiles
NEEDLE_CASES = [(1, 2), (16, 3), (17, 5), (31, 2), (32, 3), (32, 2), (33, 2), (64, 5), (127, 3), (128, 2),
                (1, 5), (17, 1), (128, 1), (33, 3)]


@pytest.mark.parametrize("width,n_kv", NEEDLE_CASES)
def test_attention_needles(cuda_device, width, n_kv):
    """Needle keys at 0, 127, 128, T-2 and T-1, each holding > 0.9 of its query's mass, and one at row 0 of the
    next image that must get no weight.  A kernel that drops key T-1 (the narrow path run one key short included)
    or admits key T falls outside the bound."""
    from multihmr_b200 import ops

    T = 128 * (n_kv - 1) + width
    B, D = 2, 128
    qkv = needle_qkv(B, T, D, _gen(width * 10 + n_kv)).to(cuda_device).half()
    out = ops.attention(qkv, B, T, D)
    ref, tol = _ref(qkv, B, T, D)
    err = (out.double() - ref).abs()
    _report(f"attention needles T={T} (width {width}, {n_kv} tiles)", err, tol)
    assert torch.all(err <= tol)
    # the needles hold their queries' mass (the property the sensitivity rests on)
    x = qkv.view(B, T, 3, D).double()
    s = x[0, :, 0, :64] @ x[0, :, 1, :64].t() / 8.0
    w = torch.softmax(s, dim=1)
    pos = needle_positions(T)
    assert all(w[p, p] > 0.9 for p in pos)
    # sensitivity, image 0 head 0: key T-1 dropped; key T (row 0 of image 1, aligned with query T-1) admitted
    got = out[:T, :64].double()
    t0 = tol[:T, :64]
    if T > 1:
        drop, _ = attn_head_ref(x[0, :, 0, :64], x[0, :T - 1, 1, :64], x[0, :T - 1, 2, :64])
        assert torch.any((got - drop).abs() > t0)
    flat = qkv.view(B * T, 3, D)
    admit, _ = attn_head_ref(x[0, :, 0, :64], flat[:T + 1, 1, :64], flat[:T + 1, 2, :64])
    assert torch.any((got - admit).abs() > t0)


def test_attention_guard_bands_and_pitches(cuda_device):
    """out with ldo = D + 64 inside a sentinel canvas, qkv with ld_qkv = 3D + 64 and NaN in the pad columns: the
    result equals the contiguous call bit for bit and nothing outside [B*T, D] is written."""
    from multihmr_b200 import ops

    dev = cuda_device
    B, T, D = 3, 401, 384
    qkv = torch.randn(B * T, 3 * D, generator=_gen(41)).to(dev).half()
    want = ops.attention(qkv, B, T, D)
    big = torch.full((B * T, 3 * D + 64), float("nan"), dtype=torch.float16, device=dev)
    big[:, :3 * D] = qkv
    canvas = torch.full((B * T + 3, D + 64), SENTINEL16, dtype=torch.float16, device=dev)
    ops.attention(big[:, :3 * D], B, T, D, out=canvas[:B * T, :D])
    assert torch.equal(canvas[:B * T, :D], want)
    assert torch.all(canvas[:B * T, D:] == SENTINEL16) and torch.all(canvas[B * T:] == SENTINEL16)
    # determinism: the same call twice
    assert torch.equal(ops.attention(qkv, B, T, D), want)


@pytest.mark.parametrize("width", [1, 17, 33, 128])
def test_attention_batch_independence(cuda_device, width):
    """Each image of a batch of 3 equals the same image run alone (the last one reads past the end of the buffer,
    which TMA zero-fills), and permuting the images permutes the outputs, bit for bit."""
    from multihmr_b200 import ops

    dev = cuda_device
    B, D = 3, 128
    T = 256 + width
    qkv = torch.randn(B * T, 3 * D, generator=_gen(width)).to(dev).half()
    out = ops.attention(qkv, B, T, D)
    for b in range(B):
        alone = ops.attention(qkv[b * T:(b + 1) * T].clone(), 1, T, D)
        assert torch.equal(out[b * T:(b + 1) * T], alone), b
    perm = [2, 0, 1]
    qp = qkv.view(B, T, 3 * D)[perm].reshape(B * T, 3 * D)
    op = ops.attention(qp, B, T, D)
    assert torch.equal(op.view(B, T, D), out.view(B, T, D)[perm])


@pytest.mark.parametrize("width", [1, 17, 33, 128])
def test_attention_nonfinite_neighbour(cuda_device, width):
    """±inf and NaN in image 1's K and V leave images 0 and 2 bit for bit unchanged: softmax attention is per image,
    so whatever image 1 holds must not reach the other images through the last, partly masked key tile."""
    from multihmr_b200 import ops

    dev = cuda_device
    B, D = 3, 128
    T = 128 + width
    qkv = torch.randn(B * T, 3 * D, generator=_gen(100 + width)).to(dev).half()
    want = ops.attention(qkv, B, T, D)
    bad = qkv.clone()
    img1 = bad[T:2 * T]
    img1[0::3, D:] = float("inf")
    img1[1::3, D:] = -float("inf")
    img1[2::3, D:] = float("nan")
    got = ops.attention(bad, B, T, D)
    for b in (0, 2):
        rows = slice(b * T, (b + 1) * T)
        assert torch.equal(got[rows], want[rows]), (b, got[rows].isnan().sum().item())


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
