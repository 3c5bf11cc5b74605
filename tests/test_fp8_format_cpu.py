"""Number format of the FP8-MLP precision study (tools/precision_study.py --fp8, DESIGN.md §3): e4m3 operands with
power-of-two block scales, one per (row, 128 columns) for activations and one per (128 rows x 128 K) for weights."""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import precision_study as ps  # noqa: E402


def test_scale_is_the_least_power_of_two_that_fits():
    amax = torch.tensor([448.0, 448.0 * 2 ** -7, 449.0, 1.0, 3.0e-5, 100.0, 0.0])
    s = ps.pow2_scale(amax)
    m, _ = torch.frexp(s)
    assert (m == 0.5).all()                                        # exact powers of two
    assert s.tolist()[:2] == [1.0, 2 ** -7]                         # amax = 448 * 2^k needs no headroom
    assert s[2].item() == 2.0 and s[-1].item() == 1.0              # just above 448; all-zero block
    assert ((amax / s)[:-1] <= 448).all() and ((amax / s)[:-1] > 224).all()


def test_activation_blocks_are_scaled_independently():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 384, generator=g)
    x[:, 130] = 300.0                                              # an outlier channel in the second block
    x[3, 256:] = 0.0                                               # an all-zero block
    q = ps.q8_act(x)
    for blk in range(3):
        sl = slice(blk * 128, (blk + 1) * 128)
        s = ps.pow2_scale(x[:, sl].abs().amax(-1, keepdim=True))
        ref = (x[:, sl] / s).to(torch.float8_e4m3fn).to(torch.float32) * s
        assert torch.equal(q[:, sl], ref)
    assert torch.equal(q[3, 256:], torch.zeros(128))
    # the outlier coarsens only its own block: the first block keeps e4m3's relative error (2^-4), or half the
    # subnormal step 2^-9 of its own scale
    s0 = ps.pow2_scale(x[:, :128].abs().amax(-1, keepdim=True))
    assert ((q[:, :128] - x[:, :128]).abs() <= torch.maximum(x[:, :128].abs() * 2 ** -4, s0 * 2 ** -10)).all()
    assert torch.equal(ps.q8_act(q), q)                            # dequantised values quantise to themselves


def test_weight_scale_covers_a_128_by_128_block_with_a_ragged_row_tail():
    g = torch.Generator().manual_seed(1)
    w = torch.randn(200, 256, generator=g) * 0.02
    w[5, 200] = 4.0                                                # raises block (0, 1) only
    q = ps.q8_w(w)
    assert q.shape == w.shape
    for r0, r1 in ((0, 128), (128, 200)):
        for k0 in (0, 128):
            blk = w[r0:r1, k0:k0 + 128]
            s = ps.pow2_scale(blk.abs().amax())
            ref = (blk / s).to(torch.float8_e4m3fn).to(torch.float32) * s
            assert torch.equal(q[r0:r1, k0:k0 + 128], ref), (r0, k0)
    # the neighbouring block's scale would be a different rounding of the same weights
    s_nb = ps.pow2_scale(w[0:128, 128:256].abs().amax())
    wrong = (w[0:128, :128] / s_nb).to(torch.float8_e4m3fn).to(torch.float32) * s_nb
    assert not torch.equal(q[0:128, :128], wrong)
