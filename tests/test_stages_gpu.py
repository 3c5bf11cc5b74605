"""Stage-level GPU parity: SMPL-X layer vs the oracle (the backbone features: test_vit_bulk_gpu.py)."""
import pytest
import torch

import parity_util as pu

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("P", [1, 5, 8, 9, 23])
def test_smplx_layer_vs_oracle(cuda_device, P):
    """fp32 kernel vs fp32 oracle: tight tolerance (summation order only)."""
    from multihmr_b200 import synth
    from oracle import multihmr_ref, smplx_ref

    case, sd, bm, x, K, _ = pu.build_inputs("s_224_S_forced")
    m = pu.build_engine(case, sd, bm, max_persons=32)
    g = torch.Generator().manual_seed(P)
    rotvec = torch.randn(P, 53, 3, generator=g) * 0.4
    rotvec[0, 0] = 0.0                      # exercises the small-angle branch of the root rotation
    shape, expr = torch.randn(P, 10, generator=g), torch.randn(P, 10, generator=g) * 0.5
    loc = torch.rand(P, 2, generator=g) * 200 + 10
    dist = torch.rand(P, 1, generator=g) * 5 + 1.5
    Kd = synth.make_cameras(P, 224, jitter=True, seed=P)
    ref = multihmr_ref.smpl_layer_forward(smplx_ref.SMPLXShim(bm, 10), rotvec, shape, loc, dist, Kd, expr, 15)
    out = m.smplx(rotvec, shape, loc, dist[:, 0], Kd, expr)
    for k, tol in (("v3d", 2e-5), ("j3d", 2e-5), ("transl", 1e-5), ("transl_pelvis", 2e-5)):
        err = (out[k].cpu() - ref[k]).abs().max().item()
        assert err <= tol, (k, err)
    for k, src in (("j2d", "j3d"), ("v2d", "v3d")):
        err = (out[k].cpu() - ref[k]).abs().max().item()
        assert err <= pu.projection_tolerance(ref[src], float(Kd[:, 0, 0].max()), tol3d=2e-5), (k, err)


def test_smplx_shape_asserts_like_reference(cuda_device):
    case, sd, bm, x, K, _ = pu.build_inputs("s_224_S_forced")
    m = pu.build_engine(case, sd, bm)
    with pytest.raises(AssertionError):     # blocks/smpl_layer.py:67
        m.smplx(torch.zeros(1, 24, 3), torch.zeros(1, 10), torch.zeros(1, 2), torch.ones(1), torch.eye(3)[None],
                torch.zeros(1, 10))
