"""CPU: the Anny variant's oracle restatement against the goldens of the unmodified reference, the synthetic Anny
assets, and the validation of the Anny engine configuration."""
import ctypes

import pytest
import torch

import anny_util as au


@pytest.mark.parametrize("name", sorted(au.CASES))
def test_oracle_restatement_matches_anny_goldens(name):
    case, sd, bm, x, K, idx = au.build_inputs(name)
    gold = au.load_golden(name)
    with torch.no_grad():
        out = au.oracle(case, sd, bm, x, K, idx)
    if idx is None:
        out = au.flatten_persons(out)
    for k in gold:
        if k == "idx":
            continue
        err = (out[k].float() - gold[k].float()).abs().max().item()
        assert err <= 2e-5 * max(1.0, gold[k].abs().max().item()), (k, err)


def test_oracle_rejects_even_nms_and_returns_tuple_without_detections():
    from oracle import anny_ref

    case, sd, bm, x, K, _ = au.build_inputs("anny_224_S_detect")
    with pytest.raises(ValueError):
        au.oracle(case, sd, bm, x, K, None, nms_kernel_size=4)
    with torch.no_grad():
        assert au.oracle(case, sd, bm, x, K, None, det_thresh=1.01) == ({}, [])
    assert anny_ref.nms_pad(3) == 1 and anny_ref.nms_pad(5) == 2


def test_synth_anny_assets_are_deterministic_and_named_like_the_reference():
    from multihmr_b200 import synth

    a = synth.make_anny_state_dict("dinov2_vits14", 224, xat_depth=2, seed=3)
    b = synth.make_anny_state_dict("dinov2_vits14", 224, xat_depth=2, seed=3)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    # Multi_HMR.state_dict() names (multi_hmr_anny/multi_hmr.py:46-95, encoder.py:21-31, hph.py:114-131)
    for k in ("encoder.backbone.blocks.11.mlp.fc2.weight", "encoder.backbone.norm.bias", "encoder.mlp_det.2.bias",
              "encoder.mlp_fov_unique.0.weight", "encoder.fov_max", "dec_to_token.weight",
              "decoder.transformer.layers.1.1.fn.to_kv.weight", "decoder.transformer.layers.1.2.fn.net.3.bias",
              "mlp_offset.2.bias", "mlp_dist.0.weight", "useful_rotmat", "init_body_pose", "eye"):
        assert k in a, k
    assert a["dec_pos_emb"].shape == (256, 512)
    assert a["mlp_pose.0.weight"].shape == (512, 512 + 163 * 6) and a["mlp_shape.2.weight"].shape == (11, 512)
    assert a["useful_rotmat"].shape == (1, 163) and a["init_body_pose"].shape == (1, 163 * 6)
    bm1, bm2 = synth.AnnyLikeBodyModel(300, seed=1), synth.AnnyLikeBodyModel(300, seed=1)
    assert len(bm1.bone_labels) == 163 and bm1.bone_labels.index("head") == synth.ANNY_HEAD_BONE
    pose = torch.eye(4).repeat(2, 163, 1, 1)
    pheno = {k: torch.full((2,), 0.3) for k in bm1.SHAPE_KEYS}
    o1, o2 = bm1(pose_parameters=pose, phenotype_kwargs=pheno), bm2(pose_parameters=pose, phenotype_kwargs=pheno)
    assert torch.equal(o1["vertices"], o2["vertices"]) and o1["bone_poses"].shape == (2, 163, 4, 4)


def test_sincos_table_layout():
    """Row n = y * grid + x; first half of the channels from the row index, second half from the column index."""
    from multihmr_b200 import synth

    t = synth.sincos_pos_embed_2d(16, 5)
    n = 2 * 5 + 3
    w = 1.0 / 10000 ** (torch.arange(4, dtype=torch.float64) / 4)
    want = torch.cat([torch.sin(2 * w), torch.cos(2 * w), torch.sin(3 * w), torch.cos(3 * w)]).float()
    assert torch.allclose(t[n], want)


def test_create_validates_anny_config_without_gpu():
    from multihmr_b200 import _lib
    from multihmr_b200.model import _Config

    lib = _lib.load()
    h = ctypes.c_void_p()

    def rc(*fields):
        return lib.mhmr_create(ctypes.byref(_Config(*fields)), ctypes.byref(h))

    base = [0, 224, 2, 8, 8, 16, 11, 9, 0, 1]
    assert rc(*base, 1, 500, 2048, 163) == -2                         # xat_dim not a multiple of 32
    assert rc(*base, 1, 512, 0, 163) == -2                            # no FeedForward width
    assert rc(*base, 2, 512, 2048, 163) == -2                         # unknown head kind
    assert rc(*base[:7], 163, 0, 1, 1, 512, 2048, 163) == -2          # centre bone out of range
    assert b"person_center" in lib.mhmr_last_error()
    assert rc(*base, 1, 512, 2048, 163) == 0
    assert lib.mhmr_destroy(h) == 0
