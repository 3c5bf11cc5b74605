"""CPU: the C-ABI library builds, loads and exports every symbol include/mhmr.h declares; host logic that
needs no GPU."""
import pytest
import torch


def test_library_exports_every_declared_symbol():
    from multihmr_b200 import _lib

    lib = _lib.load()
    names = _lib.declared_symbols()
    assert len(names) >= 12 and "mhmr_forward" in names and "mhmr_op_gemm_f16" in names
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/mhmr.h but not exported"


def test_create_validates_config_without_gpu():
    from multihmr_b200 import _lib

    lib = _lib.load()
    h = torch.zeros(1, dtype=torch.int64)
    cfg = dict(arch=2, img_size=896, max_batch=1, max_persons=8, xat_depth=2, xat_num_heads=8, num_betas=10,
               person_center_idx=15, num_verts=10475)
    create = lambda **change: lib.mhmr_create(_lib.struct("mhmr_config", **{**cfg, **change}), h)
    assert create(img_size=900) == -2  # 900 % 14 != 0  (model.py:65 "Invalid img size")
    assert b"img size" in lib.mhmr_last_error()
    assert create(arch=5) == -2
    assert create() == 0
    assert lib.mhmr_destroy(h.item()) == 0


def test_model_requires_cuda_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from multihmr_b200.model import Model

    with pytest.raises(RuntimeError, match="no CPU fallback"):
        Model(backbone="dinov2_vits14", img_size=224)


def test_model_constructor_errors_match_reference():
    from multihmr_b200.model import Model

    with pytest.raises(AssertionError, match="Invalid img size"):
        Model(backbone="dinov2_vits14", img_size=225)
    with pytest.raises(NotImplementedError):
        Model(backbone="dinov2_vits14", img_size=224, camera_embedding="learned")


def test_pos_embed_interpolation_matches_oracle():
    from multihmr_b200.model import interpolate_pos_embed
    from oracle import dinov2_ref

    pos = torch.randn(1, 1 + 37 * 37, 64)
    for grid in (16, 37, 48, 64):
        mine = interpolate_pos_embed(pos, grid)
        ref = dinov2_ref.interpolate_pos_encoding(pos, grid * 14, grid * 14)
        assert mine.shape == (1, 1 + grid * grid, 64)
        assert torch.equal(mine, ref)


def test_synth_assets_are_deterministic_and_named_like_the_reference():
    from multihmr_b200 import synth

    a = synth.make_state_dict("dinov2_vits14", 224, seed=3)
    b = synth.make_state_dict("dinov2_vits14", 224, seed=3)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    for k in ("backbone.encoder.blocks.11.mlp.fc2.weight", "mlp_classif.2.bias",
              "x_attention_head.transformer.transformer.layers.1.1.fn.to_kv.weight",
              "x_attention_head.cross_values_y", "x_attention_head.decexpression.bias"):
        assert k in a
    assert a["x_attention_head.transformer.to_token_embedding.weight"].shape == (1024, 318 + 10 + 3 + 384 + 99)
    idx = synth.make_forced_idx(3, 16, [2, 0, 3], seed=1)
    assert idx[0].tolist() == [0, 0, 2, 2, 2]
    flat = (idx[0] * 256 + idx[1] * 16 + idx[2]).tolist()
    assert flat == sorted(flat)  # torch.where order
