"""GPU parity of the Anny variant: the engine (sm_90a kernels behind mhmr_forward_anny / mhmr_anny_place) vs the
goldens of the unmodified reference Multi_HMR and vs the oracle restatement at full size."""
import argparse
import os

import pytest
import torch

import anny_util as au
import parity_util as pu

pytestmark = pytest.mark.gpu

TRAIN_KEYS = ("scores", "offset", "dist", "dist_postprocessed", "shape", "rotmat", "rotvec", "transl", "transl_pelvis",
              "v3d", "j3d", "loc", "j2d", "v2d", "fov_regressed")


def _compare(got, gold, keys, focal):
    tol = dict(pu.TOL, fov_regressed=1e-3, fov=1e-3)
    for k in keys:
        g, r = got[k].detach().float().cpu(), gold[k].float()
        assert g.shape == r.shape, (k, tuple(g.shape), tuple(r.shape))
    special = ("fov_regressed", "fov", "K_regressed")
    bad = pu.compare(got, gold, [k for k in keys if k not in special], focal=focal, verbose=True)
    for k in keys:
        if k in ("fov_regressed", "fov"):
            e = (got[k].float().cpu() - gold[k].float()).abs().max().item()
            print(f"  {k:20s} err={e:.3e} tol={tol[k]:.1e}")
            if e > tol[k]:
                bad.append((k, e, tol[k]))
    for k in ("K_regressed",):
        if k in gold:
            rel = ((got[k].float().cpu() - gold[k].float()).abs() / gold[k].float().abs().clamp_min(1.0)).max().item()
            print(f"  {k:20s} rel={rel:.3e} tol=1.0e-03")
            if rel > 1e-3:
                bad.append((k, rel, 1e-3))
    return bad


def _focal(out):
    return float(out["K"][..., 0, 0].max())


@pytest.mark.parametrize("name", ["anny_224_S_forced", "anny_224_S_noK", "anny_280_L_forced"])
def test_forced_training_mode_matches_reference(cuda_device, name):
    case, sd, bm, x, K, idx = au.build_inputs(name)
    gold = au.load_golden(name)
    m = au.build_engine(case, sd, bm)
    out = m(x, K=K, idx=idx, is_training=True)
    assert out["feat"].shape == (case["batch"], case["img_size"] // 14, case["img_size"] // 14, sd["encoder.backbone.norm.bias"].numel())
    bad = _compare(out, gold, list(TRAIN_KEYS) + ["K_regressed"], _focal(gold))
    assert not bad, bad


def test_natural_detection_inference_mode_and_depth_order(cuda_device):
    name = "anny_224_S_detect"
    case, sd, bm, x, K, _ = au.build_inputs(name)
    gold = au.load_golden(name)
    m = au.build_engine(case, sd, bm)
    persons = m(x, K=K, det_thresh=0.3, nms_kernel_size=3)
    assert isinstance(persons, list) and len(persons) == gold["loc"].shape[0]
    assert set(persons[0]) == {"K", "K_regressed", "loc", "transl", "transl_pelvis", "rotvec", "rotmat", "shape",
                               "v3d", "j3d", "j2d", "fov"}
    z = [float(p["transl"][2]) for p in persons]
    assert z == sorted(z)
    got = au.flatten_persons(persons)
    bad = _compare(got, gold, ["loc", "transl", "transl_pelvis", "rotvec", "rotmat", "shape", "v3d", "j3d", "j2d",
                               "fov", "K_regressed"], _focal(gold))
    assert not bad, bad


def test_fullsize_672_L_against_oracle_on_gpu(cuda_device):
    """multiHMR_672_L_anny geometry, batch 4, forced persons [2, 1, 3, 2]: engine vs the fp32 oracle on this GPU."""
    from multihmr_b200 import synth

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    S, B, seed = 672, 4, 41
    case = dict(backbone="dinov2_vitl14", img_size=S, batch=B, persons=[2, 1, 3, 2])
    sd = synth.make_anny_state_dict("dinov2_vitl14", S, seed=seed)
    bm = synth.AnnyLikeBodyModel(14000, seed)
    x, K = synth.make_images(B, S, seed), synth.make_cameras(B, S, jitter=True, seed=seed)
    idx = synth.make_forced_idx(B, S // 14, case["persons"], seed)
    m = au.build_engine(case, sd, bm.to(cuda_device), max_persons=16)
    out = m(x, K=K, idx=idx, is_training=True)
    dev = cuda_device
    with torch.no_grad():
        ref = au.oracle(case, {k: v.to(dev) for k, v in sd.items()}, bm, x.to(dev), K.to(dev),
                        tuple(i.to(dev) for i in idx))
    ref = {k: v.cpu() for k, v in ref.items()}
    bad = _compare(out, ref, list(TRAIN_KEYS) + ["K_regressed"], _focal(ref))
    pve_mm = (out["v3d"].cpu() - ref["v3d"]).norm(dim=-1).mean().item() * 1000
    print(f"  PVE {pve_mm:.4f} mm")
    assert pve_mm < 1.0
    assert not bad, bad


def test_load_model_on_a_reference_checkpoint(cuda_device, tmp_path, monkeypatch):
    from multihmr_b200 import api

    name = "anny_224_S_forced"
    case, sd, bm, x, K, idx = au.build_inputs(name)
    args = argparse.Namespace(img_size=[case["img_size"]], backbone=case["backbone"], xat_depth=8, xat_heads=16,
                              xat_dim=512, xat_mlp_dim=2048, num_betas=11, simple_depth_encoding=1,
                              pretrained_backbone=False, person_center="head")
    os.makedirs(tmp_path / "models" / "multiHMR")
    torch.save({"args": args, "model_state_dict": sd}, tmp_path / "models" / "multiHMR" / "multiHMR_224_S_anny.pt")
    monkeypatch.chdir(tmp_path)
    m = api.load_model("multiHMR_224_S_anny", device=cuda_device, max_batch=3, body_model=bm)
    out = m(x, K=K, idx=idx, is_training=True)
    bad = _compare(out, au.load_golden(name), list(TRAIN_KEYS), float(K[:, 0, 0].max()))
    assert not bad, bad
    persons = api.forward_model(m, x[:1], K[:1], det_thresh=0.0001, nms_kernel_size=3)
    assert isinstance(persons, list) and len(persons) > 0


def test_no_detection_even_nms_and_bulk_path(cuda_device):
    name = "anny_224_S_forced"
    case, sd, bm, x, K, idx = au.build_inputs(name)
    m = au.build_engine(case, sd, bm)
    assert m(x, K=K, det_thresh=1.01, nms_kernel_size=3) == ({}, [])          # multi_hmr.py:123-124
    with pytest.raises(ValueError):
        m(x, K=K, nms_kernel_size=4)
    gold = au.load_golden(name)
    bulk = au.build_engine(case, sd, bm, refine_central=False)
    out = bulk(x, K=K, idx=idx, is_training=True)
    err = {k: (out[k].cpu() - gold[k]).abs().max().item() for k in ("v3d", "rotmat", "shape", "fov_regressed")}
    print("bulk fp16 path", {k: f"{v:.3e}" for k, v in err.items()})
    assert all(torch.isfinite(out[k]).all() for k in ("v3d", "rotmat", "shape"))
    assert err["v3d"] < 1e-2
