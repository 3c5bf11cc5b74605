"""GPU parity of the Anny variant: the engine (sm_90a kernels behind mhmr_forward_anny / mhmr_anny_place) vs the
goldens of the unmodified reference Multi_HMR and vs the oracle restatement at full size."""
import argparse
import math
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


def test_forced_idx_validation(cuda_device):
    """Forced persons are checked before anything is enqueued: an index outside the batch or the token grid raises
    IndexError, persons not grouped by image raise ValueError, more persons than max_persons raise MhmrError."""
    from multihmr_b200 import _lib

    case, sd, bm, x, K, idx = au.build_inputs("anny_224_S_forced")
    m = au.build_engine(case, sd, bm, max_persons=8)
    for row, value in ((0, case["batch"]), (1, case["img_size"] // 14), (2, -1)):
        bad = tuple(t.clone() for t in idx)
        bad[row][0] = value
        with pytest.raises(IndexError):
            m(x, K=K, idx=bad, is_training=True)
    P = idx[0].shape[0]
    perm = torch.tensor([P - 1 - i for i in range(P)])
    with pytest.raises(ValueError, match="contiguously"):
        m(x, K=K, idx=tuple(t[perm] for t in idx), is_training=True)
    crowd = tuple(torch.cat([t] * 2) for t in idx)   # 10 persons, still grouped by image
    crowd = tuple(t[torch.argsort(crowd[0], stable=True)] for t in crowd)
    with pytest.raises(_lib.MhmrError, match="max_persons"):
        m(x, K=K, idx=crowd, is_training=True)


def _anny_head_reference(z, sd, idx, K, depth, heads, fp16_context=True):
    """The Anny head of oracle/anny_ref.py (hph, _mlp and the post-processing of anny_forward) in fp64 on the engine's
    final-normed features z [B, N, D], rounded to fp16 where the engine rounds (engine.cu, Anny setup):
      * context tokens: fp16(fp16(z) . fp16(W_dt)^T + fp32(b_dt + dec_pos_emb))   (EPI_ROWADD_F16 GEMM on ctx16)
      * keys / values of every layer: fp16(context) . fp16(W_kv)^T, fp32 out     (the to_kv GEMM)
      * the query side (dec_to_token of the person's own fp32 row, HPH, regressors, post-processing): fp32.
    What is left between the two is the order of the fp32 sums (and a rare fp16 rounding tie of a context value)."""
    from oracle import anny_ref, roma_ref

    d = {k: v.double() for k, v in sd.items()}
    B, N, D = z.shape
    w = int(round(N ** 0.5))
    dim = d["dec_to_token.weight"].shape[0]
    pos = d["dec_pos_emb"].reshape(N, dim)
    rowadd = (sd["dec_pos_emb"].float().reshape(N, dim) + sd["dec_to_token.bias"].float()).double()
    if fp16_context:
        ctx = (z.half().double() @ sd["dec_to_token.weight"].half().double().t() + rowadd).half().double()
        for l in range(depth):
            key = f"decoder.transformer.layers.{l}.1.fn.to_kv.weight"
            d[key] = sd[key].half().double()
    else:
        ctx = z.double() @ d["dec_to_token.weight"].t() + d["dec_to_token.bias"] + pos
    zq = z.double()
    b_idx, y_idx, x_idx = (i.long() for i in idx[:3])
    q_all = zq[b_idx, y_idx * w + x_idx] @ d["dec_to_token.weight"].t() + d["dec_to_token.bias"] + pos[y_idx * w + x_idx]
    ys = []
    for b in torch.unique(b_idx, sorted=True).tolist():
        sel = b_idx == b
        ys.append(anny_ref.hph(q_all[sel], ctx[b], d, depth, heads))
    y = torch.cat(ys, 0)
    offset = anny_ref._mlp(y, d, "mlp_offset")
    loc = (torch.stack([x_idx, y_idx], 1).double() + 0.5 + offset) * 14
    Kp = K.double()[b_idx]
    dist_pp = anny_ref._mlp(y, d, "mlp_dist")
    dist = Kp[:, 0, 0].unsqueeze(1) / torch.clamp(torch.exp(dist_pp), 1e-5)
    transl = torch.einsum("pij,pj->pi", torch.inverse(Kp), torch.cat([loc, torch.ones_like(loc[:, :1])], 1)) * dist
    init = d["init_body_pose"]
    J = init.shape[1] // 6
    shape = torch.sigmoid(anny_ref._mlp(y, d, "mlp_shape"))
    rot6d = anny_ref._mlp(torch.cat([y, init.repeat(y.shape[0], 1)], 1), d, "mlp_pose") + init
    rotmat = roma_ref.special_gramschmidt(rot6d.reshape(-1, 3, 2)).view(-1, J, 3, 3)
    u = d["useful_rotmat"].reshape(1, -1, 1, 1)
    rotmat = u * rotmat + (1 - u) * torch.eye(3, dtype=torch.float64, device=rotmat.device).reshape(1, 1, 3, 3)
    rotvec = roma_ref.rotmat_to_rotvec(rotmat)
    return {"offset": offset, "dist_pp": dist_pp[:, 0], "shape": shape, "rotmat": rotmat, "rotvec": rotvec, "loc": loc,
            "transl": transl}


@pytest.mark.parametrize("name", ["anny_224_S_forced", "anny_280_L_forced"])
def test_anny_head_stage_vs_oracle_on_engine_features(cuda_device, name):
    """Stage-level parity of the Anny head (dec_to_token GEMM with its fp16 row-add epilogue, anny_gather, the 8-layer
    16-head HPH, the stacked regressors, anny_person_post): the oracle's head evaluated in fp64 on the ENGINE's own
    backbone features (bulk pass, refinement off, K given) must reproduce the engine's outputs tightly, so a head bug
    cannot hide behind the end-to-end tolerance.  anny_224_S_forced has an image with no person."""
    from oracle import anny_ref, roma_ref

    case, sd, bm, x, K, idx = au.build_inputs(name)
    m = au.build_engine(case, sd, bm, refine_central=False)
    t, P = m.forward_raw(x, K, idx=idx, want_z=True)
    torch.cuda.synchronize()
    assert P == sum(case["persons"])
    cfg = anny_ref.AnnyConfig(case["backbone"], case["img_size"])
    with torch.no_grad():
        want = _anny_head_reference(t["z"].cpu(), sd, idx, K, cfg.xat_depth, cfg.xat_heads)
        plain = _anny_head_reference(t["z"].cpu(), sd, idx, K, cfg.xat_depth, cfg.xat_heads, fp16_context=False)
    got = {"offset": t["offset"][:P], "dist_pp": t["dist_pp"][:P], "shape": t["shape"][:P], "rotmat": t["rotmat"][:P],
           "rotvec": t["rotvec"][:P], "loc": t["loc"][:P], "transl": t["transl"][:P]}
    got = {k: v.cpu().double() for k, v in got.items()}
    # What remains is fp32 summation order through 8 layers (order 1e-6 on values of order 1) and the rare fp16 rounding
    # tie of a context value.  The tolerances are set against the 6e-6 .. 8e-4 by which the outputs move when the context
    # is NOT rounded to fp16 (checked below), so a rounding point missing on either side is caught.  loc is 14 * offset;
    # transl scales with the distance, so it is compared relative to its norm; rotvec within 1e-3 of pi is compared as
    # a rotation.
    tol = {"offset": 1e-5, "dist_pp": 5e-6, "shape": 1e-5, "rotmat": 1e-5, "rotvec": 1e-5, "loc": 1.4e-4, "transl": 1e-5}

    def err(a, ref, k):
        if k == "transl":
            return ((a - ref[k]).norm(dim=-1) / ref[k].norm(dim=-1)).max().item()
        if k == "rotvec":
            near_pi = (math.pi - ref[k].norm(dim=-1)) < 1e-3
            d = (a - ref[k]).abs().amax(dim=-1)
            d_pi = (roma_ref.rotvec_to_rotmat(a) - ref["rotmat"]).abs().amax(dim=(-1, -2))
            return torch.where(near_pi, d_pi, d).max().item()
        return (a - ref[k]).abs().max().item()

    worst_plain = 0.0
    for k in tol:
        e, e_plain = err(got[k], want, k), err(got[k], plain, k)
        worst_plain = max(worst_plain, e_plain / tol[k])
        print(f"  anny head stage {k:8s} err {e:.3e} (tol {tol[k]:.0e}); vs an fp32-context reference {e_plain:.3e}")
        assert e <= tol[k], (k, e)
    # sensitivity: the reference without the engine's fp16 context rounding falls outside the tolerances
    assert worst_plain > 1.0, worst_plain
