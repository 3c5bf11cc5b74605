"""GPU parity proper: the engine (sm_90a kernels behind the C-ABI) vs the golden fixtures = outputs of
the unmodified reference `Model.forward` on identical seeded inputs.  Tolerance: 1e-3 abs on detection
scores, SMPL-X parameters and 3-D vertices (BASELINE.json north_star); see parity_util.TOL."""
import pytest
import torch

import parity_util as pu

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["s_224_S_forced", "s_448_B_forced", "c1_672_S_forced", "s_224_S_asymK",
                                  "s_280_L_forced", "s_224_S_outliers"])
def test_forced_idx_matches_reference(cuda_device, name):
    case, sd, bm, x, K, idx = pu.build_inputs(name)
    gold = pu.load_golden(name)
    m = pu.build_engine(case, sd, bm)
    out = m(x, idx=idx, K=K, is_training=True)
    bad = pu.compare(out, gold, [k for k in gold if k != "idx"], focal=float(K[:, 0, 0].max()), verbose=True)
    assert not bad, bad


def test_natural_detection_matches_reference(cuda_device):
    name = "s_224_S_detect"
    case, sd, bm, x, K, _ = pu.build_inputs(name)
    gold = pu.load_golden(name)
    m = pu.build_engine(case, sd, bm)
    persons = m(x, K=K, det_thresh=0.3, nms_kernel_size=3)
    assert len(persons) == gold["scores"].shape[0]
    assert set(persons[0]) == {"scores", "loc", "transl", "transl_pelvis", "rotvec", "expression", "shape", "v3d",
                               "j3d", "j2d"}                                         # model.py:329-347
    got = {k: torch.stack([p[k] for p in persons]) for k in gold}
    bad = pu.compare(got, gold, list(gold), focal=float(K[:, 0, 0].max()), verbose=True)
    assert not bad, bad


def test_no_detection_returns_empty_list(cuda_device):
    case, sd, bm, x, K, _ = pu.build_inputs("s_224_S_detect")
    m = pu.build_engine(case, sd, bm)
    assert m(x, K=K, det_thresh=0.999, nms_kernel_size=3) == []                      # model.py:241-243


def test_detection_set_and_order_vs_oracle(cuda_device):
    """Many natural detections: same cells in torch.where order, except cells within 1e-3 of the threshold
    or of a 3x3 tie (score discontinuities, SURVEY.md §7)."""
    from multihmr_b200 import synth
    from oracle import dinov2_ref, multihmr_ref

    backbone, S, B = "dinov2_vits14", 224, 3
    sd = synth.make_state_dict(backbone, S, seed=11, det_bias=-1.0)
    bm = synth.make_body_model(11)
    x, K = synth.make_images(B, S, 11), synth.make_cameras(B, S, seed=11)
    m = pu.build_engine(dict(backbone=backbone, img_size=S, batch=B), sd, bm, max_persons=256)
    t, P = m.forward_raw(x, K, det_thresh=0.3, nms_kernel_size=3)
    with torch.no_grad():
        z = dinov2_ref.get_intermediate_layers(x, sd, backbone, "backbone.encoder.")
        s_raw, _, _ = multihmr_ref.detection(z, sd, 1, 0.3, None, False)            # no NMS: raw scores
        s_nms, _, idx = multihmr_ref.detection(z, sd, 3, 0.3, None, False)
    ref_cells = set(zip(idx[0].tolist(), idx[1].tolist(), idx[2].tolist()))
    got = t["det_idx"][:, :P].cpu()
    got_list = list(zip(got[0].tolist(), got[1].tolist(), got[2].tolist()))
    assert got_list == sorted(got_list), "persons must come in (b, y, x) order"
    s_raw = s_raw[..., 0]
    ambiguous = set()
    pooled = torch.nn.functional.max_pool2d(s_raw[:, None], 3, 1, 1)[:, 0]
    second = (pooled - s_raw).abs()
    for b, y, xx in ref_cells.symmetric_difference(got_list):
        near_thr = abs(s_raw[b, y, xx].item() - 0.3) < 1e-3
        near_tie = second[b, y, xx].item() < 1e-3
        assert near_thr or near_tie, ("detection differs away from a discontinuity", (b, y, xx))
        ambiguous.add((b, y, xx))
    assert P >= 5 and len(ambiguous) <= max(2, P // 10)
    err = (t["scores_map"].cpu() - s_nms[..., 0]).abs()
    assert (err > 1e-3).sum().item() <= 2 * len(ambiguous) + 2  # NMS flips only at ambiguous cells


def test_capacity_overflow_is_an_error_not_a_truncation(cuda_device):
    from multihmr_b200 import _lib, synth

    backbone, S = "dinov2_vits14", 224
    sd = synth.make_state_dict(backbone, S, seed=11, det_bias=2.0)  # nearly every NMS maximum fires
    m = pu.build_engine(dict(backbone=backbone, img_size=S, batch=1), sd, synth.make_body_model(11), max_persons=4)
    with pytest.raises(_lib.MhmrError, match="max_persons"):
        m(synth.make_images(1, S, 11), K=synth.make_cameras(1, S, seed=11), det_thresh=0.3, nms_kernel_size=3)


def test_batch_invariance_and_smaller_batches(cuda_device):
    """Images are independent units (SURVEY.md §8e): running images one by one gives the same persons."""
    case, sd, bm, x, K, idx = pu.build_inputs("s_224_S_forced")
    m = pu.build_engine(case, sd, bm)
    full = m(x, idx=idx, K=K, is_training=True)
    b_idx = idx[0]
    for b in range(case["batch"]):
        sel = b_idx == b
        if sel.sum() == 0:
            continue
        sub = tuple(t[sel] if i else torch.zeros_like(t[sel]) for i, t in enumerate(idx))
        one = m(x[b:b + 1], idx=sub, K=K[b:b + 1], is_training=True)
        for k in ("v3d", "rotmat", "shape", "dist", "loc"):
            assert (one[k] - full[k][sel.to(full[k].device)]).abs().max().item() <= 1e-4, k


def test_forward_is_bit_reproducible(cuda_device):
    """No atomics on the data path: the same inputs give the same bits run after run, like the reference on CPU."""
    case, sd, bm, x, K, idx = pu.build_inputs("s_224_S_forced")
    m = pu.build_engine(case, sd, bm)
    a = {k: v.clone() for k, v in m(x, idx=idx, K=K, is_training=True).items()}
    for _ in range(3):
        b = m(x, idx=idx, K=K, is_training=True)
        for k in ("scores", "v3d", "rotmat", "shape", "dist", "loc", "j2d"):
            assert torch.equal(a[k], b[k]), k


def _oracle_cpu(sd, bm, backbone, S, x, K, num_betas=10, **kw):
    from oracle import multihmr_ref, smplx_ref

    cfg = multihmr_ref.RefConfig(backbone=backbone, img_size=S, num_betas=num_betas)
    with torch.no_grad():
        return multihmr_ref.model_forward(sd, smplx_ref.SMPLXShim(bm, num_betas), cfg, x, K, **kw)


def test_num_betas_11_layer(cuda_device):
    """Model(num_betas=11) uses the 'neutral_11' SMPL-X layer (model.py:104-110, :319): 11 shape components."""
    from multihmr_b200 import synth
    from multihmr_b200.model import Model

    backbone, S, B, seed = "dinov2_vits14", 224, 2, 31
    sd = synth.make_state_dict(backbone, S, num_betas=11, seed=seed)
    bm = synth.make_body_model(seed)
    x, K = synth.make_images(B, S, seed), synth.make_cameras(B, S, jitter=True, seed=seed)
    idx = synth.make_forced_idx(B, S // 14, [2, 1], seed)
    ref = _oracle_cpu(sd, bm, backbone, S, x, K, num_betas=11, idx=idx, is_training=True)
    m = Model(backbone=backbone, img_size=S, num_betas=11, max_batch=B, max_persons=8, body_model=bm)
    m.load_state_dict(sd)
    out = m(x, idx=idx, K=K, is_training=True)
    assert out["shape"].shape == (3, 11)
    bad = pu.compare(out, {k: v.float() for k, v in ref.items()},
                     ["shape", "rotmat", "expression", "dist", "v3d", "j3d", "transl"], verbose=True)
    assert not bad, bad


def test_forced_persons_sharing_a_cell(cuda_device):
    """Two forced persons on the same cell (b, y, x): the reference adds the learned values to that context cell with a
    non-accumulating index_put (model.py:517), so the cell holds ctx + v once, not ctx + 2v."""
    from multihmr_b200 import synth
    from multihmr_b200.model import Model

    backbone, S, B, seed = "dinov2_vits14", 224, 2, 43
    sd = synth.make_state_dict(backbone, S, seed=seed)
    # value embeddings 5x their synthetic scale: adding them once or twice at the shared cell then moves every person
    # output of image 1 by 3.5e-3 (dist) to 1.5e-2 (v3d), well outside the 1e-3 tolerance (checked below)
    h = "x_attention_head."
    for n in ("cross_values_x", "cross_values_y"):
        sd[h + n] = 5.0 * sd[h + n]
    bm = synth.make_body_model(seed)
    x, K = synth.make_images(B, S, seed), synth.make_cameras(B, S, jitter=True, seed=seed)
    t = lambda v: torch.tensor(v, dtype=torch.int64)
    idx = (t([0, 0, 1, 1]), t([3, 10, 5, 5]), t([4, 2, 7, 7]), t([0, 0, 0, 0]))  # image 1: both persons on (5, 7)
    keys = ["rotmat", "shape", "expression", "dist", "v3d", "j3d", "transl"]
    ref = _oracle_cpu(sd, bm, backbone, S, x, K, idx=idx, is_training=True)
    # sensitivity: image 1 holds only the shared cell, so doubling the value tables is ctx + 2v there
    sd2 = dict(sd)
    for n in ("cross_values_x", "cross_values_y"):
        sd2[h + n] = 2.0 * sd[h + n]
    twice = _oracle_cpu(sd2, bm, backbone, S, x, K, idx=idx, is_training=True)
    caught = pu.compare({k: twice[k][2:] for k in keys}, {k: ref[k][2:] for k in keys}, keys)
    assert [k for k, _, _ in caught] == keys, caught
    m = Model(backbone=backbone, img_size=S, max_batch=B, max_persons=8, body_model=bm)
    m.load_state_dict(sd)
    out = m(x, idx=idx, K=K, is_training=True)
    bad = pu.compare(out, {k: v.float() for k, v in ref.items()}, keys, verbose=True)
    assert not bad, bad


def test_nms_off_threshold_list_and_partial_batch(cuda_device):
    """nms_kernel_size=1 (forward_model's default, demo.py:110), det_thresh given as a list
    (model.py:614-615), and a batch smaller than max_batch."""
    from multihmr_b200 import synth

    backbone, S, seed = "dinov2_vits14", 224, 11
    sd = synth.make_state_dict(backbone, S, seed=seed, det_bias=-1.0)
    bm = synth.make_body_model(seed)
    x, K = synth.make_images(2, S, seed), synth.make_cameras(2, S, seed=seed)
    m = pu.build_engine(dict(backbone=backbone, img_size=S, batch=4), sd, bm, max_batch=4, max_persons=256)
    persons = m(x, K=K, det_thresh=[0.3], nms_kernel_size=1)
    ref = _oracle_cpu(sd, bm, backbone, S, x, K, det_thresh=[0.3], nms_kernel_size=1)
    assert len(ref) > 0, "workload must produce detections"
    s_ref = torch.stack([p["scores"] for p in ref])
    near = ((s_ref - 0.3).abs() < 1e-3).sum().item()
    assert abs(len(persons) - len(ref)) <= near
    if len(persons) == len(ref):
        got = {k: torch.stack([p[k] for p in persons]) for k in ("scores", "loc", "v3d", "transl")}
        want = {k: torch.stack([p[k] for p in ref]) for k in got}
        assert not pu.compare(got, want, list(got), verbose=True)


def test_refinement_lowers_the_error_on_vit_l(cuda_device):
    """The fp32 refinement of the detected tokens' streams (DESIGN.md §3) must beat the bulk fp16 pass on the
    ViT-L golden case by a wide margin (CPU emulation, tools/precision_study.py: 1.08e-3 -> 2.3e-4 on v3d)."""
    name = "s_280_L_forced"
    case, sd, bm, x, K, idx = pu.build_inputs(name)
    gold = pu.load_golden(name)
    err = {}
    for refine in (False, True):
        m = pu.build_engine(case, sd, bm, refine_central=refine)
        out = m(x, idx=idx, K=K, is_training=True)
        err[refine] = {k: (out[k].cpu() - gold[k]).abs().max().item() for k in ("v3d", "rotmat", "shape", "dist")}
        print("refine" if refine else "bulk  ", {k: f"{v:.3e}" for k, v in err[refine].items()})
    # max-norm of one case: the ratio moves with the rounding realisation of the bulk pass (0.27 ... 0.66 between
    # builds whose CPU emulation, tools/ln_fold_study.py, has the same rms error); rotmat is the steadier indicator
    assert err[True]["v3d"] < err[False]["v3d"] and err[True]["rotmat"] < 0.6 * err[False]["rotmat"]
    assert err[True]["v3d"] < 5e-4 and err[True]["rotmat"] < 2.5e-4


def test_forced_idx_validation_and_unsorted_order(cuda_device):
    """Out-of-range idx raises IndexError like the reference's tensor indexing (model.py:246-255); persons given
    in a non image-sorted order come back in the caller's order."""
    case, sd, bm, x, K, idx = pu.build_inputs("s_224_S_forced")
    m = pu.build_engine(case, sd, bm)
    ref = m(x, idx=idx, K=K, is_training=True)
    ref = {k: v.clone() for k, v in ref.items()}
    P = idx[0].shape[0]
    perm = torch.tensor([P - 1 - i for i in range(P)])
    shuffled = tuple(t[perm] for t in idx)
    out = m(x, idx=shuffled, K=K, is_training=True)
    for k in ("v3d", "rotmat", "shape", "loc", "dist", "transl"):
        assert (out[k] - ref[k][perm.to(ref[k].device)]).abs().max().item() <= 1e-4, k
    bad = tuple(t.clone() for t in idx)
    bad[1][0] = case["img_size"] // 14  # one row beyond the token grid
    with pytest.raises(IndexError):
        m(x, idx=bad, K=K, is_training=True)
    bad = tuple(t.clone() for t in idx)
    bad[0][0] = case["batch"]
    with pytest.raises(IndexError):
        m(x, idx=bad, K=K, is_training=True)


def test_head_stage_vs_oracle_on_engine_features(cuda_device):
    """Stage-level parity of detection + HPH + post-processing: the oracle's head evaluated on the ENGINE's own
    backbone features (bulk pass, refinement off) must reproduce the engine's head outputs tightly — a decoder
    bug cannot hide behind the end-to-end tolerance."""
    import torch.nn.functional as F
    from oracle import multihmr_ref

    name = "s_448_B_forced"
    case, sd, bm, x, K, idx = pu.build_inputs(name)
    m = pu.build_engine(case, sd, bm, refine_central=False)
    t, P = m.forward_raw(x, K, idx=idx, want_z=True, want_v2d=True)
    z = t["z"].cpu()
    cfg = multihmr_ref.RefConfig(backbone=case["backbone"], img_size=case["img_size"])
    B, N, D = z.shape
    w = int(N ** 0.5)
    with torch.no_grad():
        scores, _, _ = multihmr_ref.detection(z, sd, 3, 0.3, idx, True)
        b_idx, y_idx, x_idx = idx[0], idx[1], idx[2]
        zc = z[b_idx, y_idx * w + x_idx]
        offset = multihmr_ref.regression_mlp(zc, sd, "mlp_offset")
        z_K = multihmr_ref.embed_camera(K, w, w, cfg)
        zc = torch.cat([zc, z_K[b_idx, y_idx, x_idx]], 1)
        z_all = torch.cat([z, z_K.reshape(B, N, -1)], 2)
        rotmat, shape, expr, cam = multihmr_ref.hph_forward(zc, z_all, idx, sd, cfg, F.linear, None)
    got = {"scores": t["scores_map"].cpu()[..., None], "offset": t["offset"][:P].cpu(), "rotmat": t["rotmat"][:P].cpu(),
           "shape": t["shape"][:P].cpu(), "expression": t["expression"][:P].cpu(), "dist_pp": t["dist_pp"][:P].cpu()}
    want = {"scores": scores, "offset": offset, "rotmat": rotmat, "shape": shape, "expression": expr,
            "dist_pp": cam[:, 0]}
    # only the two token-side GEMMs (detection hidden layer, to_kv) use fp16 operands; everything else is fp32
    tol = {"scores": 3e-4, "offset": 5e-5, "rotmat": 1e-4, "shape": 1e-4, "expression": 1e-4, "dist_pp": 1e-4}
    for k in got:
        e = (got[k] - want[k]).abs().max().item()
        print(f"  head stage {k:12s} err {e:.3e} (tol {tol[k]:.0e})")
        assert e <= tol[k], (k, e)


def test_separate_layernorm_path_stays_green(cuda_device):
    """`MHMR_LN_FOLD=0` (fp32 residual stream + LayerNorm kernels: the A/B side of DESIGN.md §5 "LayerNorm folded into
    the GEMMs") must keep matching the reference goldens; the switch is read once per engine, so a child process."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = r'''
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import parity_util as pu
for name in ("s_224_S_forced", "s_280_L_forced"):
    case, sd, bm, x, K, idx = pu.build_inputs(name)
    gold = pu.load_golden(name)
    m = pu.build_engine(case, sd, bm)
    out = m(x, idx=idx, K=K, is_training=True)
    bad = pu.compare(out, gold, [k for k in gold if k != "idx"], focal=float(K[:, 0, 0].max()))
    assert not bad, (name, bad)
    assert m.last_launch_count() > 0
print("separate-LN ok")
''' % (root, os.path.join(root, "tests"))
    env = dict(os.environ, MHMR_LN_FOLD="0")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "separate-LN ok" in r.stdout, (r.stdout[-1000:], r.stderr[-2000:])
