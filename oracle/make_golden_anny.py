"""Pins the Anny oracle (oracle/anny_ref.py) against the reference's OWN multi_hmr_anny/ and writes its goldens.

Runs ONLY in the build container (needs /root/reference).  It imports /root/reference/multi_hmr_anny/multi_hmr.py
UNMODIFIED, with the same third-party shims as oracle/make_golden.py plus two: `anny` (whose full-body model is the
seeded synthetic body model of multihmr_b200.synth) and a DINOv2 hub shim that also returns the cls token.  For each
case it runs the reference and oracle.anny_ref.anny_forward on the same seeded inputs, asserts that they agree
(<= 2e-5 abs, relative above 1) and stores the reference outputs under tests/golden/<case>.npz.

Usage:  python -m oracle.make_golden_anny [case ...]            (from the repo root)
"""
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from multihmr_b200 import synth  # noqa: E402
from oracle import anny_ref, make_golden  # noqa: E402

REFERENCE = make_golden.REFERENCE

# Forced persons are given in training mode (flat dict), natural detections in inference mode (person list sorted by
# depth).  The detection case's scores keep a margin of more than 2e-3 from the 0.3 threshold.
ANNY_CASES = {
    "anny_224_S_forced": dict(backbone="dinov2_vits14", img_size=224, batch=3, persons=[2, 0, 3], seed=21),
    "anny_224_S_detect": dict(backbone="dinov2_vits14", img_size=224, batch=2, persons=None, seed=22, det_bias=-1.5),
    "anny_224_S_noK": dict(backbone="dinov2_vits14", img_size=224, batch=2, persons=[2, 2], seed=23, no_K=True),
    "anny_280_L_forced": dict(backbone="dinov2_vitl14", img_size=280, batch=2, persons=[2, 1], seed=24),
}
ANNY_NUM_VERTS = 1500
ANNY_TRAIN_KEYS = ("scores", "scores_logits", "K", "K_regressed", "fov_regressed", "loc", "offset", "dist",
                   "dist_postprocessed", "shape", "rotvec", "rotmat", "v3d", "j3d", "j2d", "v2d", "transl",
                   "transl_pelvis", "blendshape_coeffs")
ANNY_PERSON_KEYS = ("K", "K_regressed", "loc", "transl", "transl_pelvis", "rotvec", "rotmat", "shape", "v3d", "j3d",
                    "j2d")

_CURRENT = {}


def install_shims():
    make_golden.install_shims()
    torch.hub.load = lambda repo, name, pretrained=False, **kw: anny_ref.HubModelShimWithCls(name)
    anny_ref.install_anny_shim(sys.modules, lambda: _CURRENT["bm"])


def run_anny_case(name, case, out_dir):
    """Anny golden: the reference's Multi_HMR (multi_hmr_anny/multi_hmr.py, unmodified, `anny` shimmed with the
    synthetic body model) vs oracle.anny_ref.anny_forward on identical seeded inputs."""
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count())
    seed = case["seed"]
    sd = synth.make_anny_state_dict(case["backbone"], case["img_size"], seed=seed,
                                    det_bias=case.get("det_bias", -4.0))
    bm = synth.AnnyLikeBodyModel(ANNY_NUM_VERTS, seed)
    _CURRENT["bm"] = bm
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    from multi_hmr_anny.multi_hmr import Multi_HMR  # the reference, unmodified

    model = Multi_HMR(img_size=case["img_size"], backbone=case["backbone"], simple_depth_encoding=1)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all(k.startswith("body_model.") for k in missing), [k for k in missing if not k.startswith("body_model.")]
    model.eval()
    x = synth.make_images(case["batch"], case["img_size"], seed)
    K = None if case.get("no_K") else synth.make_cameras(case["batch"], case["img_size"], jitter=True, seed=seed)
    cfg = anny_ref.AnnyConfig(case["backbone"], case["img_size"])
    gold = {}
    with torch.no_grad():
        if case["persons"] is not None:
            idx = synth.make_forced_idx(case["batch"], case["img_size"] // 14, case["persons"], seed)
            ref = model(x, K=K, idx=idx, is_training=True)
            mine = anny_ref.anny_forward(sd, bm, cfg, x, K, idx=idx, is_training=True)
            keys = list(ANNY_TRAIN_KEYS)
            gold["idx"] = torch.stack(idx[:3])
        else:
            persons = model(x, K=K, det_thresh=0.3, nms_kernel_size=3)
            assert len(persons) >= 4, "too few natural detections: adjust det_bias"
            flat = lambda ps: {k: torch.stack([p[k] for p in ps]) for k in ANNY_PERSON_KEYS}
            ref = flat(persons)
            mine = flat(anny_ref.anny_forward(sd, bm, cfg, x, K, det_thresh=0.3, nms_kernel_size=3))
            keys = list(ANNY_PERSON_KEYS)
            ref["fov"] = persons[0]["fov"]
            mine["fov"] = ref["fov"]
            keys.append("fov")
            # the depth order must differ from the (b, y, x) order somewhere, or the sort is not exercised
            locs = ref["loc"]
            assert any(locs[i + 1, 1] < locs[i, 1] for i in range(len(locs) - 1)), "depth order == raster order"
    for k in keys:
        gold[k] = ref[k]
    worst = 0.0
    for k in keys:
        assert ref[k].shape == mine[k].shape, (k, ref[k].shape, mine[k].shape)
        err = (ref[k].float() - mine[k].float()).abs().max().item()
        worst = max(worst, err)
        assert err <= 2e-5 * max(1.0, ref[k].abs().max().item()), (name, k, err)
    np.savez_compressed(os.path.join(out_dir, name + ".npz"), **{k: v.numpy() for k, v in gold.items()})
    print(f"{name}: reference == oracle (max abs err {worst:.2e}), persons={gold['loc'].shape[0]}, keys={len(keys)}")


def main():
    assert os.path.isdir(REFERENCE), "make_golden_anny needs the reference checkout (build container only)"
    install_shims()
    out_dir = os.path.join(REPO, "tests", "golden")
    only = sys.argv[1:]
    for name, case in ANNY_CASES.items():
        if not only or name in only:
            run_anny_case(name, case, out_dir)


if __name__ == "__main__":
    main()
