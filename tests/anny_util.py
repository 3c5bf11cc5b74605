"""Shared helpers of the Anny tests: the seeded cases of oracle/make_golden_anny.py::ANNY_CASES, their goldens (outputs of
the unmodified reference Multi_HMR), the oracle restatement and the engine."""
import os

import numpy as np
import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NUM_VERTS = 1500

# Must stay in sync with oracle/make_golden_anny.py::ANNY_CASES (the fixture generator).
CASES = {
    "anny_224_S_forced": dict(backbone="dinov2_vits14", img_size=224, batch=3, persons=[2, 0, 3], seed=21),
    "anny_224_S_detect": dict(backbone="dinov2_vits14", img_size=224, batch=2, persons=None, seed=22, det_bias=-1.5),
    "anny_224_S_noK": dict(backbone="dinov2_vits14", img_size=224, batch=2, persons=[2, 2], seed=23, no_K=True),
    "anny_280_L_forced": dict(backbone="dinov2_vitl14", img_size=280, batch=2, persons=[2, 1], seed=24),
}
PERSON_KEYS = ("K", "K_regressed", "loc", "transl", "transl_pelvis", "rotvec", "rotmat", "shape", "v3d", "j3d", "j2d")


def load_golden(name):
    with np.load(os.path.join(GOLDEN_DIR, name + ".npz")) as f:
        return {k: torch.from_numpy(f[k]) for k in f.files}


def build_inputs(name, num_verts=NUM_VERTS):
    from multihmr_b200 import synth

    case = CASES[name]
    seed = case["seed"]
    sd = synth.make_anny_state_dict(case["backbone"], case["img_size"], seed=seed, det_bias=case.get("det_bias", -4.0))
    bm = synth.AnnyLikeBodyModel(num_verts, seed)
    x = synth.make_images(case["batch"], case["img_size"], seed)
    K = None if case.get("no_K") else synth.make_cameras(case["batch"], case["img_size"], jitter=True, seed=seed)
    idx = None
    if case["persons"] is not None:
        idx = synth.make_forced_idx(case["batch"], case["img_size"] // 14, case["persons"], seed)
    return case, sd, bm, x, K, idx


def oracle(case, sd, bm, x, K, idx, **kw):
    from oracle import anny_ref

    cfg = anny_ref.AnnyConfig(case["backbone"], case["img_size"])
    if idx is not None:
        return anny_ref.anny_forward(sd, bm, cfg, x, K, idx=idx, is_training=True, **kw)
    kw.setdefault("det_thresh", 0.3)
    kw.setdefault("nms_kernel_size", 3)
    return anny_ref.anny_forward(sd, bm, cfg, x, K, **kw)


def flatten_persons(persons):
    out = {k: torch.stack([p[k] for p in persons]) for k in PERSON_KEYS}
    out["fov"] = persons[0]["fov"]
    return out


def build_engine(case, sd, bm, max_batch=None, max_persons=32, **kw):
    from multihmr_b200.model_anny import ModelAnny

    m = ModelAnny(img_size=case["img_size"], backbone=case["backbone"], simple_depth_encoding=1, body_model=bm,
                  max_batch=max_batch or case["batch"], max_persons=max_persons, **kw)
    m.load_state_dict(sd, strict=False)
    return m
