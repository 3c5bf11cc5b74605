"""Pins oracle/eval_bench_ref.py against the reference's OWN `Trainer.prepare_gt` / `Trainer.evaluate` and writes
tests/golden/eval_{3dpw,ehf,bedlam}.npz.

Runs ONLY in the build container (needs /root/reference).  It imports /root/reference/train.py UNMODIFIED and calls
`Trainer.evaluate` on an instance made with `Trainer.__new__`:
  * smplx.create -> the oracle body-model shims (SMPLShim, SMPLXFullShim); roma -> roma_ref; SummaryWriter -> a
    recorder; plyfile / pyrender / trimesh -> empty modules (render-only imports);
  * the model is a stub returning prescribed person dicts, the loader a list whose `dataset.name` is the protocol;
  * `evaluate` loads models/smpl/J_regressor_h36m.npy relative to the working directory: it runs in a temporary
    directory holding the synthetic regressor there; the module-global `args` of train.py is set;
  * `train.AverageMeter` is replaced by a subclass that records every value, so the per-pair errors are kept.
The restatement must agree with the reference (<= 1e-4 mm per pair, exact detection counts); the npz files hold the
reference's final meters and per-pair values (inputs are regenerated from seeds by eval_bench_ref.make_cases).

Usage:  python -m oracle.make_golden_eval            (from the repo root)
"""
import argparse
import os
import sys
import tempfile
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
REFERENCE = "/root/reference"

from oracle import eval_bench_ref, roma_ref, smplx_ref  # noqa: E402

_MODELS = {}


def install_shims():
    roma = types.ModuleType("roma")
    for k in ("special_gramschmidt", "rotvec_to_rotmat", "rotmat_to_rotvec", "rigid_points_registration"):
        setattr(roma, k, getattr(roma_ref, k))
    sys.modules["roma"] = roma
    smplx = types.ModuleType("smplx")

    def create(model_path, model_type="smplx", gender="neutral", use_pca=False, flat_hand_mean=True, num_betas=10,
               **kw):
        if model_type == "smpl":
            return _MODELS["smpl_" + gender]
        assert model_type == "smplx" and not use_pca and flat_hand_mean
        return _MODELS["smplx"]

    smplx.create = create
    jn = types.ModuleType("smplx.joint_names")
    jn.JOINT_NAMES = smplx_ref.JOINT_NAMES
    smplx.joint_names = jn
    sys.modules["smplx"] = smplx
    sys.modules["smplx.joint_names"] = jn
    for name in ("pyrender", "trimesh", "plyfile"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["plyfile"].PlyData = None  # datasets/ehf.py:22 (mesh files are not read here)
    tb = types.ModuleType("torch.utils.tensorboard")

    class SummaryWriter:
        def __init__(self, *a, **k):
            self.scalars = []

        def add_scalar(self, tag, value, step=None):
            self.scalars.append((tag, float(value), step))

        def flush(self):
            pass

    tb.SummaryWriter = SummaryWriter
    sys.modules["torch.utils.tensorboard"] = tb


class StubModel:
    """Returns the prescribed persons of image i on the i-th call (Trainer.evaluate calls it once per image)."""

    def __init__(self, persons_per_image, img_size):
        self.persons, self.i = persons_per_image, 0
        self.nearness, self.img_size, self.patch_size = True, img_size, 14

    def eval(self):
        return self

    def __call__(self, x, is_training=False, K=None, det_thresh=None, nms_kernel_size=None):
        out = self.persons[self.i]
        self.i += 1
        return out


class Loader(list):
    def __init__(self, items, name):
        super().__init__(items)
        self.dataset = types.SimpleNamespace(name=name, split="test", subsample=1)


def run_reference(train, dataset, cases, assets):
    meters_seen = []
    base = _MODELS.setdefault("AverageMeter", train.AverageMeter)  # the reference's own, whatever ran before

    class RecordingMeter(base):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.values = []
            meters_seen.append(self)

        def update(self, val, n=1):
            self.values.append(float(val))
            super().update(val, n)

    train.AverageMeter = RecordingMeter
    train.args = argparse.Namespace(person_center="head", img_size=eval_bench_ref.IMG_SIZE, amp=0, det_thresh=0.3,
                                    nms_kernel_size=3, log_freq=1000, visu_to_save=0)
    t = train.Trainer.__new__(train.Trainer)
    t.device = torch.device("cpu")
    t.args = train.args
    t.model = StubModel([c[2] for c in cases], eval_bench_ref.IMG_SIZE)
    t.smplx_neutral_11 = _MODELS["smplx"]
    t.smpl_male_10, t.smpl_female_10 = _MODELS["smpl_male"], _MODELS["smpl_female"]
    t.smplx2smpl_regressor = assets["smplx2smpl"].to_dense().float()  # train.py:44-45 (dense, like the pickle)
    t.writer = sys.modules["torch.utils.tensorboard"].SummaryWriter()
    t.current_iter = t.current_epoch = 0
    loader = Loader([(c[0], c[1]) for c in cases], dataset)
    t.evaluate(loader)
    meters = {m.name: m for m in meters_seen if m.name in eval_bench_ref.METERS}
    return ({k: float(meters[k].avg) for k in eval_bench_ref.METERS},
            {k: np.asarray(meters[k].values, dtype=np.float64) for k in ("pve", "pa_pve", "mpjpe", "pa_mpjpe")})


def main():
    assert os.path.isdir(REFERENCE), "make_golden_eval needs the reference checkout (build container only)"
    install_shims()
    torch.manual_seed(0)
    assets = eval_bench_ref.eval_assets(0)
    _MODELS.update(eval_bench_ref.shim_models(assets))
    out_dir = os.path.join(REPO, "tests", "golden")
    cwd = os.getcwd()
    tmp = tempfile.mkdtemp(prefix="mhmr_eval_")
    os.makedirs(os.path.join(tmp, "models", "smpl"))
    np.save(os.path.join(tmp, "models", "smpl", "J_regressor_h36m.npy"), assets["j_regressor_h36m"].numpy())
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    # the reference's datasets/ has no __init__.py: an installed `datasets` package would win over it
    ds = types.ModuleType("datasets")
    ds.__path__ = [os.path.join(REFERENCE, "datasets")]
    sys.modules["datasets"] = ds
    os.chdir(tmp)
    try:
        import train  # the reference, unmodified
    finally:
        os.chdir(cwd)
    only = sys.argv[1:]
    for dataset in eval_bench_ref.DATASETS:
        if only and dataset not in only:
            continue
        cases = eval_bench_ref.make_cases(dataset, assets)
        os.chdir(tmp)
        try:
            with torch.no_grad():
                ref_m, ref_v = run_reference(train, dataset, cases, assets)
        finally:
            os.chdir(cwd)
        mine_m, mine_v = eval_bench_ref.evaluate(cases, _MODELS, assets["smplx2smpl"], assets["j_regressor_h36m"],
                                                 dataset, eval_bench_ref.IMG_SIZE)
        for k in ("precision", "recall", "f1_score"):
            assert ref_m[k] == mine_m[k], (dataset, k, ref_m[k], mine_m[k])
        for k in ("pve", "pa_pve", "mpjpe", "pa_mpjpe"):
            assert ref_v[k].shape == mine_v[k].shape, (dataset, k, ref_v[k].shape, mine_v[k].shape)
            err = np.abs(ref_v[k] - mine_v[k]).max() if ref_v[k].size else 0.0
            assert err <= 1e-4, (dataset, k, err)
            assert abs(ref_m[k] - mine_m[k]) <= 1e-4, (dataset, k, ref_m[k], mine_m[k])
        gold = {f"meter_{k}": np.float64(v) for k, v in ref_m.items()}
        gold.update({f"pairs_{k}": v for k, v in ref_v.items()})
        np.savez_compressed(os.path.join(out_dir, f"eval_{dataset}.npz"), **gold)
        print(f"eval_{dataset}: reference == restatement; " +
              ", ".join(f"{k}={v:.3f}" for k, v in ref_m.items()) + f"; pairs={ref_v['pve'].size}")


if __name__ == "__main__":
    main()
