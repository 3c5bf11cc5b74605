"""Times the evaluation of one 3DPW-sized image on the device (CUDA events, after warm-up): the ground-truth SMPL
forward for 2 persons (male and female, as prepare_gt runs both when a female is present), matching, the SMPL-X ->
SMPL regression of the 2 matched predictions, PVE / PA-PVE and MPJPE / PA-MPJPE.  Prints one JSON line.

Usage:  python tools/bench_eval.py [--iters 200]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from multihmr_b200 import metrics, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    assets = metrics.EvalAssets(synth.make_body_model(0), synth.make_smpl_body_model(0, "male"),
                                synth.make_smpl_body_model(0, "female"), synth.make_smplx2smpl(0),
                                synth.make_j_regressor_h36m(0), device=dev, max_persons=8)
    g = torch.Generator().manual_seed(0)
    P = 2
    pose = (torch.randn(P, 24, 3, generator=g) * 0.3).to(dev)
    betas = torch.randn(P, 10, generator=g).to(dev)
    transl = torch.tensor([[-0.8, 0.0, 6.0], [0.8, 0.0, 6.5]], device=dev)
    K = torch.tensor([[776.0, 0, 448], [0, 776.0, 448], [0, 0, 1]], device=dev).expand(P, 3, 3).contiguous()
    # predictions: SMPL-X bodies near the two persons
    px = assets["smplx"](torch.randn(P, 55, 3, generator=g).to(dev) * 0.1, torch.zeros(P, 11, device=dev),
                         transl, K)
    persons = [dict(j2d=px["j2d"][i], v3d=px["v3d"][i], transl_pelvis=px["transl_pelvis"][i:i + 1]) for i in range(P)]
    # the two ground truths must be matched for the timing to include the 3-D errors: use the predictions' 2-D joints
    male, female = assets["smpl_male"], assets["smpl_female"]

    def one_image():
        gt = male(pose, betas, transl, K)
        fem = female(pose, betas, transl, K)
        for k in gt:
            gt[k][1] = fem[k][1]
        gt["j2d"] = px["j2d"][:, :45]
        ev = metrics.Evaluator(assets.smplx2smpl, assets.j_regressor_h36m, device=dev)
        ev.update(persons, gt)
        return ev

    for _ in range(args.warmup):
        ev = one_image()
    assert len(ev.values["pve"]) == 2 and len(ev.values["mpjpe"]) == 2
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.iters):
        one_image()
    stop.record()
    stop.synchronize()
    ms = start.elapsed_time(stop) / args.iters
    print(json.dumps({"metric": "eval_3dpw_image_ms", "value": round(ms, 4), "persons": P, "iters": args.iters,
                      "device": torch.cuda.get_device_name(dev),
                      "note": "GT SMPL forward x2 genders + matching + SMPL-X->SMPL regression + PVE/MPJPE, "
                              "one host read-back per image"}))


if __name__ == "__main__":
    main()
