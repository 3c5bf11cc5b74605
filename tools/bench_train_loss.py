"""Times the training loss and its backward (mhmr_train_loss, csrc/train_loss.cu) at the 896_L workload: ViT-L, 896 px,
batch 8, 16 forced persons per image (P = 128), SMPL-X with 11 betas, 2-D terms on.  Reports, with CUDA events after
warm-up:
  * the loss + backward on its own, on one forward's outputs;
  * Model.training_loss (forced-index forward + loss + backward) and the forward alone;
  * torch autograd (forward + backward) through the fp32 oracle statement of the same loss on the same outputs
    (tests/train_loss_util: head post-processing, placed SMPL-X layer, loss.py).
Prints the card name and power limit.  Targets are the outputs moved by 5 cm / 5 px noise.

    python tools/bench_train_loss.py [--calls 50] [--out /tmp/bench_train_loss.json]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _time(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls  # ms per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_loss needs a CUDA device")
    import train_loss_util as tl
    from multihmr_b200 import synth
    from multihmr_b200.loss import TARGETS, run_train_loss
    from multihmr_b200.model import Model

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"GPU: {q}")
    dev = torch.device("cuda")
    B, S, per, nb = 8, 896, 16, 11
    bm = synth.make_body_model(0)
    m = Model(backbone="dinov2_vitl14", img_size=S, num_betas=nb, max_batch=B, max_persons=B * per, body_model=bm,
              device=dev)
    m.load_state_dict(synth.make_state_dict("dinov2_vitl14", S, num_betas=nb, seed=0), strict=False)
    res = m.res
    x = synth.make_images(B, S, 0).to(dev)
    K = synth.make_cameras(B, S, jitter=True, seed=0).to(dev)
    idx = synth.make_forced_idx(B, res, per, 0)
    t, P = m.forward_raw(x, K, idx=idx, want_v2d=True, want_dec=True)
    g = torch.Generator(device="cpu").manual_seed(0)
    noise = lambda a, s: (a + s * torch.randn(a.shape, generator=g).to(dev)).contiguous()
    y = {k: noise(t[k][:P], 0.05) for k in ("offset", "rotmat", "transl", "transl_pelvis", "j3d", "v3d")}
    y.update(j2d=noise(t["j2d"][:P], 5.0), v2d=noise(t["v2d"][:P], 5.0), dist_postprocessed=noise(t["dist_pp"][:P], 0.05),
             shape=noise(t["shape"][:P], 0.05))
    y["scores"] = torch.zeros(B, res, res, device=dev)
    y["scores"][idx[0], idx[1], idx[2]] = 1.0
    y.update(idx=idx, K=K)
    largs = types.SimpleNamespace(**{"alpha_" + k: v for k, v in tl.WEIGHTS.items()}, start_2d_epoch=10)
    assert all(k in y for k in TARGETS)

    loss_ms = _time(lambda: run_train_loss(m, t, P, K, y, 12, largs), args.calls, args.warmup)
    step_ms = _time(lambda: m.training_loss(x, y, 12, largs), max(10, args.calls // 5), 2)
    fwd_ms = _time(lambda: m.forward_raw(x, K, idx=idx, want_v2d=True, want_dec=True), max(10, args.calls // 5), 2)

    # torch autograd through the fp32 oracle statement on the same head outputs
    bm_dev = {k: (torch.as_tensor(v).to(dev) if torch.is_tensor(v) else v) for k, v in bm.items()}
    det = t["det_idx"][:, :P].long()
    cells = torch.stack([det[2], det[1]], 1)
    K_det = K[det[0]]
    logit = torch.logit(t["scores_map"].double()).float()
    leaves = [a.detach().clone().requires_grad_() for a in (logit, t["dec"][:P], t["offset"][:P])]
    yf = {k: y[k].float() for k in TARGETS}

    def oracle():
        yh = tl.forward(bm_dev, leaves[0], leaves[1], leaves[2], cells, K_det, nb, S)
        L = tl.total(tl.loss_terms(yh, yf, S), tl.WEIGHTS, True)
        return torch.autograd.grad(L, leaves)

    orc_ms = _time(oracle, 5, 1)
    r = dict(gpu=q, workload="896_L batch 8, 16 persons per image", persons=P, loss_backward_ms=loss_ms,
             training_loss_ms=step_ms, forward_ms=fwd_ms, torch_oracle_fp32_ms=orc_ms)
    print(f"P={P}: loss + backward {loss_ms:.3f} ms; training_loss {step_ms:.2f} ms (forward alone {fwd_ms:.2f} ms); "
          f"torch autograd through the fp32 oracle {orc_ms:.1f} ms ({orc_ms / loss_ms:.0f}x)")
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(r, fh, indent=1)


if __name__ == "__main__":
    main()
