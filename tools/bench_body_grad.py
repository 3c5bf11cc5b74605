"""Times the body-model backward (mhmr_body_backward, csrc/smplx_lbs.cu) against its forward, with CUDA events over
>= 200 calls after warm-up: SMPL-X (V = 10475, 11 betas) at P = 1, 16 and 48 and SMPL (V = 6890) at P = 2, with random
upstream gradients on every output (v3d, v2d, j3d, j2d, transl_pelvis).  Reports the backward's HBM bytes (from the
shapes, below) over its time against the 3.35 TB/s data-sheet bandwidth of the H100 SXM, and, for context, torch
autograd (forward + backward) through the fp32 oracle on the same GPU.  Prints the card name and power limit.

    python tools/bench_body_grad.py [--calls 200] [--out /tmp/bench_body_grad.json]

Bytes of one backward call: the pose / shape matrix PDX [KT, 3V] once for the recomputed forward and once per pass of
16 persons of the gradient stream, the upstream gradients, the recomputed vertices (written and read back), and the
per-tile partials (written and read back).  The skinning weights, per-person tables and outputs are < 1 % and left out.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_PEAK = 3.35e12


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
    return e0.elapsed_time(e1) * 1e3 / calls  # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_body_grad needs a CUDA device")
    import body_grad_util as bg
    from multihmr_b200 import metrics, synth

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"GPU: {q}")
    res = {"gpu": q, "calls": args.calls, "workloads": {}}
    dev = torch.device("cuda")
    models = {"smplx": (synth.make_body_model(0), 11), "smpl": (synth.make_smpl_body_model(0, "male"), 10)}
    for kind, P in (("smplx", 1), ("smplx", 16), ("smplx", 48), ("smpl", 2)):
        bm, nb = models[kind]
        body = metrics.BodyModel(bm, kind, nb, max_persons=48, device=dev)
        g = torch.Generator().manual_seed(P)
        NJ, V, J = body.num_pose_joints, body.num_verts, body.num_joints
        pose = bg.poses(P, NJ, g)
        betas = torch.randn(P, nb, generator=g)
        transl = torch.randn(P, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 6.0])
        K = torch.tensor([[388.0, 0, 224.0], [0, 388.0, 224.0], [0, 0, 1.0]]).repeat(P, 1, 1)
        expr = torch.randn(P, 10, generator=g) * 0.5 if kind == "smplx" else None
        up = {k: v.to(dev) for k, v in bg.upstream(P, V, J, g, "all").items() if k != "transl"}
        x = body._inputs(pose, betas, transl, K, expr)
        fwd = _time(lambda: body._forward(*x), args.calls, args.warmup)
        bwd = _time(lambda: body._backward(*x, g_v3d=up["v3d"], g_v2d=up["v2d"], g_j3d=up["j3d"], g_j2d=up["j2d"],
                                           g_transl_pelvis=up["transl_pelvis"]), args.calls, args.warmup)
        bwd3 = _time(lambda: body._backward(*x, g_v3d=up["v3d"], g_j3d=up["j3d"]), args.calls, args.warmup)
        KT = 9 * (NJ - 1) + nb + (10 if kind == "smplx" else 0)
        tiles = (V + 79) // 80
        passes = (P + 15) // 16
        pdx = KT * 3 * V * 4
        up_bytes = P * (V * 5 + J * 5 + 3) * 4
        nbytes = pdx * (1 + passes) + up_bytes + 2 * P * V * 3 * 4 + 2 * tiles * P * (NJ * 12 + KT + 12) * 4
        nbytes3 = pdx * passes + P * (V * 3 + J * 3) * 4 + 2 * tiles * P * (NJ * 12 + KT + 12) * 4
        # torch autograd through the fp32 oracle (body_grad_util restates smplx_ref.lbs with autograd-friendly ops)
        leaves = [t.to(dev).requires_grad_() for t in (pose, betas, transl)] + \
                 ([expr.to(dev).requires_grad_()] if expr is not None else [])
        Kd = K.to(dev)

        def oracle():
            out = bg.raw_outputs(bm, leaves[0], leaves[1], leaves[2], Kd, leaves[3] if expr is not None else None)
            return torch.autograd.grad(sum((out[k] * up[k]).sum() for k in up), leaves)

        orc = _time(oracle, max(20, args.calls // 10), 3)
        name = f"{kind}_P{P}"
        r = dict(forward_us=fwd, backward_us=bwd, backward_3d_only_us=bwd3, backward_over_forward=bwd / fwd,
                 backward_bytes=nbytes, backward_GBps=nbytes / bwd * 1e-3, frac_of_3350GBps=nbytes / bwd * 1e6 / HBM_PEAK,
                 backward_3d_only_GBps=nbytes3 / bwd3 * 1e-3, torch_oracle_fp32_fwd_bwd_us=orc)
        res["workloads"][name] = r
        print(f"{name}: forward {fwd:.1f} us, backward {bwd:.1f} us ({bwd / fwd:.2f}x forward; "
              f"{r['backward_GBps']:.0f} GB/s = {100 * r['frac_of_3350GBps']:.0f}% of 3.35 TB/s), 3-D upstream only "
              f"{bwd3:.1f} us ({r['backward_3d_only_GBps']:.0f} GB/s); torch autograd through the fp32 oracle "
              f"{orc:.0f} us")
        del body
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
