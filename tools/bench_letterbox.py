"""Times the letterbox of full-resolution photos into the model input (`ImageOps.contain` + `ImageOps.pad`, BICUBIC):
Pillow on one host thread per photo, and the device kernels (csrc/letterbox.cu) with CUDA events per batch of 8
photos.  Prints the card name and power limit of the same run, and one JSON object.

    python tools/bench_letterbox.py [--calls 50] [--out /tmp/bench_letterbox.json]

Workloads: 8 photos of 1920 x 1080 (camera frames) and of 4032 x 3024 (12 Mpixel phone pictures) into S = 896 and
1288.  Device GB/s is over the bytes the two passes must move at least: each photo read once and the S x S x 3 output
written once; the uint8 workspace between the passes (written and read once) is reported beside it.  The first
photo's device output is checked against Pillow's in the same run.  `call_return_ms_behind_busy_stream` is the host
time of one letterbox call enqueued behind ~50 ms of queued GPU work: near zero if the call does not wait for the
stream, near 50 if the table upload synchronises it.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH = 8
PHOTOS = [(1920, 1080), (4032, 3024)]
SIZES = [896, 1288]


def workspace_bytes(W, H, S):
    """Bytes of the workspace of one photo: the horizontal pass over the rows the vertical windows touch."""
    from oracle import letterbox_ref as lr

    nw, nh = lr.contain_size(W, H, S)
    if nw == W:
        return 0
    xmin, n, _ = lr.coefficients(H, nh) if nh != H else (np.arange(H), np.ones(H, np.int64), None)
    return int(xmin[-1] + n[-1] - xmin[0]) * nw * 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--host-reps", type=int, default=2, help="Pillow letterboxes of each of the 8 photos")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_letterbox needs a CUDA device")
    from PIL import Image, ImageOps

    from multihmr_b200 import ops

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"GPU: {q}")
    dev = torch.device("cuda")
    res = {"gpu": q, "batch": BATCH, "calls": args.calls, "workloads": {}}
    for W, H in PHOTOS:
        rng = np.random.default_rng(W)
        imgs = [rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8) for _ in range(BATCH)]
        pils = [Image.fromarray(im) for im in imgs]
        photos = [torch.from_numpy(im).to(dev) for im in imgs]
        for S in SIZES:
            name = f"{BATCH}x{W}x{H}_to_{S}"
            host = []
            for _ in range(args.host_reps):
                for im in pils:
                    t0 = time.perf_counter()
                    ImageOps.pad(ImageOps.contain(im, (S, S)), size=(S, S))
                    host.append(time.perf_counter() - t0)
            for _ in range(args.warmup):
                out, _ = ops.letterbox_u8(photos, S)
            torch.cuda.synchronize()
            ref = np.asarray(ImageOps.pad(ImageOps.contain(pils[0], (S, S)), size=(S, S)))
            exact = bool(np.array_equal(out[0].cpu().numpy(), ref))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.calls):
                ops.letterbox_u8(photos, S)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.calls
            moved = BATCH * (W * H * 3 + S * S * 3)
            ws = BATCH * workspace_bytes(W, H, S)
            r = {"host_pil_ms_per_photo_median": 1e3 * float(np.median(host)),
                 "host_pil_ms_per_photo_min": 1e3 * float(np.min(host)),
                 "device_ms_per_batch": ms, "device_ms_per_photo": ms / BATCH,
                 "bytes_photo_plus_output": moved, "device_gbps_photo_plus_output": moved / ms / 1e6,
                 "bytes_workspace_write_plus_read": 2 * ws,
                 "device_gbps_with_workspace": (moved + 2 * ws) / ms / 1e6, "first_photo_equals_pillow": exact}
            res["workloads"][name] = r
            print(name, json.dumps(r))
    # Does the call wait for work already queued on its stream?  ~50 ms of sleep kernel, then one call.
    S = SIZES[0]
    ops.letterbox_u8(photos, S)
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)                     # 1e8 SM cycles, ~50 ms at the H100's ~2 GHz

    t0 = time.perf_counter()
    ops.letterbox_u8(photos, S)
    res["call_return_ms_behind_busy_stream"] = 1e3 * (time.perf_counter() - t0)
    torch.cuda.synchronize()
    res["busy_stream_total_ms"] = 1e3 * (time.perf_counter() - t0)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
