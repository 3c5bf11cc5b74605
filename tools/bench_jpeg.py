"""Times the device JPEG decode (csrc/jpeg.cu) against Pillow, and `api.open_images` through the device path against
the host-decode path.  Prints the card name and power limit of the same run, and one JSON object.

    python tools/bench_jpeg.py [--calls 30] [--out /tmp/bench_jpeg.json]

Workloads: 8 photos of 1920 x 1080 (camera frames) and of 4032 x 3024 (12 Mpixel phone pictures), each encoded by
Pillow as 4:2:0 q90, 4:4:4 q95, and 4:2:0 q90 with a restart marker every 4 MCUs.  The photos are ramps, edges and
noise, so the compressed sizes sit above typical camera JPEGs of the same quality (the harder case for the entropy
stage).  Per workload:
  - device decode of the batch (CUDA events around `ops.jpeg_decode`, after warm-up), and decode + letterbox to 896;
  - the synchronisation passes the parallel Huffman decoder needed, and the entropy stage's time
    (`ops.jpeg_coefficients`, CUDA events), at subsequence lengths of 256, 1024 (production) and 4096 bits;
  - Pillow's `Image.open(...).convert("RGB")` per photo on one host thread;
  - `open_images(paths, 896)` wall time (host clock, ending in a synchronise) through the device path and through
    the host-decode path (Pillow decode, upload, device letterbox), alternated in the same process;
  - whether every device photo equals Pillow's.
With --profile, one decode of each workload is also traced (torch.profiler, a run of its own after the timings) and
the device time of every kernel is printed, so the single-CTA planning and scan kernels show beside the decode ones.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BATCH = 8
PHOTOS = [(1920, 1080), (4032, 3024)]
CODINGS = {"420_q90": dict(subsampling=2, quality=90), "444_q95": dict(subsampling=0, quality=95),
           "420_q90_rst4": dict(subsampling=2, quality=90, restart_marker_blocks=4)}


def host_path(paths, S, dev):
    from PIL import Image

    from multihmr_b200 import api

    with torch.cuda.device(dev):
        return api._letterbox_photos([Image.open(p).convert("RGB") for p in paths], S, dev, True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5, help="alternated open_images runs of each path")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true", help="per-kernel device times of one decode per workload")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg needs a CUDA device")
    from PIL import Image

    import jpeg_util as ju
    from multihmr_b200 import api, ops, preprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"GPU: {q}")
    dev = torch.device("cuda")
    res = {"gpu": q, "batch": BATCH, "calls": args.calls, "workloads": {}}
    tmp = tempfile.mkdtemp(prefix="bench_jpeg_")
    for W, H in PHOTOS:
        imgs = [ju.photo(W, H, i) for i in range(BATCH)]
        for cname, kw in CODINGS.items():
            name = f"{BATCH}x{W}x{H}_{cname}"
            blobs = []
            for im in imgs:
                b = io.BytesIO()
                Image.fromarray(im).save(b, format="JPEG", **kw)
                blobs.append(b.getvalue())
            paths = []
            for i, b in enumerate(blobs):
                paths.append(os.path.join(tmp, f"{name}_{i}.jpg"))
                with open(paths[-1], "wb") as fh:
                    fh.write(b)
            host_ms = []
            for b in blobs:
                t0 = time.perf_counter()
                Image.open(io.BytesIO(b)).convert("RGB")
                host_ms.append(1e3 * (time.perf_counter() - t0))
            hostb, devb, spans = preprocess.upload_bytes(blobs, dev)
            outs = [torch.empty(H, W, 3, dtype=torch.uint8, device=dev) for _ in blobs]
            for _ in range(args.warmup):
                st = ops.jpeg_decode(hostb, devb, spans, outs)
            torch.cuda.synchronize()
            exact = st.cpu().tolist() == [0] * BATCH and all(
                np.array_equal(o.cpu().numpy(), ju.pillow_rgb(b)) for o, b in zip(outs, blobs))
            sweep = {}
            for bits in (256, 1024, 4096):
                _, _, passes = ops.jpeg_coefficients(hostb, devb, spans, bits)
                c0, c1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                c0.record()
                for _ in range(5):
                    ops.jpeg_coefficients(hostb, devb, spans, bits)
                c1.record()
                torch.cuda.synchronize()
                sweep[bits] = {"sync_passes": int(passes.item()), "entropy_ms_per_batch": c0.elapsed_time(c1) / 5}
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            for _ in range(args.calls):
                ops.jpeg_decode(hostb, devb, spans, outs)
            e1.record()
            for _ in range(args.calls):
                ops.jpeg_decode(hostb, devb, spans, outs)
                preprocess.letterbox(outs, 896)
            e2.record()
            torch.cuda.synchronize()
            dec_ms = e0.elapsed_time(e1) / args.calls
            both_ms = e1.elapsed_time(e2) / args.calls
            for _ in range(2):   # warm both open_images paths
                api.open_images(paths, 896, dev, fused=True)
                host_path(paths, 896, dev)
            torch.cuda.synchronize()
            dev_wall, host_wall = [], []
            for _ in range(args.reps):
                for fn, acc in ((lambda: api.open_images(paths, 896, dev, fused=True), dev_wall),
                                (lambda: host_path(paths, 896, dev), host_wall)):
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    acc.append(1e3 * (time.perf_counter() - t0))
            a = api.open_images(paths, 896, dev, fused=True)
            h = host_path(paths, 896, dev)
            same = torch.equal(a[0], h[0]) and all(torch.equal(x, y) for x, y in zip(a[1], h[1]))
            r = {"file_kb_mean": sum(len(b) for b in blobs) / BATCH / 1024,
                 "device_decode_ms_per_batch": dec_ms, "device_decode_plus_letterbox_ms_per_batch": both_ms,
                 "subsequence_sweep": sweep,
                 "host_pil_decode_ms_per_photo_median": float(np.median(host_ms)),
                 "open_images_device_path_ms_median": float(np.median(dev_wall)),
                 "open_images_host_path_ms_median": float(np.median(host_wall)),
                 "device_equals_pillow": bool(exact), "open_images_paths_equal": bool(same)}
            if args.profile:
                from torch.profiler import ProfilerActivity, profile

                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    ops.jpeg_decode(hostb, devb, spans, outs)
                    torch.cuda.synchronize()
                r["kernel_us"] = {e.key: round(getattr(e, "device_time_total", 0.0), 1) for e in prof.key_averages()
                                  if getattr(e, "device_time_total", 0.0) > 0}
            res["workloads"][name] = r
            print(name, json.dumps(r), flush=True)
            for p in paths:
                os.remove(p)
    os.rmdir(tmp)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
