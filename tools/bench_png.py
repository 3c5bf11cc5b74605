"""Times the device PNG decode (csrc/png.cu) against Pillow, and `api.open_images` through the device path against
the host-decode path.  Prints the card name and power limit of the same run, and one JSON object.

    python tools/bench_png.py [--calls 10] [--profile] [--out /tmp/bench_png.json]

Workloads, 8 photos per call: 1280 x 720 RGB (BEDLAM frames), 1600 x 1200 RGB (EHF), 1920 x 1080 RGBA and
4032 x 3024 RGB, each encoded by Pillow at its default level and by OpenCV at its default, plus zlib's Z_FIXED strategy
at 1280 x 720 (every block a fixed-Huffman one: the chain's sequential worst case).  The photos are the two
tests/golden photos upscaled (BICUBIC) to the size, with seeded noise of +-3 added so no two are alike.  Per
workload:
  - device decode of the batch (CUDA events around `ops.png_decode`, after warm-up), and decode + letterbox to 896;
  - Pillow's `Image.open(...).convert("RGB")` per photo on one host thread;
  - `open_images(paths, 896)` wall time through the device path and through the host-decode path, alternated;
  - chain blocks per photo, header candidates (true: on the chain; false: not) and slow-path blocks
    (`ops.png_inflate` counts);
  - whether every device photo equals Pillow's.
With --profile, one decode per workload is traced (torch.profiler) and the device time of every kernel is printed.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BATCH = 8
WORKLOADS = [("1280x720_rgb", 1280, 720, 2), ("1600x1200_rgb", 1600, 1200, 2), ("1920x1080_rgba", 1920, 1080, 6),
             ("4032x3024_rgb", 4032, 3024, 2)]


def photos(W, H, ctype):
    from PIL import Image

    import png_util as U

    gold = U.golden_photos()
    out = []
    for i in range(BATCH):
        im = np.asarray(Image.fromarray(gold[i % len(gold)]).resize((W, H), Image.BICUBIC)).astype(np.int16)
        im = im + np.random.default_rng(i).integers(-3, 4, im.shape)
        im = np.clip(im, 0, 255).astype(np.uint8)
        if ctype == 6:
            a = (np.arange(W)[None, :, None] + np.arange(H)[:, None, None]) % 256
            im = np.concatenate([im, np.broadcast_to(a, (H, W, 1)).astype(np.uint8)], axis=2)
        out.append(im)
    return out


def encode(px, how):
    import cv2

    import png_writer as pw
    from PIL import Image

    if how == "pillow":
        b = io.BytesIO()
        Image.fromarray(px).save(b, "PNG")
        return b.getvalue()
    if how == "opencv":
        conv = cv2.COLOR_RGBA2BGRA if px.shape[2] == 4 else cv2.COLOR_RGB2BGR
        ok, buf = cv2.imencode(".png", cv2.cvtColor(px, conv))
        assert ok
        return buf.tobytes()
    ct = 6 if px.shape[2] == 4 else 2
    return pw.make_png(px, ct, strategy=zlib.Z_FIXED)


def host_path(paths, S, dev):
    from PIL import Image

    from multihmr_b200 import api

    with torch.cuda.device(dev):
        return api._letterbox_photos([Image.open(p).convert("RGB") for p in paths], S, dev, True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3, help="alternated open_images runs of each path")
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true", help="per-kernel device times of one decode per workload")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_png needs a CUDA device")
    import png_util as U
    from multihmr_b200 import api, ops, preprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"GPU: {q}")
    dev = torch.device("cuda")
    res = {"gpu": q, "batch": BATCH, "calls": args.calls, "workloads": {}}
    tmp = tempfile.mkdtemp(prefix="bench_png_")
    runs = [(n, W, H, ct, how) for n, W, H, ct in WORKLOADS for how in ("pillow", "opencv")]
    runs.append(("1280x720_rgb", 1280, 720, 2, "zfixed"))
    cache = {}
    for base, W, H, ct, how in runs:
        name = f"{BATCH}x{base}_{how}"
        if base not in cache:
            cache = {base: photos(W, H, ct)}
        blobs = [encode(p, how) for p in cache[base]]
        paths = []
        for i, b in enumerate(blobs):
            paths.append(os.path.join(tmp, f"{name}_{i}.png"))
            with open(paths[-1], "wb") as fh:
                fh.write(b)
        host_ms, refs = [], []
        for b in blobs:
            t0 = time.perf_counter()
            refs.append(U.pillow(b))
            host_ms.append(1e3 * (time.perf_counter() - t0))
        streams = [ops.png_idat(b) for b in blobs]
        hostb, devb, spans = preprocess.upload_bytes(streams, dev)
        outs = [torch.empty(H, W, 3, dtype=torch.uint8, device=dev) for _ in blobs]
        for _ in range(args.warmup):
            st = ops.png_decode(blobs, hostb, devb, spans, outs)
        torch.cuda.synchronize()
        exact = st.cpu().tolist() == [0] * BATCH and all(np.array_equal(o.cpu().numpy(), r) for o, r in zip(outs, refs))
        raw = H * (1 + W * (4 if ct == 6 else 3))
        _, ist, counts = ops.png_inflate(devb, spans, [raw] * BATCH)
        counts = counts.cpu().numpy()
        assert ist.cpu().tolist() == [0] * BATCH
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        for _ in range(args.calls):
            ops.png_decode(blobs, hostb, devb, spans, outs)
        e1.record()
        for _ in range(args.calls):
            ops.png_decode(blobs, hostb, devb, spans, outs)
            preprocess.letterbox(outs, 896)
        e2.record()
        torch.cuda.synchronize()
        dec_ms = e0.elapsed_time(e1) / args.calls
        both_ms = e1.elapsed_time(e2) / args.calls
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
        r = {"file_mb_mean": sum(len(b) for b in blobs) / BATCH / 2 ** 20,
             "device_decode_ms_per_batch": dec_ms, "device_decode_plus_letterbox_ms_per_batch": both_ms,
             "host_pil_decode_ms_per_photo_median": float(np.median(host_ms)),
             "open_images_device_path_ms_median": float(np.median(dev_wall)),
             "open_images_host_path_ms_median": float(np.median(host_wall)),
             "chain_blocks_per_photo": float(counts[:, 0].mean()),
             "candidates_true_per_photo": float((counts[:, 0] - counts[:, 2]).mean()),
             "candidates_false_per_photo": float((counts[:, 1] - (counts[:, 0] - counts[:, 2])).mean()),
             "slow_path_blocks_per_photo": float(counts[:, 2].mean()),
             "device_equals_pillow": bool(exact), "open_images_paths_equal": bool(same)}
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ops.png_decode(blobs, hostb, devb, spans, outs)
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
