"""Times the device JPEG encode (csrc/jpeg_encode.cu) against Pillow, and `api.create_jpeg` against the same loop run
through Pillow.  Prints the card name and power limit of the same run, and one JSON object.

    python tools/bench_jpeg_encode.py [--calls 20] [--out /tmp/bench_jpeg_encode.json]

Workloads, each a batch of 8 photos (ramps, edges and noise, so the files are larger than typical camera JPEGs of the
same quality, the harder case for the entropy stages):
  - 1920 x 1080 at quality 75, 4:2:0 (Pillow's defaults, what `Image.save(f)` writes);
  - 2688 x 896 at quality 75, 4:2:0: the [photo | prediction | ground truth] panel of the evaluation at 896;
  - 4032 x 3024 at quality 95, 4:4:4.
Per workload: the C entry's device time for the batch (CUDA events around `mhmr_op_jpeg_encode`, after warm-up),
`preprocess.encode_jpeg` wall time (host clock; it ends in its read-back of the files), Pillow's `save` per photo on
one host thread, and whether every device file equals Pillow's.  Then `create_jpeg(root, 512)` over a directory of
1280 x 720 PNGs (BEDLAM's size), in images/s, against datasets/bedlam.py:449-479's loop restated with Pillow (the
files are compared too).
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

BATCH = 8
WORKLOADS = {"1920x1080_q75_420": (1080, 1920, 75, 2), "2688x896_q75_420": (896, 2688, 75, 2),
             "4032x3024_q95_444": (3024, 4032, 95, 0)}


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:h, :w]
    img = np.stack([(x * 255 // w + seed * 17) % 256, (y * 255 // h) * np.ones_like(x), ((x // 64 + y // 64) % 2) * 200],
                   -1).astype(np.int32)
    img += rng.integers(-12, 13, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def pillow_save(img, q, s):
    from PIL import Image

    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "JPEG", quality=q, subsampling=s)
    return buf.getvalue()


def pillow_create_jpeg(root_dir, target_size):
    """datasets/bedlam.py:449-479's loop (without its logging), writing `.pil.jpg` files."""
    from PIL import Image

    for dirpath, _, filenames in os.walk(root_dir):
        for fn in filenames:
            if fn[-4:] == ".png" and fn[0] != ".":
                img_pil = Image.open(os.path.join(dirpath, fn)).convert("RGB")
                width, height = img_pil.size
                if width > height:
                    other = int(float(img_pil.size[1]) * float(target_size / float(img_pil.size[0])))
                    img_pil = img_pil.resize((target_size, other))
                else:
                    other = int(float(img_pil.size[0]) * float(target_size / float(img_pil.size[1])))
                    img_pil = img_pil.resize((other, target_size))
                img_pil.save(os.path.join(dirpath, fn[:-4] + f"_{target_size}.pil.jpg"), "JPEG")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pngs", type=int, default=64, help="1280 x 720 PNGs in the create_jpeg directory")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg_encode needs a CUDA device")
    from PIL import Image

    from multihmr_b200 import api, ops, preprocess
    from multihmr_b200._lib import call, stream

    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"device: {gpu}")
    result = {"device": gpu, "batch": BATCH, "workloads": {}}
    for name, (h, w, q, s) in WORKLOADS.items():
        imgs = [photo(h, w, i) for i in range(BATCH)]
        t0 = time.perf_counter()
        want = [pillow_save(i, q, s) for i in imgs]
        pil_ms = (time.perf_counter() - t0) * 1e3 / BATCH
        timgs = [torch.from_numpy(i).to(dev) for i in imgs]
        got = preprocess.encode_jpeg(timgs, q, s)
        cap = ops.jpeg_capacity(h, w, 3, s)
        out = torch.empty(BATCH * cap, dtype=torch.uint8, device=dev)
        desc = torch.tensor([[t.data_ptr(), h, w, 3 * w, 3, q, s, out.data_ptr() + i * cap, cap]
                             for i, t in enumerate(timgs)], dtype=torch.int64)
        sizes = torch.empty(BATCH, dtype=torch.int64, device=dev)
        status = torch.empty(BATCH, dtype=torch.int32, device=dev)
        for _ in range(args.warmup):
            call("mhmr_op_jpeg_encode", desc, BATCH, sizes, status, stream())
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        times = []
        for _ in range(args.calls):
            ev[0].record()
            call("mhmr_op_jpeg_encode", desc, BATCH, sizes, status, stream())
            ev[1].record()
            torch.cuda.synchronize()
            times.append(ev[0].elapsed_time(ev[1]))
        walls = []
        for _ in range(max(3, args.calls // 4)):
            t0 = time.perf_counter()
            preprocess.encode_jpeg(timgs, q, s)
            walls.append((time.perf_counter() - t0) * 1e3)
        r = {"device_ms_per_batch": float(np.median(times)), "device_ms_min": float(np.min(times)),
             "encode_jpeg_wall_ms_per_batch": float(np.median(walls)), "pillow_ms_per_photo": pil_ms,
             "bytes_per_photo": int(np.mean([len(x) for x in want])), "equal_to_pillow": got == want}
        result["workloads"][name] = r
        print(name, json.dumps(r))

    with tempfile.TemporaryDirectory() as root:
        for i in range(args.pngs):
            Image.fromarray(photo(720, 1280, 100 + i)).save(os.path.join(root, f"{i:04d}.png"))
        api.create_jpeg(root, 512, device=dev)   # warm-up, and the files to compare
        t0 = time.perf_counter()
        api.create_jpeg(root, 512, device=dev)
        dev_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        pillow_create_jpeg(root, 512)
        pil_s = time.perf_counter() - t0
        same = all(open(os.path.join(root, f"{i:04d}_512.jpg"), "rb").read()
                   == open(os.path.join(root, f"{i:04d}_512.pil.jpg"), "rb").read() for i in range(args.pngs))
        result["create_jpeg_1280x720"] = {"device_images_per_s": args.pngs / dev_s,
                                          "pillow_images_per_s": args.pngs / pil_s, "files_equal": same}
        print("create_jpeg", json.dumps(result["create_jpeg_1280x720"]))
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
