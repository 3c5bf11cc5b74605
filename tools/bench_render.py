"""Times the mesh renderer (csrc/render.cu) on three workloads, with CUDA events over >= 200 calls after warm-up, and
per-kernel times from torch.profiler in a separate pass.  Prints the card name and power limit of the same run.

    python tools/bench_render.py [--calls 200] [--out /tmp/bench_render.json]

Workloads: an 896 x 896 image with 4 persons; a 1920 x 1080 photo with 20 persons (the size demo.py renders at);
a 20-frame rotating view of one image with 3 persons in one call (demo.py:160-195).  Meshes are seeded blob people
(`synth.make_blob_people`) of 18 432 faces each, close to SMPL-X's 20 908, between 3 and 8 m from the camera.
Then two `Renderer.render_views` workloads (see `view_workloads`; `--skip-views` leaves them out).  `--dump x.npz`
saves every workload's outputs (overlay, depth and index; for the views also orbit and side), to compare builds bit
for bit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _people(n, W, H, f, seed):
    from multihmr_b200 import synth

    g = np.random.default_rng(seed)
    z = g.uniform(3.0, 8.0, n)
    x = (g.uniform(0.05, 0.95, n) * W - W / 2) * z / f
    y = (g.uniform(0.4, 0.6, n) * H - H / 2) * z / f
    # 32 x 48 segments per ellipsoid: 6 parts -> 9 012 vertices, 18 432 faces, close to SMPL-X (10 475 / 20 908)
    return synth.make_blob_people(np.stack([x, y, z], 1), seed=seed, n_lat=32, n_lon=48)


def _kernel_ms(fn, n=20):
    """Device time per call of each renderer kernel over n calls of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if "render_" in ev.key:
            short = ev.key.split("render_")[1].split("_kernel")[0]
            kern[short] = round(ev.device_time_total / n / 1000.0, 4)
    return kern


def workloads():
    out = {}
    for name, (W, H, n, views) in {"896x896_4p": (896, 896, 4, 1), "1920x1080_20p": (1920, 1080, 20, 1),
                                   "rotate20_1920x1080_3p": (1920, 1080, 3, 20)}.items():
        f = max(W, H) / (2 * np.tan(np.radians(30)))
        verts, faces = _people(n, W, H, f, seed=len(name))
        K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], dtype=torch.float32).expand(views, 3, 3)
        pose = None
        if views > 1:
            c = verts[0].mean(0)
            pose = np.zeros((views, 3, 4))
            for i, a in enumerate(np.deg2rad(np.linspace(0, 60, views))):
                R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
                pose[i, :, :3], pose[i, :, 3] = R, c - R @ c
        out[name] = dict(verts=verts, faces=faces, K=K, pose=pose, W=W, H=H, views=views)
    return out


def view_workloads(res, args, dev, dumps):
    """Renderer.render_views: the demo orbit of one 1920 x 1080 photo with 3 persons (n_frames 20, angle_range 60:
    61 distinct views), and a batch of 8 images at 896 x 896 with 4 persons each taking the overlay, a 20-frame orbit
    and the three side views (with the camera glyph) in one call."""
    from multihmr_b200.render import Renderer, camera_glyph

    for name, (W, H, B, n, side) in {"demo_orbit_1920x1080_3p": (1920, 1080, 1, 3, False),
                                     "views_896_8x4p": (896, 896, 8, 4, True)}.items():
        f = max(W, H) / (2 * np.tan(np.radians(30)))
        verts, faces = _people(n * B, W, H, f, seed=len(name))
        P = n * B
        r = Renderer(faces, dev, topologies=camera_glyph()[0])
        t = {"v3d": torch.from_numpy(verts).to(dev),
             "det_idx": torch.arange(P, dtype=torch.int32, device=dev).div(n, rounding_mode="floor").expand(3, P)
             .contiguous(), "count": torch.full((1,), P, dtype=torch.int32, device=dev),
             "transl_pelvis": torch.from_numpy(verts.mean(1)).to(dev)}
        photos = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device=dev,
                               generator=torch.Generator(dev).manual_seed(len(name)))
        K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], dtype=torch.float32).expand(B, 3, 3).to(dev)
        kw = dict(orbit=(20, 60), side=side, alpha=0.8)
        if args.dump:
            o = r.render_views(t, photos, K, depth=True, index=True, **kw)
            dumps.update({f"{name}_{k}": o[k].cpu().numpy() for k in ("overlay", "orbit", "side", "depth", "index")
                          if k in o})
        for _ in range(args.warmup):
            r.render_views(t, photos, K, **kw)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        calls = max(args.calls // 10, 10)
        e0.record()
        for _ in range(calls):
            r.render_views(t, photos, K, **kw)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / calls
        kern = _kernel_ms(lambda: r.render_views(t, photos, K, **kw), 10)
        views = B * (1 + 60 + (3 if side else 0))
        res["workloads"][name] = {"ms_per_call": round(ms, 4), "ms_per_view": round(ms / views, 4), "views": views,
                                  "persons": P, "faces_per_person": int(faces.shape[0]), "calls": calls,
                                  "kernel_ms_per_call": kern}
        print(f"{name}: {ms:.3f} ms per call, {ms / views:.4f} ms per view ({views} views); kernels {kern}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-views", action="store_true", help="only the three one-topology workloads")
    ap.add_argument("--dump", default=None, help="write the outputs of each workload to this .npz")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_render needs a CUDA device")
    from multihmr_b200.render import Renderer

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    res = {"gpu": q, "calls": args.calls, "workloads": {}}
    print(f"GPU: {q}")
    dev = torch.device("cuda")
    dumps = {}
    for name, w in workloads().items():
        r = Renderer(w["faces"], dev)
        imgs = torch.randint(0, 256, (1, w["H"], w["W"], 3), dtype=torch.uint8, device=dev,
                             generator=torch.Generator(dev).manual_seed(len(name)))
        verts = torch.from_numpy(w["verts"]).to(dev)
        P = verts.shape[0]
        kw = dict(person_image=torch.zeros(P, dtype=torch.int32, device=dev),
                  count=torch.full((1,), P, dtype=torch.int32, device=dev), view_image=[0] * w["views"],
                  pose=w["pose"], alpha=0.8)
        K = w["K"].to(dev)
        if args.dump:
            o = r.render(verts, K, imgs, depth=True, index=True, **kw)
            dumps.update({f"{name}_{k}": v.cpu().numpy() for k, v in o.items()})
        for _ in range(args.warmup):
            r.render(verts, K, imgs, **kw)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.calls):
            r.render(verts, K, imgs, **kw)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.calls
        kern = _kernel_ms(lambda: r.render(verts, K, imgs, **kw))
        res["workloads"][name] = {"ms_per_call": round(ms, 4), "ms_per_view": round(ms / w["views"], 4),
                                  "views": w["views"], "persons": P, "faces_per_person": int(w["faces"].shape[0]),
                                  "kernel_ms_per_call": kern}
        print(f"{name}: {ms:.3f} ms per call, {ms / w['views']:.3f} ms per view; kernels {kern}")
    if not args.skip_views:
        view_workloads(res, args, dev, dumps)
    if args.dump:
        np.savez_compressed(args.dump, **dumps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
