#!/usr/bin/env python
"""Benchmark of the Multi-HMR hot path (BASELINE.json: images/sec, multiHMR_896_L, batch 8 per GPU).

  python bench.py --gpus N --steps K --warmup W            this repo: sm_90a engine through the C-ABI
  python bench.py ... --dump-outputs DIR                   also writes what the last timed step computed as
                                                           DIR/<name>.npy (float32 / float64)
  python bench.py --impl reference --gpus N --steps K ...  reference arm: the reference's algorithm on the
                                                           host CPU cores (oracle port, fp32 PyTorch)

One "step" = one pass of `Model.forward(x, K)` over one batch of 8 synthetic 896x896 images per GPU
(random-init weights of the ViT-L architecture, seeded).  N > 1 is launched by torchrun, one rank per GPU,
image shards per rank (weak scaling) + one NCCL all-gather of the per-person records per step.

Prints ONE JSON line (rank 0):  value = whole-job images/s with inputs resident in HBM; e2e = the same
metric through the public API with pinned HOST inputs (H2D) and host outputs (D2H) inside the timed
region; roofline = live CUDA-event timing of the dominant kernel family vs the measured peak;
cpu_baseline = the oracle port timed on this box's host cores on a bounded sample (1 image).
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# BASELINE.json configs that fit one GPU (c1 is the CPU-runnable plumbing case, c4 = c3 under --gpus 8).
# The headline (metric quoted in BASELINE.json) is c3; c2 / c5 are selectable with --config and c2 is also
# measured as a short secondary leg of the default run (north_star asks for 672x672 images/s as well).
CONFIGS = {
    "c2": dict(name="multiHMR_672_L", backbone="dinov2_vitl14", img_size=672, batch_per_gpu=4, det_thresh=0.3,
               nms_kernel_size=3, target_persons_per_image=2, seed=0),
    "c3": dict(name="multiHMR_896_L", backbone="dinov2_vitl14", img_size=896, batch_per_gpu=8, det_thresh=0.3,
               nms_kernel_size=3, target_persons_per_image=2, seed=0),
    "c5": dict(name="multiHMR_1288_L_bedlam", backbone="dinov2_vitl14", img_size=1288, batch_per_gpu=2,
               det_thresh=0.3, nms_kernel_size=3, target_persons_per_image=20, seed=0),
}
WORKLOAD = dict(CONFIGS["c3"])
ARCH = {"dinov2_vits14": (384, 12), "dinov2_vitb14": (768, 12), "dinov2_vitl14": (1024, 24)}
METRIC = "images/sec multiHMR_896_L bs=8"


def set_workload(key: str):
    global METRIC
    WORKLOAD.clear()
    WORKLOAD.update(CONFIGS[key])
    METRIC = f"images/sec {WORKLOAD['name']} bs={WORKLOAD['batch_per_gpu']}"


def vit_flops_per_image(backbone: str, img_size: int) -> float:
    """SURVEY.md §8(d): depth*(24 T D^2 + 4 T^2 D) + 2 N 588 D (matmul 2mnk only)."""
    D, depth = ARCH[backbone]
    N = (img_size // 14) ** 2
    T = N + 1
    return depth * (24.0 * T * D * D + 4.0 * T * T * D) + 2.0 * N * 588 * D


def measured_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as fh:
            p = json.load(fh)
        return dict(tflops=float(p.get("bf16_tflops_sustained", p.get("bf16_tflops", 989.0))),
                    hbm_gbs=float(p.get("hbm_gbs", 3350.0)), source="MEASURED_PEAKS.json (measured)")
    # NVIDIA H100 SXM data sheet (700 W card), dense fp16 tensor-core rate and HBM3 bandwidth: not measured
    return dict(tflops=989.0, hbm_gbs=3350.0, source="H100 SXM data sheet, dense fp16")


class ClockSampler:
    """nvidia-smi clocks + throttle reasons sampled DURING the timed region: the sampler runs from before the warm-up, and only samples stamped inside [mark_start, mark_stop] count."""

    Q = ("timestamp,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index, self.proc, self.t0, self.t1 = index, None, None, None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "50"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self.proc = None

    def mark_start(self):
        import datetime
        self.t0 = datetime.datetime.now()

    def mark_stop(self):
        import datetime
        self.t1 = datetime.datetime.now()

    def stop(self) -> dict:
        import datetime
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.12)
        self.proc.terminate()
        try:
            out, _ = self.proc.communicate(timeout=5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            out, _ = self.proc.communicate()
        sm, mx, pw, reasons, n_all = [], [], [], set(), 0
        names = ("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap")
        for line in out.strip().splitlines():
            f = [c.strip() for c in line.split(",")]
            if len(f) < 8:
                continue
            try:
                ts = datetime.datetime.strptime(f[0], "%Y/%m/%d %H:%M:%S.%f")
                vals = (float(f[1]), float(f[2]), float(f[3]))
            except ValueError:
                continue
            n_all += 1
            if self.t0 is not None and not (self.t0 <= ts <= self.t1):
                continue
            sm.append(vals[0]); mx.append(vals[1]); pw.append(vals[2])
            for n, v in zip(names, f[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "samples": 0, "samples_total": n_all,
                    "reasons": ["no samples inside the timed region"]}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "power_w_max": max(pw),
                "samples": len(sm), "reasons": sorted(reasons)}


def dist_env():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    return world, rank, local


# ------------------------------------------------------------------------------------------------
# synthetic workload
# ------------------------------------------------------------------------------------------------
def build_workload(det_bias: float):
    from multihmr_b200 import synth

    w = WORKLOAD
    sd = synth.make_state_dict(w["backbone"], w["img_size"], seed=w["seed"], det_bias=det_bias)
    bm = synth.make_body_model(w["seed"])
    return sd, bm


def calibrate_det_bias(model, x, K, target_total: int, det_thresh: float) -> float:
    """Random-init weights have no meaningful detection density: shift the detection logit so that about
    `target_total` NMS maxima pass the threshold on this batch (setup, untimed)."""
    import torch

    res = model.res
    idx = (torch.zeros(1, dtype=torch.int64),) * 4
    out = model(x, idx=idx, K=K, is_training=True)  # training-style: raw sigmoid scores, no NMS
    s = out["scores"][..., 0].float().cpu().clamp(1e-4, 1 - 1e-4)
    logit = torch.log(s / (1 - s))
    mx = torch.nn.functional.max_pool2d(logit[:, None], 3, 1, 1)[:, 0]
    peaks = logit[(mx == logit)].flatten().sort(descending=True).values
    k = min(target_total, peaks.numel() - 1)
    cut = 0.5 * (peaks[k - 1] + peaks[k]).item()
    want = math.log(det_thresh / (1 - det_thresh))
    return want - cut  # added to the current bias (0)


# ------------------------------------------------------------------------------------------------
# this repo's arm
# ------------------------------------------------------------------------------------------------
class OursBench:
    """One workload on this rank's GPU: calibrated synthetic detection density, device-resident steps,
    end-to-end steps through the public API, per-kernel-family profile."""

    def __init__(self, w, world, rank, dev):
        import torch

        from multihmr_b200 import synth
        from multihmr_b200.model import Model

        self.w, self.world, self.rank, self.dev = w, world, rank, dev
        B, S = w["batch_per_gpu"], w["img_size"]
        self.B, self.S = B, S
        self.max_persons = max(64, 2 * B * w["target_persons_per_image"])
        # ---- setup (untimed): weights, calibration of the synthetic detection density, final engine
        # uint8 RGB HWC, what open_image produces before normalize_rgb (demo.py:33-47): the engine's fused loader
        # normalises on the device, so a step uploads 3 bytes per pixel instead of 12
        self.x_host = synth.make_images_u8(B, S, seed=w["seed"] + rank).pin_memory()
        self.K_host = synth.make_cameras(B, S, seed=w["seed"] + rank).pin_memory()
        sd = synth.make_state_dict(w["backbone"], S, seed=w["seed"], det_bias=0.0)
        bm = synth.make_body_model(w["seed"])
        mk = lambda: Model(backbone=w["backbone"], img_size=S, max_batch=B, max_persons=self.max_persons,
                           body_model=bm, device=dev)
        model = mk()
        model.load_state_dict(sd)
        self.x_dev, self.K_dev = self.x_host.to(dev), self.K_host.to(dev)
        shift = calibrate_det_bias(model, self.x_dev, self.K_dev, w["target_persons_per_image"] * B, w["det_thresh"])
        del model
        torch.cuda.empty_cache()
        sd["mlp_classif.2.bias"] = sd["mlp_classif.2.bias"] + shift
        self.model = mk()
        self.model.load_state_dict(sd)
        self.model.finalize()
        self.sharded = None
        if world > 1:
            from multihmr_b200 import parallel
            self.sharded = parallel.RecordGather(self.model, rank, world)
        self.host_out = {}
        self.loader = None

    def step_device(self):
        w, m = self.w, self.model
        t, P = m.forward_raw(self.x_dev, self.K_dev, det_thresh=w["det_thresh"], nms_kernel_size=w["nms_kernel_size"])
        if self.sharded is not None:
            self.sharded.gather_async(t, self.rank * self.B)
        return P

    def step_e2e(self):
        # public API with HOST buffers: pinned H2D of the images, forward, D2H of every person tensor
        import torch

        from multihmr_b200.api import HostBatchLoader, forward_model
        w, m = self.w, self.model
        # every step uploads its own inputs from pinned host memory; the upload of step i+1 is submitted right after
        # step i's has been handed to the forward, so it overlaps that forward (double-buffered loader)
        if self.loader is None:
            self.loader = HostBatchLoader(self.dev)
        if not self.loader.pending:
            self.loader.submit(self.x_host, self.K_host)
        x, K = self.loader.get()
        self.loader.submit(self.x_host, self.K_host)
        persons = forward_model(m, x, K, det_thresh=w["det_thresh"], nms_kernel_size=w["nms_kernel_size"])
        t = m.last_outputs
        P = len(persons)
        nbytes = 0
        for k in ("det_score", "loc", "transl", "transl_pelvis", "rotvec", "expression", "shape", "v3d", "j3d", "j2d"):
            src = t[k][:P]
            if k not in self.host_out or self.host_out[k].shape[0] < P:
                self.host_out[k] = torch.empty((self.max_persons,) + tuple(src.shape[1:]), dtype=src.dtype).pin_memory()
            self.host_out[k][:P].copy_(src, non_blocking=True)
            nbytes += src.numel() * src.element_size()
        if self.sharded is not None:
            self.sharded.gather_async(t, self.rank * self.B)
            self.sharded.wait()
        torch.cuda.current_stream().synchronize()
        return P, nbytes

    def timed(self, fn, steps, warmup, sampler=None):
        import torch
        import torch.distributed as dist

        for _ in range(warmup):
            fn()
        if self.sharded is not None:
            self.sharded.wait()
        if self.world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        if sampler:
            sampler.mark_start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        last = None
        for _ in range(steps):
            last = fn()
        if self.sharded is not None:
            self.sharded.wait()   # the last step's gather is part of the timed region
        e1.record()
        torch.cuda.synchronize()
        if sampler:
            sampler.mark_stop()
        clocks = sampler.stop() if sampler else None
        ms = torch.tensor([e0.elapsed_time(e1)], device=self.dev)
        if self.world > 1:
            dist.barrier()
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return ms.item(), last, clocks

    def profile(self, steps):
        """Separate pass with an event pair around every launch (serialises the PDL chain: used for the family
        breakdown and the roofline of the dominant kernel, never for `value`)."""
        import torch

        m = self.model
        m.set_profiling(True)
        self.step_device()
        m.get_profile()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            self.step_device()
        e1.record()
        torch.cuda.synchronize()
        prof = m.get_profile()
        m.set_profiling(False)
        return prof, e0.elapsed_time(e1)


def run_ours(args):
    import torch
    import torch.distributed as dist

    world, rank, local = dist_env()
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("--gpus N > 1 must be launched with torchrun (one rank per GPU)")
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: the product path has no CPU fallback")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        # stdout carries exactly one JSON line: keep NCCL's "NCCL version ..." banner (NCCL_DEBUG=VERSION) out of it
        if os.environ.get("NCCL_DEBUG", "VERSION").upper() == "VERSION":
            os.environ["NCCL_DEBUG"] = "WARN"
        dist.init_process_group("nccl", device_id=dev)
    w = WORKLOAD
    B, S = w["batch_per_gpu"], w["img_size"]
    bench = OursBench(w, world, rank, dev)

    # ---- device-resident throughput (value): profiling OFF, the PDL chain runs as in production
    sampler = ClockSampler(local)
    sampler.start()
    ms_total, P_last, clocks = bench.timed(bench.step_device, args.steps, args.warmup, sampler)
    launches = bench.model.last_launch_count()
    if args.dump_outputs and rank == 0:
        dump_outputs(bench.model.last_outputs, int(P_last), args.dump_outputs)
    value = world * B * args.steps / (ms_total / 1e3)

    # ---- end to end through the public API with host buffers
    ms_e2e, last, _ = bench.timed(bench.step_e2e, args.steps, max(1, args.warmup // 2))
    e2e_value = world * B * args.steps / (ms_e2e / 1e3)
    P_e2e, d2h_bytes = last
    h2d_bytes = bench.x_host.numel() * bench.x_host.element_size() + bench.K_host.numel() * 4

    # ---- per-kernel-family breakdown (separate pass, events around every launch)
    prof_steps = max(1, min(args.steps, 5))
    prof, ms_prof = bench.profile(prof_steps)

    secondary = None
    if world == 1 and args.config == "c3" and not args.no_secondary:
        # north_star: images/s on 672x672 batches as well (BASELINE config c2), short leg
        del bench
        torch.cuda.empty_cache()
        w2 = CONFIGS["c2"]
        b2 = OursBench(w2, 1, 0, dev)
        steps2 = args.steps
        ms2, P2, _ = b2.timed(b2.step_device, steps2, 3)
        ms2e, _, _ = b2.timed(b2.step_e2e, steps2, 2)
        secondary = {"workload": f"{w2['name']} batch {w2['batch_per_gpu']}, synthetic 672x672", "steps": steps2,
                     "value": round(w2["batch_per_gpu"] * steps2 / (ms2 / 1e3), 2), "unit": "images/s",
                     "ms_per_step": round(ms2 / steps2, 3),
                     "e2e_value": round(w2["batch_per_gpu"] * steps2 / (ms2e / 1e3), 2), "persons_in_batch": int(P2),
                     "vit_flop_frac_of_peak": round(vit_flops_per_image(w2["backbone"], 672) * w2["batch_per_gpu"] * steps2
                                                    / (ms2 / 1e3) / 1e12 / measured_peaks()["tflops"], 4)}
        del b2

    if world > 1:
        bench.sharded.close()   # the library's own NCCL communicator
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    peaks = measured_peaks()
    D, depth = ARCH[w["backbone"]]
    N = (S // 14) ** 2
    T, M = N + 1, B * (N + 1)
    algo_flops = {  # algorithmic FLOPs per launch (2mnk)
        "gemm_qkv": 2.0 * M * 3 * D * D, "gemm_proj": 2.0 * M * D * D, "gemm_fc1": 2.0 * M * 4 * D * D,
        "gemm_fc2": 2.0 * M * 4 * D * D, "attention": 4.0 * B * T * T * D,
    }
    prof_sum = sum(v[0] for v in prof.values())
    fam = {}
    for k, fl in algo_flops.items():
        ms, n = prof[k]
        if n:
            fam[k] = dict(ms_per_launch=ms / n, launches_per_step=n / prof_steps,
                          tflops=fl / (ms / n) / 1e9, share_of_step=ms / prof_sum)
    dom = max(fam, key=lambda k: fam[k]["share_of_step"]) if fam else None
    # whole-step ViT FLOP rate from the UNPROFILED timed region (the head is ~3 % of the step)
    vit_tflops_step = vit_flops_per_image(w["backbone"], S) * B * args.steps / (ms_total / 1e3) / 1e12
    roofline = None
    if dom:
        roofline = {"bound": "tensor", "kernel": dom, "achieved": round(fam[dom]["tflops"], 1),
                    "peak": peaks["tflops"], "unit": "TFLOP/s", "frac": round(fam[dom]["tflops"] / peaks["tflops"], 4),
                    "peak_source": peaks["source"],
                    "timing": f"CUDA events around every launch, separate pass of {prof_steps} steps "
                              f"({ms_prof / prof_steps:.2f} ms/step with the events in)",
                    "families": {k: {a: round(b, 4) for a, b in v.items()} for k, v in fam.items()},
                    "vit_backbone": {"tflops_whole_step": round(vit_tflops_step, 1),
                                     "frac_of_peak": round(vit_tflops_step / peaks["tflops"], 4)},
                    "other_ms_per_step": {k: round(prof[k][0] / prof_steps, 3)
                                          for k in ("misc", "layernorm", "gemm_other", "head", "smplx", "refine")
                                          if k in prof}}
    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        cpu = cpu_baseline(images=1)
    line = {
        "metric": METRIC, "value": round(value, 3), "unit": "images/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": round(ms_total / args.steps, 3), "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "fp16 tensor-core operands, fp32 accumulate/residual",
        "data": "synthetic",
        "config": {"workload": f"{w['name']} batch {B}/GPU, synthetic {S}x{S}, random-init ViT-L weights",
                   "input": "uint8 RGB HWC images (fused normalize_rgb + patch-row loader on the device)",
                   "images_per_gpu": B, "global_batch": world * B, "persons_in_batch": int(P_last),
                   "det_thresh": w["det_thresh"], "nms_kernel_size": w["nms_kernel_size"],
                   "parallelism": f"dp{world} (image shards, 1 all-gather of person records)" if world > 1 else "dp1",
                   "l2": "working set per step (0.6 GB fp16 weights + >1 GB activations) exceeds the 50 MB L2"},
        "clocks": clocks, "gpu_launches": int(launches),
        "e2e": {"value": round(e2e_value, 3), "unit": "images/s", "h2d_bytes_per_step": int(h2d_bytes),
                "d2h_bytes_per_step": int(d2h_bytes), "ms_per_step": round(ms_e2e / args.steps, 3),
                "persons": int(P_e2e)},
        "roofline": roofline, "cpu_baseline": cpu, "secondary": secondary,
    }
    emit(line)
    if world > 1:
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------
# CPU side: the oracle port timed on the host cores
# ------------------------------------------------------------------------------------------------
# person-indexed outputs of Model.forward_raw: rows [0, P) are the persons of the step
PER_PERSON = ("det_score", "offset", "loc", "dist_pp", "dist", "rotmat", "rotvec", "shape", "expression", "transl",
              "transl_pelvis", "v3d", "v2d", "j3d", "j2d")
DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(t: dict, P: int, out_dir: str):
    """Writes the arrays a caller of the timed path receives (Model.forward_raw: the detection score map, the
    detected token indices and every per-person output, rows [0, P)) as out_dir/<name>.npy: floating outputs in
    float32, integer ones in float64 (exact).  Above DUMP_LIMIT_BYTES in all, every per-person array keeps the same
    fixed, seeded sample of persons (sample_rows.npy lists them)."""
    import numpy as np
    import torch

    os.makedirs(out_dir, exist_ok=True)
    arrays = {"scores_map": t["scores_map"], "det_idx": t["det_idx"][:, :P]}
    for k in PER_PERSON:
        if t.get(k) is not None:
            arrays[k] = t[k][:P]
    total = sum(v.numel() * 8 for v in arrays.values())
    if total > DUMP_LIMIT_BYTES and P > 0:
        per_row = sum(arrays[k][0].numel() * 8 for k in PER_PERSON if k in arrays)
        keep = max(1, (DUMP_LIMIT_BYTES - arrays["scores_map"].numel() * 8 - arrays["det_idx"].numel() * 8) // per_row)
        rows = torch.randperm(P, generator=torch.Generator().manual_seed(0))[:keep].sort().values
        for k in PER_PERSON:
            if k in arrays:
                arrays[k] = arrays[k][rows.to(arrays[k].device)]
        np.save(os.path.join(out_dir, "sample_rows.npy"), rows.numpy().astype(np.float64))
    for k, v in arrays.items():
        v = v.detach().cpu()
        v = v.to(torch.float32) if v.is_floating_point() else v.to(torch.float64)
        np.save(os.path.join(out_dir, f"{k}.npy"), v.numpy())


def usable_cpus() -> dict:
    """Cores this process may actually use: scheduler affinity AND the cgroup CPU quota (a container with a
    quota of 16 CPUs on a 128-thread host runs 8x oversubscribed with torch.set_num_threads(os.cpu_count()))."""
    info = {"os_cpu_count": os.cpu_count()}
    try:
        info["affinity"] = len(os.sched_getaffinity(0))
    except (AttributeError, OSError):
        info["affinity"] = os.cpu_count()
    quota = None
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            txt = open(path).read().split()
            if path.endswith("cpu.max"):
                if txt[0] != "max":
                    quota = float(txt[0]) / float(txt[1])
            else:
                q = float(txt[0])
                if q > 0:
                    quota = q / float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            break
        except (OSError, ValueError, IndexError):
            continue
    info["cgroup_quota"] = quota
    try:
        import psutil
        info["physical"] = psutil.cpu_count(logical=False)
    except Exception:
        info["physical"] = None
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                info["model"] = line.split(":", 1)[1].strip()
                break
    except OSError:
        pass
    usable = info["affinity"]
    if quota is not None:
        usable = max(1, min(usable, int(math.ceil(quota))))
    info["usable"] = usable
    return info


def pick_cpu_threads(info: dict) -> int:
    """Short probe over {usable, usable/2, physical cores}: one ViT block of the workload's width on one image's
    tokens (Linear + attention + GELU — what the forward is made of; a bare GEMM probe picked 8 of 16 threads on one box
    and 16 on another).  Keeps the fastest; ties within 5 % go to the larger count."""
    import torch

    from oracle import dinov2_ref

    cands = {info["usable"], max(1, info["usable"] // 2)}
    if info.get("physical"):
        cands.add(max(1, min(info["usable"], info["physical"])))
    D, heads, T = 1024, 16, (WORKLOAD["img_size"] // 14) ** 2 + 1
    g = torch.Generator().manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g) * 0.02
    sd = {"b.norm1.weight": torch.ones(D), "b.norm1.bias": torch.zeros(D), "b.norm2.weight": torch.ones(D),
          "b.norm2.bias": torch.zeros(D), "b.attn.qkv.weight": r(3 * D, D), "b.attn.qkv.bias": r(3 * D),
          "b.attn.proj.weight": r(D, D), "b.attn.proj.bias": r(D), "b.ls1.gamma": torch.ones(D),
          "b.ls2.gamma": torch.ones(D), "b.mlp.fc1.weight": r(4 * D, D), "b.mlp.fc1.bias": r(4 * D),
          "b.mlp.fc2.weight": r(D, 4 * D), "b.mlp.fc2.bias": r(D)}
    xx = torch.randn(1, T, D, generator=g)
    best, best_t, probe = None, None, {}
    for n in sorted(cands, reverse=True):
        torch.set_num_threads(n)
        with torch.no_grad():
            dinov2_ref.vit_block(xx, sd, "b.", heads)
            t0 = time.perf_counter()
            for _ in range(2):
                dinov2_ref.vit_block(xx, sd, "b.", heads)
            dt = (time.perf_counter() - t0) / 2
        probe[n] = round(dt * 1e3, 1)  # ms per ViT block
        if best_t is None or dt < 0.95 * best_t:
            best, best_t = n, dt
    info["probe_ms_per_vit_block_by_threads"] = probe
    torch.set_num_threads(best)
    return best


def _cpu_setup(images: int):
    import torch

    from multihmr_b200 import synth
    from oracle import multihmr_ref, smplx_ref

    info = usable_cpus()
    threads = pick_cpu_threads(info)
    info["threads_used"] = threads
    w = WORKLOAD
    sd, bm = build_workload(det_bias=-4.0)
    cfg = multihmr_ref.RefConfig(backbone=w["backbone"], img_size=w["img_size"])
    body = smplx_ref.SMPLXShim(bm, 10)
    x = synth.make_images(images, w["img_size"], seed=w["seed"])
    K = synth.make_cameras(images, w["img_size"], seed=w["seed"])
    idx = synth.make_forced_idx(images, w["img_size"] // 14, min(w["target_persons_per_image"], 4), seed=w["seed"])

    def forward():
        with torch.no_grad():
            return multihmr_ref.model_forward(sd, body, cfg, x, K, idx=idx, is_training=True)

    return forward, info


def _time_cpu(fwd, budget_s: float, max_steps: int):
    """1 warm-up forward, then up to `max_steps` timed forwards within the budget (at least 1)."""
    t0 = time.perf_counter()
    fwd()
    t_warm = time.perf_counter() - t0
    times = []
    while len(times) < max_steps and (not times or sum(times) + t_warm + times[-1] < budget_s):
        t0 = time.perf_counter()
        fwd()
        times.append(time.perf_counter() - t0)
    return t_warm, times


def cpu_baseline(images: int = 1, budget_s: float = 30.0) -> dict:
    fwd, info = _cpu_setup(images)
    t_warm, times = _time_cpu(fwd, budget_s, 3)
    dt = statistics.median(times)
    return {"value": round(images / dt, 5), "unit": "images/s", "cores": info["threads_used"], "kind": "port",
            "host": info,
            "sample": f"{images} image of {WORKLOAD['name']} (CPU images/s is batch-independent), fp32 PyTorch oracle "
                      f"port, 1 warm-up ({t_warm:.1f} s) + {len(times)} timed forwards, median {dt:.2f} s "
                      f"(min {min(times):.2f}, max {max(times):.2f})"}


def run_reference(args):
    """Reference arm: the reference's own algorithm on the host CPU (the Python reference cannot travel to
    the GPU box, so this is the oracle port pinned against it by oracle/make_golden.py)."""
    world, rank, _ = dist_env()
    if rank != 0:
        return
    fwd, info = _cpu_setup(1)
    budget_s = 240.0
    t_warm, times = _time_cpu(fwd, budget_s, max(1, args.steps))
    steps, dt = len(times), sum(times)
    value = steps / dt
    w = WORKLOAD
    sample = (f"each step = 1 image of {w['name']} (of the bs-{w['batch_per_gpu']} workload; CPU images/s is "
              f"batch-independent); 1 warm-up ({t_warm:.1f} s) + {steps} timed steps (capped to ~{budget_s:.0f} s), "
              f"per-step min {min(times):.2f} / median {statistics.median(times):.2f} / max {max(times):.2f} s")
    line = {
        "impl": "reference", "metric": METRIC, "value": round(value, 5), "unit": "images/s", "n_gpus": args.gpus,
        "steps": steps, "warmup": 1, "ms_per_step": round(dt / steps * 1e3, 1), "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
        "config": {"workload": f"{w['name']} batch {w['batch_per_gpu']}/GPU, synthetic {w['img_size']}x{w['img_size']}, "
                               "random-init ViT-L weights (CPU: 1-image sample per step)"},
        "cpu_baseline": {"value": round(value, 5), "unit": "images/s", "cores": info["threads_used"], "kind": "port",
                         "host": info, "sample": sample},
        "e2e": {"value": round(value, 5), "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    emit(line)


_JSON_FD = None


def _reserve_stdout():
    """stdout must carry exactly ONE JSON line: libraries (the NCCL version banner of a communicator, warnings of
    child processes) write to fd 1 behind Python's back, so fd 1 is pointed at stderr for the whole run and the JSON
    line goes to a private duplicate of the original stdout."""
    global _JSON_FD
    sys.stdout.flush()
    _JSON_FD = os.dup(1)
    os.dup2(2, 1)


def emit(line: dict):
    data = (json.dumps(line) + "\n").encode()
    if _JSON_FD is None:
        sys.stdout.write(data.decode())
        sys.stdout.flush()
    else:
        os.write(_JSON_FD, data)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true", help="skip the (slow) CPU oracle leg")
    ap.add_argument("--config", default="c3", choices=sorted(CONFIGS), help="BASELINE.json config (headline: c3)")
    ap.add_argument("--no-secondary", action="store_true", help="skip the short c2 (672x672) leg of the default run")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step as DIR/<name>.npy")
    args = ap.parse_args()
    set_workload(args.config)
    _reserve_stdout()
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
