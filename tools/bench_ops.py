"""Micro-benchmarks of the stage-level operators on one GPU (CUDA events, L2-flushed)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multihmr_b200 import ops  # noqa: E402


def timeit(fn, iters=10, warmup=3, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def bench_gemm(dev, flush):
    res = []
    for (M, N, K, epi, bn) in [
        (32776, 3072, 1024, ops.EPI_BIAS_F16, 256),
        (32776, 3072, 1024, ops.EPI_BIAS_F16, 512),
        (32776, 1024, 1024, ops.EPI_LS_RESID_F32, 256),
        (32776, 1024, 1024, ops.EPI_LS_RESID_F32, 512),
        (32776, 4096, 1024, ops.EPI_BIAS_GELU_F16, 256),
        (32776, 4096, 1024, ops.EPI_BIAS_GELU_F16, 512),
        (32776, 1024, 4096, ops.EPI_LS_RESID_F32, 256),
        (32776, 1024, 4096, ops.EPI_LS_RESID_F32, 512),
        (32768, 1024, 1152, ops.EPI_BIAS_F32, 256),
        (32768, 1024, 1152, ops.EPI_BIAS_F32, 512),
    ]:
        a = torch.randn(M, K, device=dev).half()
        w = (torch.randn(N, K, device=dev) * 0.03).half()
        bias = torch.randn(N, device=dev)
        gamma = torch.rand(N, device=dev)
        f16 = epi in (ops.EPI_BIAS_F16, ops.EPI_BIAS_GELU_F16, ops.EPI_BIAS_RELU_F16)
        out = torch.zeros(M, N, device=dev, dtype=torch.float16 if f16 else torch.float32)
        ms = timeit(lambda: ops.gemm_f16(a, w, epi, out, bias=bias, gamma=gamma, block_n=bn), flush=flush)
        ms_ref = timeit(lambda: torch.matmul(a, w.t()), flush=flush)
        tf = 2.0 * M * N * K / ms / 1e9
        res.append(dict(op="gemm", M=M, N=N, K=K, epi=epi, bn=bn, ms=round(ms, 4), tflops=round(tf, 1),
                        cublas_ms=round(ms_ref, 4), cublas_tflops=round(2.0 * M * N * K / ms_ref / 1e9, 1)))
        print(res[-1], flush=True)
    return res


def bench_attention(dev, flush):
    res = []
    for (B, T, D) in [(8, 4097, 1024), (4, 2305, 1024)]:
        qkv = torch.randn(B * T, 3 * D, device=dev).half()
        out = torch.empty(B * T, D, device=dev, dtype=torch.float16)
        q, k, v = qkv.view(B, T, 3, D // 64, 64).permute(2, 0, 3, 1, 4)
        ref = torch.nn.functional.scaled_dot_product_attention(q.float(), k.float(), v.float()).transpose(1, 2).reshape(B * T, D) if B * T < 20000 else None
        ms = timeit(lambda: ops.attention(qkv, B, T, D, out=out), flush=flush)
        err = (out.float() - ref).abs().max().item() if ref is not None else None
        res.append(dict(op="attention", B=B, T=T, D=D, ms=round(ms, 4),
                        tflops=round(4.0 * B * T * T * D / ms / 1e9, 1), max_err=err))
        print(res[-1], flush=True)
    return res


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="gemm")
    ap.add_argument("--out", default="bench_ops.json")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    out = {}
    for what in args.what.split(","):
        out[what] = globals()["bench_" + what](dev, flush)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(out, open(args.out, "w"), indent=1)
