"""Builds libmhmr_sm90.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

Usage: python multi-hmr_b200/build.py [--force] [--verbose]
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libmhmr_sm90.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_hash(src: str) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    for f in [src] + sorted(x for x in os.listdir(CSRC) if x.endswith((".cuh", ".h"))):
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    with open(os.path.join(HERE, "..", "include", "mhmr.h"), "rb") as fh:
        h.update(fh.read())
    return h.hexdigest()


def _compile(src: str, force: bool, verbose: bool) -> str:
    obj = os.path.join(BUILD, src.replace(".cu", ".o"))
    stamp = obj + ".hash"
    want = _deps_hash(src)
    if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == want:
        return obj
    cmd = [NVCC, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(obj + ".log", "w") as fh:
        fh.write(log)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{log}")
    if verbose:
        print(f"== {src}\n{log}")
    with open(stamp, "w") as fh:
        fh.write(want)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, force, verbose), srcs))
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("link failed:\n" + res.stdout + res.stderr)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
