"""Stage-level operators of libmhmr_sm90.so as torch-tensor functions (unit parity + ncu targets).

Each function borrows the tensors' device pointers for the duration of the call and launches on the
current torch CUDA stream.  There is no CPU path: tensors must live on a CUDA device.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import c_int, c_int64, check, ptr, stream_ptr

EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_RELU_F16, EPI_LS_RESID_F32, EPI_ROWADD_F32, EPI_BIAS_F32 = range(6)


def _cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("multihmr_b200 ops need CUDA tensors (no CPU fallback)")


def gemm_f16(a, w, epilogue, out, bias=None, gamma=None, rowadd=None, rows_in=0, rows_out=0, row_off=0,
             block_n=256):
    """out = epilogue(a[M,K] @ w[N,K]^T); a, w fp16 with contiguous K. `out` is written in place."""
    _cuda(a, w, out, bias, gamma, rowadd)
    assert a.dtype == torch.float16 and w.dtype == torch.float16
    assert a.stride(1) == 1 and w.stride(1) == 1 and out.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    lib = _lib.load()
    rc = lib.mhmr_op_gemm_f16(ptr(a), c_int64(a.stride(0)), ptr(w), c_int64(w.stride(0)), c_int(M), c_int(N),
                              c_int(K), c_int(epilogue), ptr(bias), ptr(gamma), ptr(rowadd), ptr(out),
                              c_int64(out.stride(0)), c_int(rows_in), c_int(rows_out), c_int(row_off),
                              c_int(block_n), stream_ptr())
    check(rc, "mhmr_op_gemm_f16")
    return out


def resid_ln_linear_f16(a, wp, bp, ls, x, ln_g, ln_b, w, b, gelu=False):
    """One dinov2 Block seam with the LayerNorm folded into both GEMMs (see include/mhmr.h):
    x += ls * (a @ wp^T + bp) in place (fp32 [M, D]); returns fp16 act(LayerNorm(x) @ w^T + b) of shape [M, N]."""
    _cuda(a, wp, bp, ls, x, ln_g, ln_b, w, b)
    assert a.dtype == torch.float16 and wp.dtype == torch.float16 and x.dtype == torch.float32
    assert w.dtype == torch.float32 and a.stride(1) == 1 and wp.stride(1) == 1 and x.is_contiguous() and w.is_contiguous()
    M, Ka = a.shape
    D = wp.shape[0]
    N = w.shape[0]
    assert x.shape == (M, D) and w.shape == (N, D)
    out = torch.empty(M, N, device=a.device, dtype=torch.float16)
    rc = _lib.load().mhmr_op_resid_ln_linear_f16(
        ptr(a), c_int64(a.stride(0)), ptr(wp), c_int64(wp.stride(0)), ptr(bp), ptr(ls), ptr(x), c_int(M), c_int(D),
        c_int(Ka), ptr(ln_g), ptr(ln_b), ptr(w), ptr(b), c_int(N), c_int(1 if gelu else 0), ptr(out),
        c_int64(out.stride(0)), stream_ptr())
    check(rc, "mhmr_op_resid_ln_linear_f16")
    return out


def normalize_u8(img_u8, lut):
    """uint8 [B,H,W,3] -> fp32 [B,3,H,W]: out[b,c,y,x] = lut[c, img[b,y,x,c]] (device-side `normalize_rgb`)."""
    _cuda(img_u8, lut)
    assert img_u8.dtype == torch.uint8 and img_u8.dim() == 4 and img_u8.shape[-1] == 3 and img_u8.is_contiguous()
    assert lut.dtype == torch.float32 and tuple(lut.shape) == (3, 256) and lut.is_contiguous()
    B, H, W, _ = img_u8.shape
    out = torch.empty(B, 3, H, W, device=img_u8.device, dtype=torch.float32)
    rc = _lib.load().mhmr_op_normalize_u8(ptr(img_u8), ptr(lut), ptr(out), c_int(B), c_int(H), c_int(W), stream_ptr())
    check(rc, "mhmr_op_normalize_u8")
    return out


def attention(qkv, B, T, D, out=None):
    """qkv [B*T, 3*D] fp16 -> out [B*T, D] fp16, heads of 64 dims, softmax(q k^T / 8) v per image."""
    _cuda(qkv)
    assert qkv.dtype == torch.float16 and qkv.shape == (B * T, 3 * D) and qkv.stride(1) == 1
    if out is None:
        out = torch.empty(B * T, D, device=qkv.device, dtype=torch.float16)
    lib = _lib.load()
    rc = lib.mhmr_op_attention(ptr(qkv), c_int64(qkv.stride(0)), ptr(out), c_int64(out.stride(0)), c_int(B),
                               c_int(T), c_int(D), stream_ptr())
    check(rc, "mhmr_op_attention")
    return out
