"""Stage-level operators of libmhmr_sm90.so as torch-tensor functions (unit parity + ncu targets).

Each function borrows the tensors' device pointers for the duration of the call and launches on the
current torch CUDA stream.  There is no CPU path: tensors must live on a CUDA device.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import c_float, c_int, c_int64, check, ptr, stream_ptr

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


# ---- person-decoder kernels: `count` is a device int32 tensor [1] (<= max_persons), read on the device -----------
def _f32(*ts):
    for t in ts:
        assert t is None or (t.dtype == torch.float32 and (t.dim() == 1 or t.stride(-1) == 1)), "fp32 rows expected"


def _i32(*ts):
    for t in ts:
        assert t.dtype == torch.int32 and t.is_contiguous(), "int32 contiguous tensor expected"


def skinny_linear(x, count, max_persons, K, w, out, bias=None, ln=None, act=0, resid=None, cols=0):
    """out[p, :N] = resid[p] + act(LN(x[p, :K]) @ w[:, :K]^T + bias) for p < count, N = w.shape[0]; row pitches are
    the tensors' strides.  ln = (gamma, beta, eps) or None; act 0 none, 1 ReLU, 2 erf GELU; out may be resid;
    cols 16 / 32 columns per CTA, 0 = the engine's choice."""
    _cuda(x, count, w, out, bias, resid)
    _f32(x, w, out, bias, resid)
    _i32(count)
    g, b, eps = ln if ln is not None else (None, None, 0.0)
    rc = _lib.load().mhmr_op_skinny_linear(
        ptr(x), c_int(x.stride(0)), ptr(count), c_int(max_persons), c_int(K), ptr(w), c_int(w.stride(0)), ptr(bias),
        c_int(w.shape[0]), ptr(g), ptr(b), c_float(eps), c_int(act), ptr(resid),
        c_int(resid.stride(0) if resid is not None else 0), ptr(out), c_int(out.stride(0)), c_int(cols), stream_ptr())
    check(rc, "mhmr_op_skinny_linear")
    return out


def hph_self_attn(qkv, det_b, img_off, count, max_persons, heads, out=None):
    """qkv [P, >= 3 * heads * 32] -> out [P, heads * 32]: attention among the persons of each image."""
    _cuda(qkv, det_b, img_off, count)
    _f32(qkv)
    _i32(det_b, img_off, count)
    if out is None:
        out = torch.zeros(max_persons, heads * 32, device=qkv.device)
    rc = _lib.load().mhmr_op_hph_self_attn(ptr(qkv), c_int(qkv.stride(0)), ptr(det_b), ptr(img_off), ptr(count),
                                           c_int(max_persons), c_int(heads), ptr(out), c_int(out.stride(0)), stream_ptr())
    check(rc, "mhmr_op_hph_self_attn")
    return out


def hph_cross_attn(q, kv, k_col, v_col, det_b, count, max_persons, heads, N, out=None):
    """q [P, >= heads * 32], kv [B * N, ldkv] -> out [P, heads * 32]: person p attends to image det_b[p]'s rows."""
    _cuda(q, kv, det_b, count)
    _f32(q, kv)
    _i32(det_b, count)
    if out is None:
        out = torch.zeros(max_persons, heads * 32, device=q.device)
    rc = _lib.load().mhmr_op_hph_cross_attn(ptr(q), c_int(q.stride(0)), ptr(kv), c_int64(kv.stride(0)), c_int(k_col),
                                            c_int(v_col), ptr(det_b), ptr(count), c_int(max_persons), c_int(heads),
                                            c_int(N), ptr(out), c_int(out.stride(0)), stream_ptr())
    check(rc, "mhmr_op_hph_cross_attn")
    return out


def detect(scores, nms_k, thresh, max_persons):
    """scores [B, res, res] fp32 -> dict(scores_out, det_b, det_y, det_x, det_score, count, count_clamped, img_off)."""
    _cuda(scores)
    assert scores.dtype == torch.float32 and scores.is_contiguous() and scores.dim() == 3
    B, res, _ = scores.shape
    dev = scores.device
    cap = max(max_persons, 1)
    o = {"scores_out": torch.empty_like(scores), "det_b": torch.full((cap,), -1, dtype=torch.int32, device=dev),
         "det_y": torch.full((cap,), -1, dtype=torch.int32, device=dev),
         "det_x": torch.full((cap,), -1, dtype=torch.int32, device=dev),
         "det_score": torch.full((cap,), -1.0, device=dev), "count": torch.full((1,), -1, dtype=torch.int32, device=dev),
         "count_clamped": torch.full((1,), -1, dtype=torch.int32, device=dev),
         "img_off": torch.full((B + 1,), -1, dtype=torch.int32, device=dev)}
    rc = _lib.load().mhmr_op_detect(ptr(scores), c_int(B), c_int(res), c_int(nms_k), c_float(thresh), c_int(max_persons),
                                    *(ptr(o[k]) for k in ("scores_out", "det_b", "det_y", "det_x", "det_score", "count",
                                                          "count_clamped", "img_off")), stream_ptr())
    check(rc, "mhmr_op_detect")
    return o


def _zeros(dev, *shape):
    return torch.zeros(*shape, device=dev)


def person_post(dec, num_betas, offset, K, det_b, det_y, det_x, count, max_persons, focal_norm):
    """SMPL-X per-person outputs from the decoder rows dec [P, >= 331 + num_betas]; returns a dict of [max_persons, ...]
    tensors (rows >= count stay zero)."""
    _cuda(dec, offset, K, det_b, det_y, det_x, count)
    _f32(dec, offset, K)
    _i32(det_b, det_y, det_x, count)
    assert offset.is_contiguous() and K.is_contiguous()
    Pm, dev = max_persons, dec.device
    o = {"rotmat": _zeros(dev, Pm, 53, 3, 3), "rotvec": _zeros(dev, Pm, 53, 3), "shape": _zeros(dev, Pm, num_betas),
         "expression": _zeros(dev, Pm, 10), "dist_pp": _zeros(dev, Pm), "dist": _zeros(dev, Pm),
         "loc": _zeros(dev, Pm, 2), "transl": _zeros(dev, Pm, 3), "K_det": _zeros(dev, Pm, 3, 3)}
    rc = _lib.load().mhmr_op_person_post(
        ptr(dec), c_int(dec.stride(0)), c_int(num_betas), ptr(offset), ptr(K),
        c_int(K.shape[0]), ptr(det_b), ptr(det_y), ptr(det_x), ptr(count), c_int(Pm), c_float(focal_norm),
        *(ptr(o[k]) for k in ("rotmat", "rotvec", "shape", "expression", "dist_pp", "dist", "loc", "transl", "K_det")),
        stream_ptr())
    check(rc, "mhmr_op_person_post")
    return o


def anny_person_post(hid, w2, b2, fov_max, K, img_size, rot6d, J, useful, shape, offset, dist_pp, det_b, det_y, det_x,
                     count, max_persons):
    """Anny camera (hid [B, D] -> fov, K_regressed, K_use; K None = regressed) and per-person outputs from rot6d
    [P, >= 6 J]; `shape` [P, num_betas] is replaced by its sigmoid in place.  Returns a dict."""
    _cuda(hid, w2, b2, fov_max, K, rot6d, useful, shape, offset, dist_pp, det_b, det_y, det_x, count)
    _f32(hid, w2, b2, fov_max, K, rot6d, useful, shape, offset, dist_pp)
    _i32(det_b, det_y, det_x, count)
    assert hid.is_contiguous() and shape.is_contiguous() and offset.is_contiguous() and dist_pp.is_contiguous()
    assert K is None or K.is_contiguous()
    B, D = hid.shape
    Pm, dev = max_persons, hid.device
    o = {"fov": _zeros(dev, B), "K_regressed": _zeros(dev, B, 3, 3), "K_use": _zeros(dev, B, 3, 3),
         "rotmat": _zeros(dev, Pm, J, 3, 3), "rotmat_homo": _zeros(dev, Pm, J, 4, 4), "rotvec": _zeros(dev, Pm, J, 3),
         "dist": _zeros(dev, Pm), "loc": _zeros(dev, Pm, 2), "transl": _zeros(dev, Pm, 3), "K_det": _zeros(dev, Pm, 3, 3)}
    rc = _lib.load().mhmr_op_anny_person_post(
        ptr(hid), c_int(D), ptr(w2), ptr(b2), ptr(fov_max), ptr(K), c_int(B),
        c_int(img_size), ptr(o["fov"]), ptr(o["K_regressed"]), ptr(o["K_use"]), ptr(rot6d), c_int(rot6d.stride(0)),
        c_int(J), ptr(useful), ptr(shape), c_int(shape.shape[1]), ptr(offset), ptr(dist_pp),
        ptr(det_b), ptr(det_y), ptr(det_x), ptr(count), c_int(Pm),
        *(ptr(o[k]) for k in ("rotmat", "rotmat_homo", "rotvec", "dist", "loc", "transl", "K_det")), stream_ptr())
    check(rc, "mhmr_op_anny_person_post")
    o["shape"] = shape
    return o


def refine_chain(layers, o16, rowidx, count, x):
    """Central-stream refinement of x [max_persons, D] in place through len(layers) dinov2 blocks.  `layers` maps
    Wproj, bproj, ls1, ln2_g, ln2_b, Wfc1, bfc1, Wfc2, bfc2, ls2 to fp32 tensors stacked over the blocks; o16 is the
    fp16 attention output [depth, R, D] of the bulk pass, rowidx [max_persons] int32 its row per person."""
    keys = ("Wproj", "bproj", "ls1", "ln2_g", "ln2_b", "Wfc1", "bfc1", "Wfc2", "bfc2", "ls2")
    _cuda(o16, rowidx, count, x, *(layers[k] for k in keys))
    _f32(x, *(layers[k] for k in keys))
    _i32(rowidx, count)
    assert o16.dtype == torch.float16 and o16.is_contiguous() and x.is_contiguous()
    assert all(layers[k].is_contiguous() for k in keys)
    depth, R, D = o16.shape
    assert x.shape[1] == D and rowidx.shape[0] >= x.shape[0]
    rc = _lib.load().mhmr_op_refine_chain(c_int(depth), c_int(D), ptr(count), c_int(x.shape[0]),
                                          *(ptr(layers[k]) for k in keys), ptr(o16), c_int64(R), ptr(rowidx), ptr(x),
                                          stream_ptr())
    check(rc, "mhmr_op_refine_chain")
    return x


# ---- backbone entry, folded LayerNorm and the gathers of the heads -------------------------------------------------
EPI_LS_RESID_SPLIT, EPI_LN_BIAS_F16, EPI_LN_GELU_F16, EPI_ROWADD_F16 = range(6, 10)


def _contig(*ts):
    for t in ts:
        assert t is None or t.is_contiguous(), "contiguous tensor expected"


def im2col_patch14(img, A, lut=None):
    """Patch rows of the patch-embed GEMM into A [B*(S/14)^2, ldA] fp16 (columns >= 588 untouched): img fp32
    [B, 3, S, S], or uint8 [B, S, S, 3] with its [3, 256] table `lut`."""
    _cuda(img, A, lut)
    _contig(img, lut)
    assert A.dtype == torch.float16 and A.stride(1) == 1
    u8 = img.dtype == torch.uint8
    assert (lut is not None) == u8 and (img.dtype == torch.float32 or u8)
    B, S = img.shape[0], img.shape[2] if u8 else img.shape[3]
    rc = _lib.load().mhmr_op_im2col_patch14(ptr(None if u8 else img), ptr(img if u8 else None), ptr(lut), c_int(B),
                                            c_int(S), ptr(A), c_int(A.stride(0)), stream_ptr())
    check(rc, "mhmr_op_im2col_patch14")
    return A


def layernorm(x, gamma, beta, out16=None, out32=None, eps=1e-6, rows_in=0, skip=0, xlo=None):
    """LayerNorm of the rows of x [M, D] (fp32, or the fp16 hi plane with `xlo` the lo plane) into out16 and / or
    out32 (row pitches = their strides); rows_in > 0 drops rows t < skip of every group of rows_in."""
    _cuda(x, xlo, gamma, beta, out16, out32)
    _contig(x, xlo, gamma, beta)
    assert (xlo is None and x.dtype == torch.float32) or (x.dtype == xlo.dtype == torch.float16)
    for o in (out16, out32):
        assert o is None or o.stride(1) == 1
    M, D = x.shape
    rc = _lib.load().mhmr_op_layernorm(ptr(x), ptr(xlo), ptr(gamma), ptr(beta), ptr(out16),
                                       c_int64(out16.stride(0) if out16 is not None else 0), ptr(out32),
                                       c_int64(out32.stride(0) if out32 is not None else 0), c_int(M), c_int(D),
                                       c_float(eps), c_int(rows_in), c_int(skip), stream_ptr())
    check(rc, "mhmr_op_layernorm")


def split_rowstats(x, hi, lo, stats):
    """x fp32 [M, D] -> hi, lo fp16 [M, >= D] (x = hi + lo) and stats fp32 [M, slots, 2] (slot 0 = (sum, sumsq))."""
    _cuda(x, hi, lo, stats)
    _contig(x, stats)
    assert hi.dtype == lo.dtype == torch.float16 and hi.stride() == lo.stride() and hi.stride(1) == 1
    M, D = x.shape
    rc = _lib.load().mhmr_op_split_rowstats(ptr(x), ptr(hi), ptr(lo), c_int64(hi.stride(0)), ptr(stats),
                                            c_int(stats.shape[1]), c_int(M), c_int(D), stream_ptr())
    check(rc, "mhmr_op_split_rowstats")


def fold_ln_linear(w, bias, ln_g, ln_b):
    """Folds LayerNorm(ln_g, ln_b) into the Linear (w [N, K], bias): returns (W16 fp16 [N, K], bias2 fp32 [N])."""
    _cuda(w, bias, ln_g, ln_b)
    _contig(w, bias, ln_g, ln_b)
    N, K = w.shape
    w16 = torch.empty(N, K, device=w.device, dtype=torch.float16)
    b2 = torch.empty(N, device=w.device)
    rc = _lib.load().mhmr_op_fold_ln_linear(ptr(w), ptr(bias), ptr(ln_g), ptr(ln_b), ptr(w16), ptr(b2), c_int(N),
                                            c_int(K), stream_ptr())
    check(rc, "mhmr_op_fold_ln_linear")
    return w16, b2


def gemm_internal(a, w, epilogue, block_n, out=None, bias=None, gamma=None, hi=None, lo=None, stats=None, rowadd=None,
                  rows_in=0, rows_out=0, row_off=0, m_run=None):
    """The GEMM a [M, K] @ w [N, K]^T with any epilogue kind: 0-5 as gemm_f16, 6 split residual update of (hi, lo) +
    stats, 7 / 8 folded-LN consumer from stats, 9 fp16 row add; stats fp32 [M, slots, 2].  m_run < M runs a plan
    built for M rows on its first m_run rows, as the engine does at a smaller batch."""
    _cuda(a, w, out, bias, gamma, hi, lo, stats, rowadd)
    _contig(stats, rowadd, bias, gamma)
    assert a.dtype == w.dtype == torch.float16 and a.stride(1) == 1 and w.stride(1) == 1
    assert out is None or (out.dtype in (torch.float16, torch.float32) and out.stride(1) == 1)
    assert hi is None or (hi.dtype == lo.dtype == torch.float16 and hi.stride() == lo.stride() and hi.stride(1) == 1)
    M, K = a.shape
    N = w.shape[0]
    rc = _lib.load().mhmr_op_gemm_internal(
        ptr(a), c_int64(a.stride(0)), ptr(w), c_int64(w.stride(0)), c_int(M), c_int(N), c_int(K), c_int(epilogue),
        ptr(bias), ptr(gamma), ptr(hi), ptr(lo), c_int64(hi.stride(0) if hi is not None else 0), ptr(stats),
        c_int(stats.shape[1] if stats is not None else 0), ptr(rowadd), c_int(rows_in), c_int(rows_out),
        c_int(row_off), ptr(out), c_int64(out.stride(0) if out is not None else 0), c_int(block_n),
        c_int(0 if m_run is None else m_run), stream_ptr())
    check(rc, "mhmr_op_gemm_internal")
    return out


def camera_ctx(K, freqs, ctx, res, col0, pad_cols):
    """K^-1 (returned, [B, 3, 3]) and the fp16 camera features of every cell into ctx[:, col0 : col0 + pad_cols]."""
    _cuda(K, freqs, ctx)
    _contig(K, freqs)
    assert ctx.dtype == torch.float16 and ctx.stride(1) == 1
    B = K.shape[0]
    kinv = torch.empty(B, 3, 3, device=K.device)
    rc = _lib.load().mhmr_op_camera_ctx(ptr(K), c_int(B), ptr(freqs), ptr(kinv), ptr(ctx), c_int64(ctx.stride(0)),
                                        c_int(res), c_int(col0), c_int(pad_cols), stream_ptr())
    check(rc, "mhmr_op_camera_ctx")
    return kinv


def rowdot_sigmoid(hid, D, w, b, scores, logits=None, clamp=True):
    """scores[r] = sigmoid(hid[r, :D] . w + b) (clamped to [1e-4, 1 - 1e-4] with `clamp`) for r < scores.numel()."""
    _cuda(hid, w, b, scores, logits)
    _contig(w, b, scores, logits)
    assert hid.dtype == torch.float16 and hid.stride(1) == 1
    rc = _lib.load().mhmr_op_rowdot_sigmoid(ptr(hid), c_int64(hid.stride(0)), ptr(w), ptr(b), ptr(scores), ptr(logits),
                                            c_int(1 if clamp else 0), c_int(scores.numel()), c_int(D), stream_ptr())
    check(rc, "mhmr_op_rowdot_sigmoid")


def person_gather(z32, kinv, freqs, cq_x, cq_y, cv_x, cv_y, det_b, det_y, det_x, count, max_persons, res, zc, query,
                  vals, xr=None, norm=(None, None)):
    """Per-person feature rows zc [Pm, D], queries and values [Pm, ldq] (pitch = query's stride)."""
    _cuda(z32, kinv, freqs, cq_x, cq_y, cv_x, cv_y, zc, query, vals, xr, *norm)
    _f32(z32, kinv, cq_x, cq_y, cv_x, cv_y, zc, query, vals, xr)
    _contig(z32, kinv, freqs, cq_x, cq_y, cv_x, cv_y, zc, xr, *norm)
    _i32(det_b, det_y, det_x, count)
    assert query.stride() == vals.stride()
    D = z32.shape[-1]
    rc = _lib.load().mhmr_op_person_gather(
        ptr(z32), ptr(xr), ptr(norm[0]), ptr(norm[1]), ptr(kinv), ptr(freqs), ptr(cq_x), ptr(cq_y), ptr(cv_x),
        ptr(cv_y), ptr(det_b), ptr(det_y), ptr(det_x), ptr(count), c_int(max_persons), c_int(res), c_int(D), ptr(zc),
        ptr(query), ptr(vals), c_int(query.stride(0)), stream_ptr())
    check(rc, "mhmr_op_person_gather")


def refine_prepare(img, rowadd, det_b, det_y, det_x, count, max_persons, rowidx, patch, xr, lut=None, n_cls=0,
                   cls_pos=None, rows_out=None):
    """Refinement inputs of n_cls cls rows and max_persons person rows: rowidx int32, patch fp32 [R, ldp], xr [R, D];
    img fp32 [B, 3, S, S] or uint8 [B, S, S, 3] with `lut`."""
    _cuda(img, rowadd, lut, cls_pos, rowidx, patch, xr, rows_out)
    _contig(img, rowadd, lut, cls_pos, rowidx, xr)
    _i32(det_b, det_y, det_x, count)
    assert patch.stride(1) == 1
    u8 = img.dtype == torch.uint8
    S = img.shape[2] if u8 else img.shape[3]
    rc = _lib.load().mhmr_op_refine_prepare(
        ptr(None if u8 else img), ptr(img if u8 else None), ptr(lut), c_int(S), ptr(rowadd), c_int(xr.shape[1]),
        ptr(det_b), ptr(det_y), ptr(det_x), ptr(count), c_int(max_persons), c_int(n_cls), ptr(cls_pos), ptr(rows_out),
        ptr(rowidx), ptr(patch), c_int(patch.stride(0)), ptr(xr), stream_ptr())
    check(rc, "mhmr_op_refine_prepare")


def kv_add_rows(kv, dkv, det_b, det_y, det_x, count, max_persons, res):
    """kv[b*res*res + cell, :ncols] += dkv[p] once per distinct cell of the persons p < count (in place)."""
    _cuda(kv, dkv, det_b, det_y, det_x, count)
    _f32(kv, dkv)
    _contig(dkv)
    _i32(det_b, det_y, det_x, count)
    rc = _lib.load().mhmr_op_kv_add_rows(ptr(kv), c_int64(kv.stride(0)), ptr(dkv), c_int(dkv.shape[1]), ptr(det_b),
                                         ptr(det_y), ptr(det_x), ptr(count), c_int(max_persons), c_int(res),
                                         stream_ptr())
    check(rc, "mhmr_op_kv_add_rows")


def cls_gather(x, T, B, D, xlo=None):
    """Rows b*T (b < B) of the residual stream x [B*T, ld] (fp32, or the fp16 hi plane with `xlo`) -> fp32 [B, D]."""
    _cuda(x, xlo)
    assert x.stride(1) == 1 and (xlo is None or xlo.stride() == x.stride())
    out = torch.empty(B, D, device=x.device)
    rc = _lib.load().mhmr_op_cls_gather(ptr(x), ptr(xlo), c_int64(x.stride(0)), c_int(T), c_int(B), c_int(D), ptr(out),
                                        stream_ptr())
    check(rc, "mhmr_op_cls_gather")
    return out


def vit_stream(model, x, layers):
    """The residual stream of `model`'s bulk pass after its patch embedding and first `layers` blocks: x [B,3,S,S]
    (normalised fp32) -> fp32 [B, T, D], cls row first.  On the folded-LayerNorm path it is hi + lo of the two-term
    fp16 stream the next block reads."""
    model.finalize()
    x = x.to(model.device, dtype=torch.float32).contiguous()
    B = x.shape[0]
    out = torch.empty(B, 1 + model.res * model.res, model.embed_dim, device=model.device)
    with torch.cuda.device(model.device):
        rc = _lib.load().mhmr_op_vit_stream(model._handle, ptr(x), c_int(B), c_int(layers), ptr(out), stream_ptr())
    check(rc, "mhmr_op_vit_stream")
    return out


def anny_gather(z32, pos, det_b, det_y, det_x, count, max_persons, res, zc, xa, xr=None, norm=(None, None)):
    """Anny decoder inputs: zc [Pm, D] (bulk row, or the final norm of xr), xa [Pm, dim] = pos[cell]."""
    _cuda(z32, pos, zc, xa, xr, *norm)
    _contig(z32, pos, zc, xa, xr, *norm)
    _i32(det_b, det_y, det_x, count)
    rc = _lib.load().mhmr_op_anny_gather(ptr(z32), ptr(xr), ptr(norm[0]), ptr(norm[1]), ptr(pos), ptr(det_b),
                                         ptr(det_y), ptr(det_x), ptr(count), c_int(max_persons), c_int(res),
                                         c_int(z32.shape[-1]), c_int(xa.shape[1]), ptr(zc), ptr(xa), stream_ptr())
    check(rc, "mhmr_op_anny_gather")


def anny_place(bone_poses, transl, K_det, center, v3d, j3d, j2d, transl_pelvis, v2d=None):
    """Places P bodies: v3d [P, V, 3] in place, j3d [P, J, 3] from bone_poses [P, J, 4, 4], v2d / j2d, transl_pelvis."""
    _cuda(bone_poses, transl, K_det, v3d, j3d, j2d, transl_pelvis, v2d)
    _contig(bone_poses, transl, K_det, v3d, j3d, j2d, transl_pelvis, v2d)
    P, J = bone_poses.shape[:2]
    V = v3d.shape[1]
    rc = _lib.load().mhmr_op_anny_place(ptr(bone_poses), ptr(transl), ptr(K_det), c_int(center), c_int(P), c_int(V),
                                        c_int(J), ptr(v3d), ptr(j3d), ptr(v2d), ptr(j2d), ptr(transl_pelvis),
                                        stream_ptr())
    check(rc, "mhmr_op_anny_place")
