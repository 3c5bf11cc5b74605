"""Stage-level operators of libmhmr_sm90.so as torch-tensor functions (unit parity + ncu targets).

Each function borrows the tensors' device pointers for the duration of the call and launches on the
current torch CUDA stream.  There is no CPU path: tensors must live on a CUDA device.
"""
from __future__ import annotations

import torch

from ._lib import call, stream

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
    call("mhmr_op_gemm_f16", a, a.stride(0), w, w.stride(0), M, N, K, epilogue, bias, gamma, rowadd, out, out.stride(0),
         rows_in, rows_out, row_off, block_n, stream())
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
    call("mhmr_op_resid_ln_linear_f16", a, a.stride(0), wp, wp.stride(0), bp, ls, x, M, D, Ka, ln_g, ln_b, w, b, N,
         1 if gelu else 0, out, out.stride(0), stream())
    return out


def normalize_u8(img_u8, lut):
    """uint8 [B,H,W,3] -> fp32 [B,3,H,W]: out[b,c,y,x] = lut[c, img[b,y,x,c]] (device-side `normalize_rgb`)."""
    _cuda(img_u8, lut)
    assert img_u8.dtype == torch.uint8 and img_u8.dim() == 4 and img_u8.shape[-1] == 3 and img_u8.is_contiguous()
    assert lut.dtype == torch.float32 and tuple(lut.shape) == (3, 256) and lut.is_contiguous()
    B, H, W, _ = img_u8.shape
    out = torch.empty(B, 3, H, W, device=img_u8.device, dtype=torch.float32)
    call("mhmr_op_normalize_u8", img_u8, lut, out, B, H, W, stream())
    return out


def letterbox_u8(photos, S, pad=0):
    """Photos (a list of uint8 [H, W, 3] CUDA tensors on one device, of any sizes; rows may be padded) -> (uint8
    [B, S, S, 3] on their device, int32 [B, 4] host tensor of (x0, y0, new_w, new_h)): ImageOps.pad(ImageOps.contain(
    photo, (S, S)), (S, S), color=pad) with Pillow's BICUBIC resampler, byte for byte (`mhmr_op_letterbox_u8`)."""
    _cuda(*photos)
    assert len(photos) >= 1, "letterbox needs at least one photo"
    dev = photos[0].device
    desc = torch.empty(len(photos), 4, dtype=torch.int64)
    keep = []  # contiguous copies made here stay alive until the kernels are enqueued
    for i, p in enumerate(photos):
        assert p.dtype == torch.uint8 and p.dim() == 3 and p.shape[2] == 3 and p.device == dev, \
            "uint8 [H, W, 3] photos on one device expected"
        if not (p.stride(2) == 1 and p.stride(1) == 3 and (p.shape[0] == 1 or p.stride(0) >= 3 * p.shape[1])):
            p = p.contiguous()
        keep.append(p)
        desc[i] = torch.tensor([p.data_ptr(), p.shape[0], p.shape[1], p.stride(0) if p.shape[0] > 1 else 3 * p.shape[1]])
    out = torch.empty(len(photos), S, S, 3, dtype=torch.uint8, device=dev)
    boxes = torch.empty(len(photos), 4, dtype=torch.int32)
    with torch.cuda.device(dev):
        call("mhmr_op_letterbox_u8", desc, len(photos), S, pad, out, boxes, stream())
    return out, boxes


def resize_u8(photos, sizes):
    """Photos (a list of uint8 [H, W, 3] CUDA tensors on one device, of any sizes; rows may be padded) and their
    (w, h) output sizes -> uint8 [h, w, 3] tensors on that device: `Image.resize((w, h))` with Pillow's BICUBIC
    resampler, byte for byte (`mhmr_op_resize_u8`)."""
    _cuda(*photos)
    assert len(photos) == len(sizes)
    if not photos:
        return []
    dev = photos[0].device
    desc = torch.empty(len(photos), 8, dtype=torch.int64)
    keep, outs = [], []
    for i, (p, (w, h)) in enumerate(zip(photos, sizes)):
        assert p.dtype == torch.uint8 and p.dim() == 3 and p.shape[2] == 3 and p.device == dev, \
            "uint8 [H, W, 3] photos on one device expected"
        if not (p.stride(2) == 1 and p.stride(1) == 3 and (p.shape[0] == 1 or p.stride(0) >= 3 * p.shape[1])):
            p = p.contiguous()
        keep.append(p)
        o = torch.empty(int(h), int(w), 3, dtype=torch.uint8, device=dev)
        outs.append(o)
        desc[i] = torch.tensor([p.data_ptr(), p.shape[0], p.shape[1], p.stride(0) if p.shape[0] > 1 else 3 * p.shape[1],
                                o.data_ptr(), int(h), int(w), 3 * int(w)])
    with torch.cuda.device(dev):
        call("mhmr_op_resize_u8", desc, len(photos), stream())
    return outs


def jpeg_scan_blocks(h, w, channels, subsampling):
    """Blocks of the scan `jpeg_encode` writes: ceil(W/8) x ceil(H/8) for gray, MCUs x blocks per MCU otherwise."""
    if channels == 1:
        return -(-w // 8) * -(-h // 8)
    hs, vs = (1, 1) if subsampling == 0 else (2, 1) if subsampling == 1 else (2, 2)
    return -(-w // (8 * hs)) * -(-h // (8 * vs)) * (hs * vs + 2)


def jpeg_capacity(h, w, channels, subsampling):
    """Bytes that always hold the file (`mhmr_op_jpeg_encode`'s bound): 1024 + 415 per block of the scan."""
    return 1024 + 415 * jpeg_scan_blocks(h, w, channels, subsampling)


def jpeg_encode(images, qualities, subsamplings):
    """uint8 [H, W, 3] RGB or [H, W] gray CUDA tensors on one device (rows may be padded), with each one's quality
    (1-100) and subsampling (0, 1, 2) -> the JPEG files' bytes Pillow's `save` writes (`mhmr_op_jpeg_encode`).  Every
    output gets the worst-case capacity, so none overflows; the sizes and statuses come back in one host sync and
    the files' bytes in one copy after it."""
    _cuda(*images)
    if not images:
        return []
    dev = images[0].device
    desc = torch.empty(len(images), 9, dtype=torch.int64)
    keep, offs, total = [], [], 0
    for im, s in zip(images, subsamplings):
        ch = 1 if im.dim() == 2 else im.shape[2]
        offs.append((total, jpeg_capacity(im.shape[0], im.shape[1], ch, s)))
        total += offs[-1][1]
    out = torch.empty(total, dtype=torch.uint8, device=dev)
    for i, (im, q, s, (off, cap)) in enumerate(zip(images, qualities, subsamplings, offs)):
        assert im.dtype == torch.uint8 and im.device == dev and (im.dim() == 2 or (im.dim() == 3 and im.shape[2] == 3)), \
            "uint8 [H, W, 3] or [H, W] images on one device expected"
        ch = 1 if im.dim() == 2 else 3
        if not (im.stride(-1) == 1 and (ch == 1 or im.stride(1) == 3) and (im.shape[0] == 1 or im.stride(0) >= ch * im.shape[1])):
            im = im.contiguous()
        keep.append(im)
        desc[i] = torch.tensor([im.data_ptr(), im.shape[0], im.shape[1],
                                im.stride(0) if im.shape[0] > 1 else ch * im.shape[1], ch, int(q), int(s),
                                out.data_ptr() + off, cap])
    B = len(images)
    res = torch.empty(12 * B, dtype=torch.uint8, device=dev)   # int64 sizes, then int32 statuses: one read-back
    with torch.cuda.device(dev):
        call("mhmr_op_jpeg_encode", desc, B, res[:8 * B].view(torch.int64), res[8 * B:].view(torch.int32), stream())
        host = res.cpu()
    sizes, status = host[:8 * B].view(torch.int64).tolist(), host[8 * B:].view(torch.int32).tolist()
    if any(status):
        raise RuntimeError(f"jpeg_encode: a file overflowed its worst-case capacity (statuses {status})")
    with torch.cuda.device(dev):
        data = torch.cat([out[o:o + n] for (o, _), n in zip(offs, sizes)]).cpu().numpy().tobytes()
    files, pos = [], 0
    for n in sizes:
        files.append(data[pos:pos + n])
        pos += n
    return files


def jpeg_info(data):
    """(width, height, components, luma h, luma v, eligible) of a JPEG file's bytes (host only, `mhmr_jpeg_info`):
    eligible files are the ones `jpeg_decode` takes; the sizes are 0 for the others."""
    data = bytes(data)
    info = torch.zeros(6, dtype=torch.int32)
    call("mhmr_jpeg_info", data if data else b"\0", len(data), info)
    return tuple(info.tolist())


def _jpeg_desc(host, dev, spans, sizes, outs):
    assert host.dtype == torch.uint8 and not host.is_cuda and host.is_contiguous()
    assert dev.dtype == torch.uint8 and dev.is_cuda and dev.is_contiguous() and dev.numel() == host.numel()
    desc = torch.zeros(len(spans), 7, dtype=torch.int64)
    for i, ((off, n), (h, w)) in enumerate(zip(spans, sizes)):
        assert 0 <= off and off + n <= host.numel(), "span outside the uploaded bytes"
        o = outs[i] if outs is not None else None
        desc[i] = torch.tensor([host.data_ptr() + off, n, dev.data_ptr() + off, 0 if o is None else o.data_ptr(),
                                0 if o is None else o.stride(0), h, w])
    return desc


def jpeg_decode(host, dev, spans, outs):
    """Decodes JPEG files on the device (`mhmr_op_jpeg_decode`): `host` is the uint8 CPU tensor of the files' bytes
    back to back, `dev` its copy on the device, `spans` each file's (offset, length), `outs` uint8 [H, W, 3] CUDA
    tensors (channels contiguous, rows may be padded).  Returns the device int32 [B] status (0: the photo equals
    Pillow's `convert("RGB")`); nothing waits for the device."""
    _cuda(dev, *outs)
    for o in outs:
        assert o.dtype == torch.uint8 and o.dim() == 3 and o.shape[2] == 3 and o.stride(2) == 1 and o.stride(1) == 3 \
            and o.device == dev.device, "uint8 [H, W, 3] outputs with contiguous pixels on the bytes' device expected"
    desc = _jpeg_desc(host, dev, spans, [tuple(o.shape[:2]) for o in outs], outs)
    status = torch.empty(len(spans), dtype=torch.int32, device=dev.device)
    with torch.cuda.device(dev.device):
        call("mhmr_op_jpeg_decode", desc, len(spans), status, stream())
    return status


def jpeg_plane_blocks(w, h, ncomp, hs, vs):
    """[(blocks wide, blocks high)] of each component's coefficient plane (the padded MCU grid)."""
    if ncomp == 1:
        return [(-(-w // 8), -(-h // 8))]
    mx, my = -(-w // (8 * hs)), -(-h // (8 * vs))
    return [(mx * hs, my * vs), (mx, my), (mx, my)]


def jpeg_coefficients(host, dev, spans, subseq_bits):
    """The entropy stage alone at a given subsequence length (`mhmr_op_jpeg_coefficients`): (per photo, per
    component int16 [blocks high, blocks wide, 64] natural-order coefficients on the device, device int32 [B] status,
    device int32 [1] synchronisation passes)."""
    _cuda(dev)
    infos = [jpeg_info(host[o:o + n].numpy().tobytes()) for o, n in spans]
    assert all(i[5] for i in infos), "every file must be eligible"
    planes = [jpeg_plane_blocks(*i[:5]) for i in infos]
    total = sum(bw * bh * 64 for p in planes for bw, bh in p)
    coefs = torch.empty(total, dtype=torch.int16, device=dev.device)
    status = torch.empty(len(spans), dtype=torch.int32, device=dev.device)
    passes = torch.zeros(1, dtype=torch.int32, device=dev.device)
    desc = _jpeg_desc(host, dev, spans, [(i[1], i[0]) for i in infos], None)
    with torch.cuda.device(dev.device):
        call("mhmr_op_jpeg_coefficients", desc, len(spans), subseq_bits, coefs, status, passes, stream())
    out, pos = [], 0
    for p in planes:
        out.append([])
        for bw, bh in p:
            out[-1].append(coefs[pos:pos + bw * bh * 64].view(bh, bw, 64))
            pos += bw * bh * 64
    return out, status, passes


def png_info(data):
    """(width, height, colour type, eligible) of a PNG file's bytes (host only, `mhmr_png_info`): eligible files are
    the ones `png_decode` takes; the sizes are 0 for the others."""
    data = bytes(data)
    info = torch.zeros(4, dtype=torch.int32)
    call("mhmr_png_info", data if data else b"\0", len(data), info)
    return tuple(info.tolist())


def png_idat(data):
    """The zlib stream of an eligible PNG file: its IDAT payloads back to back."""
    data = memoryview(bytes(data))
    out, pos = [], 8
    while pos + 8 <= len(data):
        n = int.from_bytes(data[pos:pos + 4], "big")
        kind = bytes(data[pos + 4:pos + 8])
        if kind == b"IDAT":
            out.append(data[pos + 8:pos + 8 + n])
        elif out:
            break
        pos += 12 + n
    return b"".join(out)


def png_decode(files, host, dev, spans, outs):
    """Decodes PNG files on the device (`mhmr_op_png_decode`): `files` the files' bytes, `host` the uint8 CPU tensor of
    their zlib streams (`png_idat`) back to back, `dev` its copy on the device, `spans` each stream's (offset, length),
    `outs` uint8 [H, W, 3] CUDA tensors (channels contiguous, rows may be padded).  Returns the device int32 [B] status
    (0: the photo equals Pillow's `convert("RGB")`); nothing waits for the device."""
    _cuda(dev, *outs)
    assert host.dtype == torch.uint8 and not host.is_cuda and host.is_contiguous()
    assert dev.dtype == torch.uint8 and dev.is_cuda and dev.is_contiguous() and dev.numel() == host.numel()
    desc = torch.zeros(len(spans), 8, dtype=torch.int64)
    keep = [bytes(f) for f in files]   # alive until the call returns: the entry reads each file's chunks
    for i, (f, (off, n), o) in enumerate(zip(keep, spans, outs)):
        assert o.dtype == torch.uint8 and o.dim() == 3 and o.shape[2] == 3 and o.stride(2) == 1 and o.stride(1) == 3 \
            and o.device == dev.device, "uint8 [H, W, 3] outputs with contiguous pixels on the bytes' device expected"
        assert 0 <= off and off + n <= host.numel(), "span outside the uploaded bytes"
        fb = torch.frombuffer(bytearray(f), dtype=torch.uint8) if f else torch.zeros(1, dtype=torch.uint8)
        keep.append(fb)
        desc[i] = torch.tensor([fb.data_ptr(), len(f), dev.data_ptr() + off, n, o.data_ptr(),
                                o.stride(0) if o.shape[0] > 1 else 3 * o.shape[1], o.shape[0], o.shape[1]])
    status = torch.empty(len(spans), dtype=torch.int32, device=dev.device)
    with torch.cuda.device(dev.device):
        call("mhmr_op_png_decode", desc, len(spans), status, stream())
    return status


def png_inflate(dev, spans, lengths):
    """Raw zlib streams -> their inflated bytes on the device (`mhmr_op_png_inflate`): `dev` the uint8 CUDA tensor of
    the streams back to back, `spans` each stream's (offset, length), `lengths` each one's expected inflated length.
    Returns (per stream a uint8 CUDA tensor of that length, device int32 [B] status, device int32 [B, 4] counts: chain
    blocks, header candidates, slow-path blocks, inflated bytes)."""
    _cuda(dev)
    assert dev.dtype == torch.uint8 and dev.is_contiguous()
    outs = [torch.empty(max(int(n), 1), dtype=torch.uint8, device=dev.device) for n in lengths]
    desc = torch.zeros(len(spans), 4, dtype=torch.int64)
    for i, ((off, n), o, want) in enumerate(zip(spans, outs, lengths)):
        assert 0 <= off and off + n <= dev.numel() and want >= 1, "span outside the bytes, or an empty output"
        desc[i] = torch.tensor([dev.data_ptr() + off, n, o.data_ptr(), want])
    status = torch.empty(len(spans), dtype=torch.int32, device=dev.device)
    counts = torch.empty(len(spans), 4, dtype=torch.int32, device=dev.device)
    with torch.cuda.device(dev.device):
        call("mhmr_op_png_inflate", desc, len(spans), status, counts, stream())
    return outs, status, counts


def attention(qkv, B, T, D, out=None):
    """qkv [B*T, 3*D] fp16 -> out [B*T, D] fp16, heads of 64 dims, softmax(q k^T / 8) v per image."""
    _cuda(qkv)
    assert qkv.dtype == torch.float16 and qkv.shape == (B * T, 3 * D) and qkv.stride(1) == 1
    if out is None:
        out = torch.empty(B * T, D, device=qkv.device, dtype=torch.float16)
    call("mhmr_op_attention", qkv, qkv.stride(0), out, out.stride(0), B, T, D, stream())
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
    call("mhmr_op_skinny_linear", x, x.stride(0), count, max_persons, K, w, w.stride(0), bias, w.shape[0], g, b, eps,
         act, resid, resid.stride(0) if resid is not None else 0, out, out.stride(0), cols, stream())
    return out


def hph_self_attn(qkv, det_b, img_off, count, max_persons, heads, out=None):
    """qkv [P, >= 3 * heads * 32] -> out [P, heads * 32]: attention among the persons of each image."""
    _cuda(qkv, det_b, img_off, count)
    _f32(qkv)
    _i32(det_b, img_off, count)
    if out is None:
        out = torch.zeros(max_persons, heads * 32, device=qkv.device)
    call("mhmr_op_hph_self_attn", qkv, qkv.stride(0), det_b, img_off, count, max_persons, heads, out, out.stride(0),
         stream())
    return out


def hph_cross_attn(q, kv, k_col, v_col, det_b, count, max_persons, heads, N, out=None):
    """q [P, >= heads * 32], kv [B * N, ldkv] -> out [P, heads * 32]: person p attends to image det_b[p]'s rows."""
    _cuda(q, kv, det_b, count)
    _f32(q, kv)
    _i32(det_b, count)
    if out is None:
        out = torch.zeros(max_persons, heads * 32, device=q.device)
    call("mhmr_op_hph_cross_attn", q, q.stride(0), kv, kv.stride(0), k_col, v_col, det_b, count, max_persons, heads, N,
         out, out.stride(0), stream())
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
    call("mhmr_op_detect", scores, B, res, nms_k, thresh, max_persons,
         *(o[k] for k in ("scores_out", "det_b", "det_y", "det_x", "det_score", "count", "count_clamped", "img_off")),
         stream())
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
    call("mhmr_op_person_post", dec, dec.stride(0), num_betas, offset, K, K.shape[0], det_b, det_y, det_x, count, Pm,
         focal_norm,
         *(o[k] for k in ("rotmat", "rotvec", "shape", "expression", "dist_pp", "dist", "loc", "transl", "K_det")),
         stream())
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
    call("mhmr_op_anny_person_post", hid, D, w2, b2, fov_max, K, B, img_size, o["fov"], o["K_regressed"], o["K_use"],
         rot6d, rot6d.stride(0), J, useful, shape, shape.shape[1], offset, dist_pp, det_b, det_y, det_x, count, Pm,
         *(o[k] for k in ("rotmat", "rotmat_homo", "rotvec", "dist", "loc", "transl", "K_det")), stream())
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
    call("mhmr_op_refine_chain", depth, D, count, x.shape[0], *(layers[k] for k in keys), o16, R, rowidx, x, stream())
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
    call("mhmr_op_im2col_patch14", None if u8 else img, img if u8 else None, lut, B, S, A, A.stride(0), stream())
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
    call("mhmr_op_layernorm", x, xlo, gamma, beta, out16, out16.stride(0) if out16 is not None else 0, out32,
         out32.stride(0) if out32 is not None else 0, M, D, eps, rows_in, skip, stream())


def split_rowstats(x, hi, lo, stats):
    """x fp32 [M, D] -> hi, lo fp16 [M, >= D] (x = hi + lo) and stats fp32 [M, slots, 2] (slot 0 = (sum, sumsq))."""
    _cuda(x, hi, lo, stats)
    _contig(x, stats)
    assert hi.dtype == lo.dtype == torch.float16 and hi.stride() == lo.stride() and hi.stride(1) == 1
    M, D = x.shape
    call("mhmr_op_split_rowstats", x, hi, lo, hi.stride(0), stats, stats.shape[1], M, D, stream())


def fold_ln_linear(w, bias, ln_g, ln_b):
    """Folds LayerNorm(ln_g, ln_b) into the Linear (w [N, K], bias): returns (W16 fp16 [N, K], bias2 fp32 [N])."""
    _cuda(w, bias, ln_g, ln_b)
    _contig(w, bias, ln_g, ln_b)
    N, K = w.shape
    w16 = torch.empty(N, K, device=w.device, dtype=torch.float16)
    b2 = torch.empty(N, device=w.device)
    call("mhmr_op_fold_ln_linear", w, bias, ln_g, ln_b, w16, b2, N, K, stream())
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
    call("mhmr_op_gemm_internal", a, a.stride(0), w, w.stride(0), M, N, K, epilogue, bias, gamma, hi, lo,
         hi.stride(0) if hi is not None else 0, stats, stats.shape[1] if stats is not None else 0, rowadd, rows_in,
         rows_out, row_off, out, out.stride(0) if out is not None else 0, block_n, 0 if m_run is None else m_run,
         stream())
    return out


def camera_ctx(K, freqs, ctx, res, col0, pad_cols):
    """K^-1 (returned, [B, 3, 3]) and the fp16 camera features of every cell into ctx[:, col0 : col0 + pad_cols]."""
    _cuda(K, freqs, ctx)
    _contig(K, freqs)
    assert ctx.dtype == torch.float16 and ctx.stride(1) == 1
    B = K.shape[0]
    kinv = torch.empty(B, 3, 3, device=K.device)
    call("mhmr_op_camera_ctx", K, B, freqs, kinv, ctx, ctx.stride(0), res, col0, pad_cols, stream())
    return kinv


def rowdot_sigmoid(hid, D, w, b, scores, logits=None, clamp=True):
    """scores[r] = sigmoid(hid[r, :D] . w + b) (clamped to [1e-4, 1 - 1e-4] with `clamp`) for r < scores.numel()."""
    _cuda(hid, w, b, scores, logits)
    _contig(w, b, scores, logits)
    assert hid.dtype == torch.float16 and hid.stride(1) == 1
    call("mhmr_op_rowdot_sigmoid", hid, hid.stride(0), w, b, scores, logits, 1 if clamp else 0, scores.numel(), D,
         stream())


def person_gather(z32, kinv, freqs, cq_x, cq_y, cv_x, cv_y, det_b, det_y, det_x, count, max_persons, res, zc, query,
                  vals, xr=None, norm=(None, None)):
    """Per-person feature rows zc [Pm, D], queries and values [Pm, ldq] (pitch = query's stride)."""
    _cuda(z32, kinv, freqs, cq_x, cq_y, cv_x, cv_y, zc, query, vals, xr, *norm)
    _f32(z32, kinv, cq_x, cq_y, cv_x, cv_y, zc, query, vals, xr)
    _contig(z32, kinv, freqs, cq_x, cq_y, cv_x, cv_y, zc, xr, *norm)
    _i32(det_b, det_y, det_x, count)
    assert query.stride() == vals.stride()
    D = z32.shape[-1]
    call("mhmr_op_person_gather", z32, xr, norm[0], norm[1], kinv, freqs, cq_x, cq_y, cv_x, cv_y, det_b, det_y, det_x,
         count, max_persons, res, D, zc, query, vals, query.stride(0), stream())


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
    call("mhmr_op_refine_prepare", None if u8 else img, img if u8 else None, lut, S, rowadd, xr.shape[1], det_b, det_y,
         det_x, count, max_persons, n_cls, cls_pos, rows_out, rowidx, patch, patch.stride(0), xr, stream())


def kv_add_rows(kv, dkv, det_b, det_y, det_x, count, max_persons, res):
    """kv[b*res*res + cell, :ncols] += dkv[p] once per distinct cell of the persons p < count (in place)."""
    _cuda(kv, dkv, det_b, det_y, det_x, count)
    _f32(kv, dkv)
    _contig(dkv)
    _i32(det_b, det_y, det_x, count)
    call("mhmr_op_kv_add_rows", kv, kv.stride(0), dkv, dkv.shape[1], det_b, det_y, det_x, count, max_persons, res,
         stream())


def cls_gather(x, T, B, D, xlo=None):
    """Rows b*T (b < B) of the residual stream x [B*T, ld] (fp32, or the fp16 hi plane with `xlo`) -> fp32 [B, D]."""
    _cuda(x, xlo)
    assert x.stride(1) == 1 and (xlo is None or xlo.stride() == x.stride())
    out = torch.empty(B, D, device=x.device)
    call("mhmr_op_cls_gather", x, xlo, x.stride(0), T, B, D, out, stream())
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
        call("mhmr_op_vit_stream", model._handle, x, B, layers, out, stream())
    return out


def anny_gather(z32, pos, det_b, det_y, det_x, count, max_persons, res, zc, xa, xr=None, norm=(None, None)):
    """Anny decoder inputs: zc [Pm, D] (bulk row, or the final norm of xr), xa [Pm, dim] = pos[cell]."""
    _cuda(z32, pos, zc, xa, xr, *norm)
    _contig(z32, pos, zc, xa, xr, *norm)
    _i32(det_b, det_y, det_x, count)
    call("mhmr_op_anny_gather", z32, xr, norm[0], norm[1], pos, det_b, det_y, det_x, count, max_persons, res,
         z32.shape[-1], xa.shape[1], zc, xa, stream())


def anny_place(bone_poses, transl, K_det, center, v3d, j3d, j2d, transl_pelvis, v2d=None):
    """Places P bodies: v3d [P, V, 3] in place, j3d [P, J, 3] from bone_poses [P, J, 4, 4], v2d / j2d, transl_pelvis."""
    _cuda(bone_poses, transl, K_det, v3d, j3d, j2d, transl_pelvis, v2d)
    _contig(bone_poses, transl, K_det, v3d, j3d, j2d, transl_pelvis, v2d)
    P, J = bone_poses.shape[:2]
    V = v3d.shape[1]
    call("mhmr_op_anny_place", bone_poses, transl, K_det, center, P, V, J, v3d, j3d, v2d, j2d, transl_pelvis, stream())
