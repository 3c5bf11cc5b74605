"""Host statement of the reference's image normalisation (utils/image.py:8-24) and the [3][256] table that the
device kernels (`mhmr_op_normalize_u8`, the fused loader of `mhmr_forward_u8`) use to reproduce it bit for bit, the
device letterbox of photos of any size (`ImageOps.contain` + `ImageOps.pad`, demo.py:27-51) and resize
(`Image.resize`), the device decode of JPEG and PNG files (`Image.open(f).convert("RGB")`, byte for byte, for the files
it takes), and the device JPEG encode (`Image.save(f, "JPEG")`, byte for byte)."""
from __future__ import annotations

import numpy as np

IMG_NORM_MEAN = [0.485, 0.456, 0.406]       # utils/image.py:8
IMG_NORM_STD = [0.229, 0.224, 0.225]        # utils/image.py:9


def normalize_rgb(img: np.ndarray, imagenet_normalization: bool = True) -> np.ndarray:
    """uint8 HWC -> float32 CHW (utils/image.py:12-24)."""
    img = img.astype(np.float32) / 255.0
    img = np.transpose(img, (2, 0, 1))
    if imagenet_normalization:
        img = (img - np.asarray(IMG_NORM_MEAN).reshape(3, 1, 1)) / np.asarray(IMG_NORM_STD).reshape(3, 1, 1)
    return img.astype(np.float32)


def normalize_rgb_table() -> np.ndarray:
    """[3, 256] fp32: `normalize_rgb` of every uint8 value in every channel (the table of the device kernels)."""
    ramp = np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, axis=2)
    return np.ascontiguousarray(normalize_rgb(ramp)[:, 0, :])


def letterbox(photos, img_size: int, color: int = 0):
    """`ImageOps.pad(ImageOps.contain(photo, (S, S)), (S, S), color)` of every photo, on the device and byte for byte
    (csrc/letterbox.cu; the arithmetic is restated in oracle/letterbox_ref.py).  `photos` is a list of uint8 [H, W, 3]
    RGB tensors of any sizes: CUDA tensors are read where they are, host tensors are uploaded (pinned, non-blocking)
    to the current CUDA device.  Returns (uint8 [B, S, S, 3] on the device, int32 [B, 4] host tensor of (x0, y0,
    new_w, new_h), the box of each photo in the square).  The uint8 batch is what `Model.forward` / `forward_model`
    take through the fused loader."""
    import torch

    from . import ops

    dev = next((p.device for p in photos if p.is_cuda), torch.device("cuda"))
    photos = [p if p.is_cuda else p.pin_memory().to(dev, non_blocking=True) for p in photos]
    return ops.letterbox_u8(photos, img_size, color)


def upload_bytes(blobs, device):
    """The byte strings back to back in one pinned host tensor and one non-blocking upload: (host, device copy,
    [(offset, length)])."""
    import torch

    spans, off = [], 0
    for b in blobs:
        spans.append((off, len(b)))
        off += len(b)
    host = torch.empty(max(off, 1), dtype=torch.uint8, pin_memory=True)
    view = host.numpy()
    for (o, n), b in zip(spans, blobs):
        view[o:o + n] = np.frombuffer(b, dtype=np.uint8)
    return host, host.to(device, non_blocking=True), spans


def decode_jpeg(blobs, device):
    """JPEG files' bytes -> (uint8 [H, W, 3] RGB device photos, ok flags), byte for byte `Image.open(f).convert("RGB")`
    (csrc/jpeg.cu; the arithmetic is restated in oracle/jpeg_ref.py).  Eligible files (`ops.jpeg_info`) are decoded in
    one call; a photo is None and its flag False when the file is not eligible, has more pixels than Pillow's
    `Image.MAX_IMAGE_PIXELS` (Pillow warns about such files or refuses them as decompression bombs; nothing is
    allocated for them here), or its entropy data was flagged (the caller decodes those with Pillow).  The bytes go up
    in one pinned upload; the statuses come back in one host sync."""
    import torch
    from PIL import Image

    from . import ops

    device = torch.device(device)
    limit = Image.MAX_IMAGE_PIXELS
    infos = [ops.jpeg_info(b) for b in blobs]
    idx = [i for i, info in enumerate(infos) if info[5] and (limit is None or info[0] * info[1] <= limit)]
    photos, ok = [None] * len(blobs), [False] * len(blobs)
    if not idx:
        return photos, ok
    with torch.cuda.device(device):
        host, dev, spans = upload_bytes([blobs[i] for i in idx], device)
        outs = [torch.empty((infos[i][1], infos[i][0], 3), dtype=torch.uint8, device=device) for i in idx]
        status = ops.jpeg_decode(host, dev, spans, outs).cpu().tolist()
    for i, o, s in zip(idx, outs, status):
        if s == 0:
            photos[i], ok[i] = o, True
    return photos, ok


def decode_png(blobs, device):
    """PNG files' bytes -> (uint8 [H, W, 3] RGB device photos, ok flags), byte for byte `Image.open(f).convert("RGB")`
    (csrc/png.cu; the arithmetic is restated in oracle/png_ref.py).  The contract of `decode_jpeg`: eligible files
    (`ops.png_info`) are decoded in one call; a photo is None and its flag False when the file is not eligible, has
    more pixels than Pillow's `Image.MAX_IMAGE_PIXELS`, or was flagged on the device (the caller decodes those with
    Pillow).  Each file's zlib stream (its IDAT payloads) goes up in one pinned upload; the statuses come back in one
    host sync."""
    import torch
    from PIL import Image

    from . import ops

    device = torch.device(device)
    limit = Image.MAX_IMAGE_PIXELS
    infos = [ops.png_info(b) for b in blobs]
    idx = [i for i, info in enumerate(infos) if info[3] and (limit is None or info[0] * info[1] <= limit)]
    photos, ok = [None] * len(blobs), [False] * len(blobs)
    if not idx:
        return photos, ok
    with torch.cuda.device(device):
        host, dev, spans = upload_bytes([ops.png_idat(blobs[i]) for i in idx], device)
        outs = [torch.empty((infos[i][1], infos[i][0], 3), dtype=torch.uint8, device=device) for i in idx]
        status = ops.png_decode([blobs[i] for i in idx], host, dev, spans, outs).cpu().tolist()
    for i, o, s in zip(idx, outs, status):
        if s == 0:
            photos[i], ok[i] = o, True
    return photos, ok


def resize(photos, sizes):
    """`Image.resize((w, h))` (BICUBIC) of every uint8 [H, W, 3] RGB photo to its own (w, h), on the device and byte
    for byte (csrc/letterbox.cu's coefficient rows and passes, without the pad).  CUDA tensors are read where they
    are, host tensors are uploaded (pinned, non-blocking) to the current CUDA device.  Returns uint8 [h, w, 3] device
    tensors; nothing waits for the device."""
    import torch

    from . import ops

    dev = next((p.device for p in photos if p.is_cuda), torch.device("cuda"))
    photos = [p if p.is_cuda else p.pin_memory().to(dev, non_blocking=True) for p in photos]
    for w, h in sizes:
        if w < 1 or h < 1:
            raise ValueError("height and width must be > 0")   # as Image.resize
    return ops.resize_u8(photos, sizes)


_SUBSAMPLING = {-1: None, 0: 0, 1: 1, 2: 2, "4:4:4": 0, "4:2:2": 1, "4:2:0": 2}


def _device_setting(img, quality, subsampling):
    """(quality, subsampling) of the device encode for one save, or None when Pillow writes it."""
    if not (hasattr(img, "is_cuda") and img.is_cuda and str(img.dtype) == "torch.uint8"):
        return None
    if not (img.dim() == 2 or (img.dim() == 3 and img.shape[2] == 3)):
        return None                                       # modes other than L and RGB
    if not (1 <= img.shape[0] <= 65535 and 1 <= img.shape[1] <= 65535):
        return None
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)):
        return None
    if subsampling is None or isinstance(subsampling, (str, int, np.integer)) and subsampling in _SUBSAMPLING:
        s = _SUBSAMPLING[subsampling] if subsampling is not None else None
    else:
        return None
    q = 75 if quality == -1 else min(max(int(quality), 1), 100)   # Pillow's default, then libjpeg's clamp
    return q, (2 if img.dim() == 3 else 0) if s is None else s


def _pillow_jpeg(img, quality, subsampling, options):
    import io

    from PIL import Image

    arr = img.cpu().numpy() if hasattr(img, "cpu") else np.asarray(img)
    kw = dict(options, quality=quality)
    if subsampling is not None:
        kw["subsampling"] = subsampling
    buf = io.BytesIO()
    Image.fromarray(arr).save(buf, "JPEG", **kw)
    return buf.getvalue()


def encode_jpeg(images, quality=75, subsampling=None, **options):
    """The bytes of `Image.fromarray(img).save(f, "JPEG", quality=quality, subsampling=subsampling, **options)` for
    every image, byte for byte.  `images` are uint8 [H, W, 3] RGB or [H, W] gray tensors (rows may be padded);
    `quality` and `subsampling` are one value for all or a list with one per image.  Quality is clamped to 1-100 as
    libjpeg does (-1 is Pillow's default, 75); subsampling 0, 1, 2 (or "4:4:4", "4:2:2", "4:2:0") is 4:4:4, 4:2:2,
    4:2:0, and None (or -1) Pillow's default, 4:2:0 for RGB.  CUDA images with these settings are encoded on the
    device in one call (csrc/jpeg_encode.cu; the arithmetic is restated in oracle/jpeg_encode_ref.py), which waits
    for the device once; any other image, setting or save option (`optimize`, `progressive`, `qtables`, `dpi`,
    `exif`, ...) goes to Pillow unchanged."""
    from . import ops

    n = len(images)
    qs = list(quality) if isinstance(quality, (list, tuple)) else [quality] * n
    ss = list(subsampling) if isinstance(subsampling, (list, tuple)) else [subsampling] * n
    assert len(qs) == n and len(ss) == n, "one quality and one subsampling per image"
    out = [None] * n
    dev = {}
    for i, (img, q, s) in enumerate(zip(images, qs, ss)):
        setting = None if options else _device_setting(img, q, s)
        if setting is None:
            out[i] = _pillow_jpeg(img, q, s, options)
        else:
            dev.setdefault(img.device, []).append((i, setting))
    for device, items in dev.items():
        files = ops.jpeg_encode([images[i] for i, _ in items], [q for _, (q, _) in items],
                                [s for _, (_, s) in items])
        for (i, _), f in zip(items, files):
            out[i] = f
    return out


_LUT_CACHE = {}


def device_table(device):
    """The table as a cached device tensor."""
    import torch

    key = (device.type, device.index)
    if key not in _LUT_CACHE:
        _LUT_CACHE[key] = torch.from_numpy(normalize_rgb_table()).to(device)
    return _LUT_CACHE[key]
