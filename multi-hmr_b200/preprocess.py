"""Host statement of the reference's image normalisation (utils/image.py:8-24) and the [3][256] table that the
device kernels (`mhmr_op_normalize_u8`, the fused loader of `mhmr_forward_u8`) use to reproduce it bit for bit, the
device letterbox of photos of any size (`ImageOps.contain` + `ImageOps.pad`, demo.py:27-51), and the device decode of
JPEG and PNG files (`Image.open(f).convert("RGB")`, byte for byte, for the files it takes)."""
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


_LUT_CACHE = {}


def device_table(device):
    """The table as a cached device tensor."""
    import torch

    key = (device.type, device.index)
    if key not in _LUT_CACHE:
        _LUT_CACHE[key] = torch.from_numpy(normalize_rgb_table()).to(device)
    return _LUT_CACHE[key]
