"""Fixtures of the JPEG encoder tests (CPU and device): Pillow's bytes and the images that reach every path of
libjpeg-turbo's baseline encoder."""
import io

import numpy as np
from PIL import Image

# (subsampling passed to save, gray?) cases: 4:4:4, 4:2:2, 4:2:0, Pillow's default, and gray with each setting
SETTINGS = [(0, False), (1, False), (2, False), (None, False), (None, True), (0, True), (1, True), (2, True)]


def pillow_jpeg(img, quality=75, subsampling=None, **options):
    kw = dict(options, quality=quality)
    if subsampling is not None:
        kw["subsampling"] = subsampling
    buf = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(img)).save(buf, "JPEG", **kw)
    return buf.getvalue()


def image(kind, h, w, seed=0, gray=False):
    """uint8 [h, w, 3] (or [h, w]) test image of one kind."""
    rng = np.random.default_rng(seed + 1000 * h + w)
    shape = (h, w) if gray else (h, w, 3)
    if kind == "noise":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if kind == "flat0":
        return np.zeros(shape, np.uint8)
    if kind == "flat255":
        return np.full(shape, 255, np.uint8)
    y, x = np.mgrid[:h, :w]
    if kind == "gradient":
        planes = [(x * 7 + y * 3) % 256, (x * y) % 256, (255 - x * 5 + y) % 256]
    elif kind == "checker":   # pixel checkerboard: the largest AC coefficients
        planes = [((x + y) % 2) * 255, ((x + y + 1) % 2) * 255, ((x // 2 + y) % 2) * 255]
    elif kind == "blocks":    # 0 / 255 alternating 8 x 8 blocks: DC differences of category 11 at q100
        planes = [((x // 8 + y // 8) % 2) * 255, ((x // 8 + y // 8 + 1) % 2) * 255, ((x // 16 + y // 8) % 2) * 255]
    elif kind == "basis":     # one high DCT basis function per block: long zero runs (ZRL)
        base = 128 + 100 * np.cos(np.pi * (2 * (x % 8) + 1) * 7 / 16) * np.cos(np.pi * (2 * (y % 8) + 1) * 6 / 16)
        planes = [base, 255 - base, base]
    else:
        raise ValueError(kind)
    img = np.stack(planes, -1).astype(np.uint8)
    return img[..., 0].copy() if gray else img


KINDS = ["noise", "flat0", "flat255", "gradient", "checker", "blocks", "basis"]
