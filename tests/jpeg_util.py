"""Seeded photos, Pillow encodings and header edits for the JPEG decode tests (oracle/jpeg_ref.py, csrc/jpeg.cu)."""
import io
import os

import numpy as np

GOLDEN = [os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f)
          for f in ("170149601_13aa4e4483_c.jpg", "3692623581_aca6eb02d4_e.jpg")]
MODES = ("L", "444", "422", "420")
_SUB = {"444": 0, "422": 1, "420": 2}


def photo(w: int, h: int, seed: int = 0) -> np.ndarray:
    """uint8 [h, w, 3]: ramps, a sharp diagonal edge and noise, so every coefficient band is busy."""
    rng = np.random.default_rng(seed + 7919 * w + 104729 * h)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([x * 255.0 / max(w - 1, 1), y * 255.0 / max(h - 1, 1), ((x + 2 * y) % 23 < 11) * 200.0], -1)
    return np.clip(base + rng.normal(0, 40, (h, w, 3)), 0, 255).astype(np.uint8)


def encode(img: np.ndarray, mode: str, **kw) -> bytes:
    """Pillow's JPEG of `img` in mode L (gray) or 444 / 422 / 420 (YCbCr subsampling)."""
    from PIL import Image, ImageFile

    b = io.BytesIO()
    keep = ImageFile.MAXBLOCK   # optimised noisy photos can exceed the buffer Pillow sizes for them
    ImageFile.MAXBLOCK = max(keep, 4 * img.shape[0] * img.shape[1] + 65536)
    try:
        if mode == "L":
            Image.fromarray(img[:, :, 0]).save(b, format="JPEG", **kw)
        else:
            Image.fromarray(img).save(b, format="JPEG", subsampling=_SUB[mode], **kw)
    finally:
        ImageFile.MAXBLOCK = keep
    return b.getvalue()


def pillow_rgb(data: bytes) -> np.ndarray:
    from PIL import Image

    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB")).copy()


def segment(data: bytes, marker: int) -> int:
    """Offset of the first segment with this marker byte (0xC0 for SOF0, ...) before the scan."""
    pos = 2
    while data[pos + 1] != marker:
        assert data[pos + 1] != 0xDA, f"no 0x{marker:02x} segment"
        pos += 2 + (data[pos + 2] << 8 | data[pos + 3])
    return pos


def edit(data: bytes, at: int, values) -> bytes:
    out = bytearray(data)
    out[at:at + len(values)] = bytes(values)
    return bytes(out)


def insert_segment(data: bytes, marker: int, payload: bytes) -> bytes:
    """A segment inserted right after SOI."""
    n = len(payload) + 2
    return data[:2] + bytes([0xFF, marker, n >> 8, n & 255]) + payload + data[2:]


def ecs_span(data: bytes):
    """(start, end) of the entropy-coded segment of a Pillow JPEG (after the SOS header, before EOI)."""
    sos = segment(data, 0xDA)
    return sos + 2 + (data[sos + 2] << 8 | data[sos + 3]), len(data) - 2


def saturating_quantisers() -> bytes:
    """A full-contrast q100 4:4:4 stream whose quantisation tables are rewritten to 255: its dequantised coefficients
    leave int16, where libjpeg-turbo's SIMD IDCT (which Pillow runs) saturates and its C IDCT wraps."""
    img = np.repeat(((np.indices((32, 32)).sum(0) % 2) * 255).astype(np.uint8)[:, :, None], 3, 2)
    data = encode(img, "444", quality=100)
    at = segment(data, 0xDB)
    n = data[at + 2] << 8 | data[at + 3]
    edited = bytearray(data)
    for t in range(at + 4, at + 2 + n, 65):
        edited[t + 1:t + 65] = b"\xff" * 64
    return bytes(edited)


def bomb_header() -> bytes:
    """A small 4:4:4 JPEG whose SOF claims 65535 x 65535 pixels: eligible by its header, a decompression bomb to
    Pillow."""
    data = encode(photo(16, 16), "444", quality=90)
    sof = segment(data, 0xC0)
    return edit(data, sof + 5, [0xFF, 0xFF, 0xFF, 0xFF])
