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


def bit_readers(data: bytes):
    """The bit readers of the restatement's sequential decode, one per restart interval it decoded, as they stopped:
    `pos` is where the interval's last block ended (its 1-padding follows) or where an anomaly stopped the decode,
    `n` the interval's destuffed bits."""
    from oracle import jpeg_ref as jr

    made = []

    class Recorder(jr._Bits):
        def __init__(self, buf):
            super().__init__(buf)
            made.append(self)

    keep, jr._Bits = jr._Bits, Recorder
    try:
        jr.decode_coefficients(data, jr.parse(data))
    finally:
        jr._Bits = keep
    return made


def _kept_offsets(data: bytes):
    """Per restart interval, the file offset of each destuffed byte (the 0xFF of a stuffed pair stands for it)."""
    s, e = ecs_span(data)
    out, cur, i = [], [], s
    while i < e:
        if data[i] == 0xFF:
            if data[i + 1] == 0:
                cur.append(i)
            else:
                out.append(cur)
                cur = []
            i += 2
            continue
        cur.append(i)
        i += 1
    out.append(cur)
    return out


def corruptions(rng, data):
    """Seeded corruptions of a clean file's entropy-coded segment: (kind, bytes).  Bit flips, truncation (EOI kept),
    and with restart markers: one dropped or swapped, non-0xFF garbage before one (libjpeg skips it), an empty interval
    (two adjacent RSTn), a truncation exactly at an interval boundary, bit flips confined to an interval's 1-padding
    (nothing reads those bits: the file must stay exact), and a duplicated RSTn once the index has wrapped past 7."""
    s, e = ecs_span(data)
    out = []
    for _ in range(12):
        b = bytearray(data)
        for _ in range(int(rng.integers(1, 4))):
            i = int(rng.integers(s, e))
            b[i] ^= 1 << int(rng.integers(0, 8))
        out.append(("flip", bytes(b)))
    for _ in range(4):
        cut = int(rng.integers(s, e))
        out.append(("truncate", data[:cut] + b"\xff\xd9"))
    ends, kept = [b.pos for b in bit_readers(data)], _kept_offsets(data)
    padded = [i for i, (end, k) in enumerate(zip(ends, kept)) if end < 8 * len(k)]
    for _ in range(2 if padded else 0):
        iv = padded[int(rng.integers(0, len(padded)))]
        p = int(rng.integers(ends[iv], 8 * len(kept[iv])))
        out.append(("padding flip", edit(data, kept[iv][p >> 3], [data[kept[iv][p >> 3]] ^ (0x80 >> (p & 7))])))
    rst = [i for i in range(s, e - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7]
    if len(rst) >= 2:
        i = rst[int(rng.integers(0, len(rst)))]
        out.append(("drop rst", data[:i] + data[i + 2:]))
        i, j = rst[0], rst[1]
        out.append(("swap rst", edit(edit(data, i + 1, [data[j + 1]]), j + 1, [data[i + 1]])))
        i = rst[int(rng.integers(0, len(rst)))]
        garbage = bytes(int(v) for v in rng.integers(0, 255, int(rng.integers(1, 6))))
        out.append(("garbage before rst", data[:i] + garbage + data[i:]))
        k = int(rng.integers(0, len(rst) - 1))
        out.append(("empty interval", data[:rst[k] + 2] + data[rst[k + 1]:]))
        out.append(("truncate at rst", data[:rst[int(rng.integers(0, len(rst)))]] + b"\xff\xd9"))
    if len(rst) >= 9:
        i = rst[int(rng.integers(8, len(rst)))]
        out.append(("duplicate wrapped rst", data[:i + 2] + data[i:]))
    return out


def bomb_header() -> bytes:
    """A small 4:4:4 JPEG whose SOF claims 65535 x 65535 pixels: eligible by its header, a decompression bomb to
    Pillow."""
    data = encode(photo(16, 16), "444", quality=90)
    sof = segment(data, 0xC0)
    return edit(data, sof + 5, [0xFF, 0xFF, 0xFF, 0xFF])
