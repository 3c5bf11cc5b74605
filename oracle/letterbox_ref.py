"""numpy restatement of `ImageOps.pad(ImageOps.contain(img, (S, S)), (S, S), color=c)` for uint8 RGB photos: the
letterbox of reference demo.py:27-51 (and app.py, the dataset loaders), written from Pillow's documented behaviour of
`contain`, `pad` and the 8-bit BICUBIC `resize`, and checked byte for byte against the installed Pillow by
tests/test_letterbox_cpu.py.  The device kernels of csrc/letterbox.cu implement the same arithmetic.

    contain   target = (S, round(h / w * S)) for a landscape photo, (round(w / h * S), S) for a portrait one (Python
              round, half to even); a square photo goes to (S, S); a zero side is a ValueError; the photo's own size
              is a copy.
    resize    separable, horizontal then vertical, except for a photo more than 100 times taller than wide that gets
              shorter: Image.resize runs the vertical pass first for it.  An axis that keeps its size is skipped, and
              the intermediate image of two passes is uint8.  Per axis (scale = in / out, filterscale = max(scale, 1), support = 2 *
              filterscale, Keys cubic a = -0.5): output i has the window [xmin, xmax) clipped to the input with
              xmin = int(center - support + 0.5), xmax = int(center + support + 0.5), center = (i + 0.5) * scale; its
              weights filter((x - center + 0.5) * (1 / filterscale)) are normalised by their sequential sum in
              double and rounded half away from zero to int32 with 22 fractional bits; a pixel is
              clip8((2^21 + sum pixel * k) >> 22) (arithmetic shift).
    pad       the contained image pasted at round((S - new) * 0.5) (half to even) on the short axis, colour c
              elsewhere.
"""
from __future__ import annotations

import numpy as np

PRECISION_BITS = 22


def contain_size(w: int, h: int, S: int) -> tuple[int, int]:
    """(new_w, new_h) of ImageOps.contain(photo w x h, (S, S)); ValueError when a side rounds to 0."""
    nw, nh = S, S
    if w / h != 1.0:
        if w / h > 1.0:
            nh = round(h / w * S)
        else:
            nw = round(w / h * S)
    if nw <= 0 or nh <= 0:
        raise ValueError(f"a {w} x {h} photo letterboxed into {S} x {S} has a side of 0 pixels")
    return nw, nh


def pad_box(w: int, h: int, S: int) -> tuple[int, int, int, int]:
    """(x0, y0, new_w, new_h): where ImageOps.pad puts the contained photo in the S x S square."""
    nw, nh = contain_size(w, h, S)
    return round((S - nw) * 0.5), round((S - nh) * 0.5), nw, nh


def _bicubic(x: np.ndarray) -> np.ndarray:
    """Keys cubic, a = -0.5, evaluated in the operation order of the 8-bit resampler (no fused multiply-add)."""
    a = -0.5
    x = np.abs(x)
    inner = ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0
    outer = (((x - 5.0) * x + 8.0) * x - 4.0) * a
    return np.where(x < 1.0, inner, np.where(x < 2.0, outer, 0.0))


def coefficients(in_size: int, out_size: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(xmin [out], n [out], k int32 [out, taps]) of one resampling axis; k[i, t] = 0 for t >= n[i]."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    taps = int(np.ceil(support)) * 2 + 1
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)          # astype truncates toward zero
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size)
    n = xmax - xmin
    t = np.arange(taps)
    w = _bicubic(((t[None, :] + xmin[:, None]).astype(np.float64) - center[:, None] + 0.5) * (1.0 / filterscale))
    w = np.where(t[None, :] < n[:, None], w, 0.0)
    ww = np.zeros(out_size)
    for j in range(taps):                                                     # sequential sum, as in C
        ww = ww + w[:, j]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    scaled = w * float(1 << PRECISION_BITS)
    k = np.where(w < 0, (-0.5 + scaled), (0.5 + scaled)).astype(np.int64)   # truncation: half away from zero
    return xmin, n, k.astype(np.int32)


def _resample_axis(img: np.ndarray, out_size: int, axis: int) -> np.ndarray:
    """One 8-bit resampling pass of uint8 HWC `img` along `axis` (1 = width, 0 = height)."""
    in_size = img.shape[axis]
    xmin, n, k = coefficients(in_size, out_size)
    idx = np.minimum(xmin[:, None] + np.arange(k.shape[1])[None, :], in_size - 1)   # taps past n have k = 0
    src = np.moveaxis(img, axis, 0).astype(np.int64)                                 # [in, other, 3]
    acc = np.full((out_size,) + src.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
    for t in range(k.shape[1]):
        acc += src[idx[:, t]] * k[:, t].astype(np.int64)[:, None, None]
    assert np.abs(acc).max(initial=0) < 2 ** 31, "the 8-bit resampler accumulates in int32"
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.ascontiguousarray(np.moveaxis(out, 0, axis))


def resize_bicubic(img: np.ndarray, new_w: int, new_h: int) -> np.ndarray:
    """Image.resize((new_w, new_h), BICUBIC) of a uint8 [H, W, 3] photo."""
    h, w = img.shape[:2]
    out = img
    if h > w * 100 and new_h < h:                      # Image.resize runs the vertical pass first for such photos
        out = _resample_axis(out, new_h, axis=0)
        return _resample_axis(out, new_w, axis=1) if new_w != w else out
    if new_w != w:
        out = _resample_axis(out, new_w, axis=1)
    if new_h != h:
        out = _resample_axis(out, new_h, axis=0)
    return out.copy() if out is img else out


def letterbox(img: np.ndarray, S: int, color: int = 0) -> tuple[np.ndarray, tuple[int, int, int, int]]:
    """(uint8 [S, S, 3], (x0, y0, new_w, new_h)) = ImageOps.pad(ImageOps.contain(img, (S, S)), (S, S), color)."""
    assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3
    h, w = img.shape[:2]
    x0, y0, nw, nh = pad_box(w, h, S)
    out = np.full((S, S, 3), color, dtype=np.uint8)
    out[y0:y0 + nh, x0:x0 + nw] = resize_bicubic(img, nw, nh)
    return out, (x0, y0, nw, nh)
