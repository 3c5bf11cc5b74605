"""Shared PNG test material: the writer's zlib stream families, PNG files from Pillow, OpenCV, zlib strategies and
the writer, Pillow's verdict on a file, and a seeded corruption generator."""
from __future__ import annotations

import io
import os
import random
import struct
import zlib

import numpy as np

import png_writer as pw

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODES = {0: "L", 2: "RGB", 3: "P", 4: "LA", 6: "RGBA"}


def pillow(data: bytes):
    """Pillow's `Image.open(f).convert("RGB")` as uint8 [H, W, 3], or the exception it raises."""
    from PIL import Image

    try:
        with Image.open(io.BytesIO(data)) as im:
            return np.asarray(im.convert("RGB"))
    except Exception as err:   # noqa: BLE001
        return err


def photo(rng, H, W, C):
    """Smooth content with noise: every filter type is chosen by the encoders somewhere."""
    y, x = np.mgrid[0:H, 0:W]
    base = np.stack([(x * (3 + c) + y * (5 - c)) for c in range(C)], axis=-1)
    return ((base + rng.integers(0, 24, (H, W, C))) % 256).astype(np.uint8)


def pillow_png(px, ctype, **save):
    from PIL import Image

    if ctype == 3:
        im = Image.fromarray(px[..., 0], "L").convert("P")
        im.putpalette((np.arange(768) * 7 % 256).astype(np.uint8).tobytes())
    else:
        im = Image.fromarray(px if px.shape[2] > 1 else px[..., 0], MODES[ctype])
    b = io.BytesIO()
    im.save(b, "PNG", **save)
    return b.getvalue()


def cv2_png(px):
    import cv2

    ok, buf = cv2.imencode(".png", np.ascontiguousarray(px[..., ::-1]))
    assert ok
    return buf.tobytes()


def golden_photos():
    from PIL import Image

    return [np.asarray(Image.open(os.path.join(GOLDEN, f)).convert("RGB"))
            for f in sorted(os.listdir(GOLDEN)) if f.endswith(".jpg")]


def palette_bytes(n):
    return ((np.arange(3 * n) * 37 + 11) % 256).astype(np.uint8).tobytes()


def pillow_files(seed=0, sizes=range(1, 18)):
    """(name, file) of every eligible colour type at sizes 1 x 1 .. 17 x 17, 1-row and 1-column images, Pillow levels
    0-9, zlib strategies, every filter forced per row, OpenCV-written files and the golden photos as PNG."""
    rng = np.random.default_rng(seed)
    out = []
    for ct, C in ((0, 1), (2, 3), (3, 1), (4, 2), (6, 4)):
        for s in sizes:
            out.append((f"pil-ct{ct}-{s}x{s}", pillow_png(photo(rng, s, s, C), ct)))
        out.append((f"pil-ct{ct}-1x29", pillow_png(photo(rng, 1, 29, C), ct)))
        out.append((f"pil-ct{ct}-29x1", pillow_png(photo(rng, 29, 1, C), ct)))
        for ft in range(5):
            px = photo(rng, 9, 11, C)
            pal = palette_bytes(200) if ct == 3 else None
            out.append((f"filter{ft}-ct{ct}", pw.make_png(px, ct, filters=[ft] * 9, palette=pal)))
        px = photo(rng, 10, 7, C)
        out.append((f"mixed-filters-ct{ct}", pw.make_png(px, ct, filters=[y % 5 for y in range(10)],
                                                       palette=palette_bytes(256) if ct == 3 else None)))
    for lvl in range(10):
        out.append((f"pil-level{lvl}", pillow_png(photo(rng, 23, 31, 3), 2, compress_level=lvl)))
    for name, st in (("filtered", zlib.Z_FILTERED), ("huffman", zlib.Z_HUFFMAN_ONLY), ("rle", zlib.Z_RLE),
                     ("fixed", zlib.Z_FIXED)):
        out.append((f"zlib-{name}", pw.make_png(photo(rng, 21, 19, 3), 2, filters=[y % 5 for y in range(21)],
                                                 strategy=st)))
    # Paeth ties: flat and ramped areas where pa == pb, pa == pc, pb == pc
    flat = np.zeros((6, 6, 3), np.uint8)
    flat[3:, :, 0] = 9
    flat[:, 3:, 1] = 9
    flat[::2, ::2, 2] = 200
    out.append(("paeth-ties", pw.make_png(flat, 2, filters=[4] * 6)))
    for i, s in enumerate(((17, 13), (1, 40), (40, 1), (64, 48))):
        out.append((f"cv2-{i}", cv2_png(photo(rng, s[0], s[1], 3))))
    for i, g in enumerate(golden_photos()):
        out.append((f"golden{i}-pil", pillow_png(g, 2)))
        out.append((f"golden{i}-cv2", cv2_png(g)))
    # palette indices past the PLTE's entries (Pillow gives black), a simple tRNS, ancillary chunks
    idx = (np.arange(60).reshape(6, 10, 1) * 5 % 256).astype(np.uint8)
    out.append(("palette-short", pw.make_png(idx, 3, palette=palette_bytes(20))))
    out.append(("palette-trns", pw.make_png(idx, 3, palette=palette_bytes(256),
                                            before=[pw.chunk(b"tRNS", b"\xff\xff\x00")])))
    out.append(("gray-trns-gama", pw.make_png(photo(rng, 5, 5, 1), 0, before=[
        pw.chunk(b"tRNS", b"\x00\x07"), pw.chunk(b"gAMA", struct.pack(">I", 45455)),
        pw.chunk(b"tEXt", b"Comment\0hello"), pw.chunk(b"prIv", b"xyz")])))
    return out


def ineligible_files(seed=1):
    """(name, file) that mhmr_png_info must refuse; Pillow decodes or refuses them on the host."""
    rng = np.random.default_rng(seed)
    px = photo(rng, 8, 8, 3)
    raw = pw.filter_rows(px.reshape(8, 24), 3, [0] * 8)
    z = zlib.compress(raw)
    out = [("interlaced", _interlaced(px))]
    out.append(("16-bit", pw.png_file(8, 8, 2, zlib.compress(bytes(8 * (1 + 48))), depth=16)))
    for d in (1, 2, 4):
        out.append((f"{d}-bit", pw.png_file(8, 8, 0, zlib.compress(bytes(8 * (1 + d))), depth=d)))
    f = pw.png_file(8, 8, 2, z)
    out.append(("bad-ihdr-crc", f[:29] + bytes([f[29] ^ 1]) + f[30:]))
    out.append(("two-idat-runs", pw.png_file(8, 8, 2, z[:10], after=[pw.chunk(b"tEXt", b"a\0b"),
                                                                         pw.chunk(b"IDAT", z[10:])])))
    out.append(("text-after-idat", pw.png_file(8, 8, 2, z, after=[pw.chunk(b"tEXt", b"a\0b")])))
    out.append(("no-plte", pw.png_file(8, 8, 3, z)))
    out.append(("iccp", pw.png_file(8, 8, 2, z, before=[pw.chunk(b"iCCP", b"x\0\0" + zlib.compress(b"p"))])))
    out.append(("trns-bytes", pw.png_file(8, 8, 3, zlib.compress(bytes(8 * 9)), palette=palette_bytes(4),
                                          before=[pw.chunk(b"tRNS", b"\x80\x00")])))
    out.append(("truncated", f[:-20]))
    out.append(("no-iend", f[:-12]))
    return out


def _interlaced(px):
    from PIL import Image

    b = io.BytesIO()
    Image.fromarray(px).save(b, "PNG")
    d = bytearray(b.getvalue())
    # the IHDR interlace flag set, CRC fixed: ineligible by its header alone, whatever Pillow makes of the data
    d[28] = 1
    d[29:33] = struct.pack(">I", zlib.crc32(bytes(d[12:29])))
    return bytes(d)


def _tokens_random(rng, n, window=0):
    """Random literals and copies reaching at most `window + produced` back."""
    toks, have = [], window
    while len(toks) < n:
        if have >= 3 and rng.random() < 0.4:
            d = int(rng.integers(1, min(have, 32768) + 1))
            ln = int(rng.integers(3, 259))
            toks.append((ln, d))
            have += ln
        else:
            toks.append(int(rng.integers(0, 256)))
            have += 1
    return toks


def stream_families(seed=0):
    """(name, zlib stream, inflated bytes or None when zlib refuses it) of the writer's families."""
    rng = np.random.default_rng(seed)
    fam = []

    def add(name, blocks):
        s, d = pw.zstream(blocks)
        fam.append((name, s, d))

    add("stored", [("stored", bytes(range(200)))])
    add("stored-empty-then-data", [("stored", b""), ("stored", b"abc"), ("stored", b"")])
    add("stored-final-after-fixed", [("fixed", [1, 2, 3, (5, 1)]), ("stored", b"xyz" * 50)])
    add("fixed", [("fixed", _tokens_random(rng, 300))])
    add("dynamic", [("dynamic", _tokens_random(rng, 500))])
    # 15-bit codes: literals 0..13 of lengths 1..14, literal 14 and the end-of-block of length 15 (complete)
    lens = [0] * 286
    for i in range(14):
        lens[i] = i + 1
    lens[14] = lens[256] = 15
    toks = [int(v) for v in rng.integers(0, 15, 400)] + [14, 13, 14]
    add("dynamic-15-bit", [("dynamic", toks, {"lit_lens": lens})])
    add("dynamic-one-distance", [("dynamic", [7, 8, 9] + [(10, 3)] * 20 + [1])])
    # a zero run over the end of the literal / length lengths and into the distance lengths (repeat 18 / 17 codes)
    add("repeat-across-boundary", [("dynamic", [65, 66, (4, 2), 67], {"nlit": 286})])
    # a run of length-2 codes from literal / length 285 into the distance lengths (repeat code 16)
    add("repeat16-across-boundary", [("dynamic", [65, (3, 1), (258, 2)], {
        "lit_lens": [0] * 65 + [2] + [0] * 190 + [2, 2] + [0] * 27 + [2], "dist_lens": [2, 2, 2, 2],
        "nlit": 286, "ndist": 4})])
    for ln in (3, 4, 10, 11, 18, 19, 34, 35, 66, 67, 130, 131, 257, 258):
        add(f"length-{ln}", [("fixed", [9, 8, 7] + [(ln, 3)])])
    data = [int(v) for v in rng.integers(0, 256, 33000)]
    for d in (1, 2, 3, 4, 5, 7, 8, 9, 24, 25, 257, 4096, 4097, 16385, 24577, 32767, 32768):
        add(f"distance-{d}", [("stored", bytes(data[:32768])), ("fixed", [(258, d), (3, d), 1])])
    add("overlap-run", [("fixed", [42] + [(258, 1)] * 40)])
    # copies of copies reaching back 1, 2 and many blocks
    blocks = [("stored", bytes(data[:1000]))]
    blocks += [("fixed", [(100, 900), (50, 1)])]
    blocks += [("dynamic", [(200, 1100), (30, 7), 5])]
    blocks += [("fixed", [(258, 1300)] * 3)]
    blocks += [("dynamic", [(40, 1800)] + _tokens_random(rng, 50, 2000), {})]
    add("copy-chains", blocks)
    many = [("dynamic", _tokens_random(rng, 64, 0) if i == 0 else [(20, 20 * i + 17), i % 256])
            for i in range(60)]
    add("copy-many-blocks", many)
    add("one-symbol-block", [("dynamic", []), ("stored", b"q"), ("dynamic", [])])
    add("one-literal-block", [("dynamic", [200]), ("dynamic", [200, 200])])
    # a valid dynamic header planted inside a stored block's bytes: the search finds it, the chain never goes there
    w = pw.BitWriter()
    pw.dynamic_block(w, _tokens_random(rng, 40), True)
    planted = w.bytes()
    add("planted-header", [("stored", planted * 3), ("dynamic", _tokens_random(rng, 100)), ("stored", planted)])
    # zlib refuses these: the device must flag them
    blocks = [("stored", b"ab"), ("fixed", [(3, 3)])]
    fam.append(("distance-too-far", pw.zlib_wrap(pw.deflate(blocks), b"ab"), None))
    return fam


def corrupt(data: bytes, rng: random.Random, body0: int = 2):
    """One seeded corruption: bit flips, truncation, header and trailer edits."""
    b = bytearray(data)
    k = rng.randrange(6)
    if k == 0:
        for _ in range(rng.randint(1, 4)):
            i = rng.randrange(len(b))
            b[i] ^= 1 << rng.randrange(8)
    elif k == 1:
        return bytes(b[:rng.randrange(len(b))]), "truncate"
    elif k == 2:
        b[rng.randrange(min(2, len(b)))] ^= 1 << rng.randrange(8)
    elif k == 3:
        b[-1 - rng.randrange(min(4, len(b)))] ^= 1 << rng.randrange(8)
    elif k == 4:
        i = rng.randrange(body0, max(body0 + 1, len(b)))
        b[i:i + rng.randint(1, 8)] = bytes(rng.randrange(256) for _ in range(rng.randint(0, 8)))
    else:
        i = rng.randrange(len(b))
        b[i] = 255 - b[i]
    return bytes(b), ["flip", "truncate", "header", "trailer", "splice", "invert"][k]
