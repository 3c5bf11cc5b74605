"""numpy restatement of Pillow's `Image.fromarray(img).save(f, "JPEG", quality=q, subsampling=s)` for the RGB and L
images the device encodes (csrc/jpeg_encode.cu), written from the JPEG standard (ITU-T T.81) and libjpeg-turbo's
documented default compression path, and checked byte for byte against the installed Pillow (libjpeg-turbo) by
tests/test_jpeg_encode_cpu.py.

    tables    jpeg_set_quality: scale 5000 / q below 50, 200 - 2 q from 50 up; each entry clamp((basic * scale + 50)
              // 100, 1, 255) of the Annex K basic tables.  The four Annex K Huffman tables (K.3), always.
    colour    RGB -> YCbCr in libjpeg's 16-bit fixed point, FIX(x) = int(x * 65536 + 0.5); gray is the Y plane.
    edges     every plane is replicated rightwards to whole blocks of its component; a subsampled chroma plane is
              formed from the full-resolution plane replicated to twice its block width, and (4:2:0) to an even row
              count, then its rows are replicated down to whole blocks.  The full-resolution plane is never padded to
              the MCU height: that changes the last chroma block row whenever ceil(H / 2) is not a multiple of 8.
    downsample  h2v2 (a + b + c + d + bias) >> 2 with bias 1, 2, 1, 2, ... along the row; h2v1 (a + b + bias) >> 1
              with bias 0, 1, 0, 1, ...
    fdct      jfdctint.c (islow): CONST_BITS 13, PASS1_BITS 2, rows then columns, on samples - 128.
    quantise  sign(x) * ((|x| + 4 q) // 8 q) (the fDCT output carries a factor 8).
    scan      one interleaved scan of MCUs for YCbCr (4:4:4 1x1, 4:2:2 2x1, 4:2:0 2x2 luma blocks per MCU), one
              non-interleaved scan of ceil(W/8) x ceil(H/8) blocks for gray.  An MCU block past the component's blocks
              at the right or bottom edge is a dummy (jccoefct.c compress_data): zero AC, DC copied from the block
              before it in the MCU, so its DC difference is 0.
    entropy   DC differences per component in scan order, AC run / size symbols with ZRL and EOB, 0x00 stuffed after
              every 0xFF byte, the last byte padded with 1-bits, then EOI.
"""
from __future__ import annotations

import numpy as np

ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], dtype=np.int64)   # zig-zag index -> natural (row-major) index

# T.81 Annex K.1, natural order
BASIC_LUMA = [
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99]
BASIC_CHROMA = [
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32

# T.81 Annex K.3: (code counts per length 1..16, values) of the DC / AC tables for luma (0) and chroma (1)
DC_BITS = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0])
DC_VALS = (list(range(12)), list(range(12)))
AC_BITS = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125], [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119])
AC_VALS = (
    [0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
     0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
     0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
     0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
     0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
     0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
     0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
     0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa],
    [0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
     0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
     0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
     0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
     0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
     0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
     0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
     0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa])

SAMPLING = {0: (1, 1), 1: (2, 1), 2: (2, 2)}   # Pillow's subsampling -> luma (h, v); chroma is 1 x 1


def clamp_quality(quality: int) -> int:
    """libjpeg's clamp: quality 0 writes what 1 does, above 100 what 100 does."""
    return min(max(int(quality), 1), 100)


def quant_tables(quality: int):
    """(luma, chroma) int [64] natural-order tables of jpeg_set_quality(quality), force_baseline."""
    q = clamp_quality(quality)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return tuple([min(max((b * scale + 50) // 100, 1), 255) for b in basic] for basic in (BASIC_LUMA, BASIC_CHROMA))


def huff_codes(bits, vals):
    """{value: (code, length)} of the canonical code (T.81 Annex C)."""
    out, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            out[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return out


def header(width: int, height: int, ncomp: int, samp: tuple, quality: int) -> bytes:
    """SOI, APP0 JFIF 1.01, DQT (luma, then chroma), SOF0, DHT (DC0, AC0[, DC1, AC1]) and SOS, as Pillow writes them;
    `samp` is the luma (h, v) written into SOF0."""
    def seg(marker, body):
        return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + bytes(body)

    out = b"\xff\xd8" + seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    tables = quant_tables(quality)
    for t in range(1 if ncomp == 1 else 2):
        out += seg(0xDB, [t] + [tables[t][z] for z in ZIGZAG])
    sof = [8, height >> 8, height & 255, width >> 8, width & 255, ncomp, 1, samp[0] * 16 + samp[1], 0]
    for c in range(1, ncomp):
        sof += [c + 1, 0x11, 1]
    out += seg(0xC0, sof)
    for t in range(1 if ncomp == 1 else 2):
        out += seg(0xC4, [t] + DC_BITS[t] + DC_VALS[t]) + seg(0xC4, [0x10 + t] + AC_BITS[t] + AC_VALS[t])
    sos = [ncomp] + sum(([c + 1, 0 if c == 0 else 0x11] for c in range(ncomp)), []) + [0, 63, 0]
    return out + seg(0xDA, sos)


def _fix(x):
    return int(x * 65536 + 0.5)


def rgb_to_ycc(rgb):
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    half = (128 << 16) + (1 << 15) - 1
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + (1 << 15)) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + half) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + half) >> 16
    return [y, cb, cr]


def _pad(p, h, w):
    if w > p.shape[1]:
        p = np.concatenate([p, np.repeat(p[:, -1:], w - p.shape[1], 1)], 1)
    if h > p.shape[0]:
        p = np.concatenate([p, np.repeat(p[-1:], h - p.shape[0], 0)], 0)
    return p


def _downsample(p, h, v):
    if v == 2:
        bias = np.tile([1, 2], p.shape[1] // 4 + 1)[: p.shape[1] // 2]
        return (p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2] + bias) >> 2
    bias = np.tile([0, 1], p.shape[1] // 4 + 1)[: p.shape[1] // 2]
    return (p[:, 0::2] + p[:, 1::2] + bias) >> 1


_C = dict(a=2446, b=3196, c=4433, d=6270, e=7373, f=9633, g=12299, h=15137, i=16069, j=16819, k=20995, l=25172)


def _ds(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, first):
    t0, t7, t1, t6 = d[0] + d[7], d[0] - d[7], d[1] + d[6], d[1] - d[6]
    t2, t5, t3, t4 = d[2] + d[5], d[2] - d[5], d[3] + d[4], d[3] - d[4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = [None] * 8
    sh = 13 - 2 if first else 13 + 2
    if first:
        o[0], o[4] = (t10 + t11) << 2, (t10 - t11) << 2
    else:
        o[0], o[4] = _ds(t10 + t11, 2), _ds(t10 - t11, 2)
    z1 = (t12 + t13) * _C["c"]
    o[2], o[6] = _ds(z1 + t13 * _C["d"], sh), _ds(z1 - t12 * _C["h"], sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * _C["f"]
    t4, t5, t6, t7 = t4 * _C["a"], t5 * _C["j"], t6 * _C["l"], t7 * _C["g"]
    z1, z2, z3, z4 = -z1 * _C["e"], -z2 * _C["k"], -z3 * _C["i"] + z5, -z4 * _C["b"] + z5
    o[7], o[5], o[3], o[1] = _ds(t4 + z1 + z3, sh), _ds(t5 + z2 + z4, sh), _ds(t6 + z2 + z3, sh), _ds(t7 + z1 + z4, sh)
    return o


def fdct_islow(blocks):
    """[..., 8, 8] int64 samples - 128 -> [..., 8, 8] fDCT outputs (scaled by 8), jfdctint.c."""
    r = np.stack(_fdct_1d([blocks[..., :, i] for i in range(8)], True), -1)
    return np.stack(_fdct_1d([r[..., i, :] for i in range(8)], False), -2)


def quantise(x, qt):
    div = np.asarray(qt, dtype=np.int64).reshape(8, 8) * 8
    return np.sign(x) * ((np.abs(x) + div // 2) // div)


def component_blocks(img, subsampling: int, quality: int):
    """Quantised coefficient planes [(int64 [blocks high, blocks wide, 8, 8] natural order)], one per component, and
    the scan's luma (h, v) sampling."""
    H, W = img.shape[:2]
    luma, chroma = quant_tables(quality)
    if img.ndim == 2:
        p = _pad(img.astype(np.int64), -(-H // 8) * 8, -(-W // 8) * 8)
        return [quantise(fdct_islow(_blocks(p) - 128), luma)], (1, 1)
    h, v = SAMPLING[subsampling]
    out = []
    for c, p in enumerate(rgb_to_ycc(img)):
        if c == 0 or (h, v) == (1, 1):
            p = _pad(p, -(-H // 8) * 8, -(-W // 8) * 8)
        else:
            cw, ch = -(-W // h), -(-H // v)
            bw, bh = -(-cw // 8), -(-ch // 8)
            p = _pad(_downsample(_pad(p, v * ch, 16 * bw), h, v), 8 * bh, 8 * bw)
        out.append(quantise(fdct_islow(_blocks(p) - 128), luma if c == 0 else chroma))
    return out, (h, v)


def _blocks(p):
    bh, bw = p.shape[0] // 8, p.shape[1] // 8
    return p.reshape(bh, 8, bw, 8).transpose(0, 2, 1, 3)


def scan_blocks(planes, samp):
    """The scan's blocks in order: [(component, zig-zag int [64], dummy: None or 'right' / 'bottom')], dummies with
    their copied DC, as compress_data forms them."""
    if len(planes) == 1:
        bh, bw = planes[0].shape[:2]
        return [(0, planes[0][y, x].reshape(64)[ZIGZAG], None) for y in range(bh) for x in range(bw)]
    hm, vm = samp
    bh0, bw0 = planes[0].shape[:2]
    mcux, mcuy = -(-bw0 // hm), -(-bh0 // vm)
    out = []
    for my in range(mcuy):
        for mx in range(mcux):
            for c, p in enumerate(planes):
                h, v = (hm, vm) if c == 0 else (1, 1)
                prev = None
                for j in range(v):
                    for i in range(h):
                        y, x = my * v + j, mx * h + i
                        if y < p.shape[0] and x < p.shape[1]:
                            z, dummy = p[y, x].reshape(64)[ZIGZAG].copy(), None
                        else:
                            z, dummy = np.zeros(64, dtype=np.int64), "bottom" if y >= p.shape[0] else "right"
                            z[0] = prev[0]
                        out.append((c, z, dummy))
                        prev = z
    return out


class _Bits:
    def __init__(self):
        self.out, self.acc, self.n, self.stuffed = bytearray(), 0, 0, 0

    def put(self, code, length):
        self.acc = (self.acc << length) | code
        self.n += length
        while self.n >= 8:
            self.n -= 8
            self._byte((self.acc >> self.n) & 255)
        self.acc &= (1 << self.n) - 1

    def _byte(self, b):
        self.out.append(b)
        if b == 0xFF:
            self.out.append(0)
            self.stuffed += 1

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)


def _category(v):
    return int(abs(int(v))).bit_length()


def _magnitude(v, s):
    return int(v) if v >= 0 else int(v) + (1 << s) - 1


def encode(img, quality: int = 75, subsampling: int | None = None, stats: dict | None = None) -> bytes:
    """The bytes Pillow writes for uint8 `img` ([H, W, 3] RGB or [H, W] gray); `stats`, when given, receives counts
    of the code paths the image reached (largest DC / AC category, ZRL symbols, dummy blocks, stuffed bytes)."""
    img = np.asarray(img, dtype=np.uint8)
    H, W = img.shape[:2]
    assert img.ndim in (2, 3) and (img.ndim == 2 or img.shape[2] == 3) and 1 <= H <= 65535 and 1 <= W <= 65535
    quality = clamp_quality(quality)
    s = 2 if subsampling is None else subsampling
    planes, samp = component_blocks(img, s, quality)
    written = samp if img.ndim == 3 else SAMPLING[s] if subsampling is not None else (1, 1)
    hdr = header(W, H, len(planes), written, quality)
    dc = [huff_codes(DC_BITS[t], DC_VALS[t]) for t in (0, 1)]
    ac = [huff_codes(AC_BITS[t], AC_VALS[t]) for t in (0, 1)]
    st = dict(dc_cat=0, ac_cat=0, zrl=0, dummy_right=0, dummy_bottom=0, stuffed=0)
    bits, pred = _Bits(), [0, 0, 0]
    for c, z, dummy in scan_blocks(planes, samp):
        t = 0 if c == 0 else 1
        if dummy:
            st["dummy_" + dummy] += 1
        diff = int(z[0]) - pred[c]
        pred[c] = int(z[0])
        cat = _category(diff)
        st["dc_cat"] = max(st["dc_cat"], cat)
        bits.put(*dc[t][cat])
        if cat:
            bits.put(_magnitude(diff, cat), cat)
        run = 0
        for k in range(1, 64):
            v = int(z[k])
            if v == 0:
                run += 1
                continue
            while run > 15:
                bits.put(*ac[t][0xF0])
                st["zrl"] += 1
                run -= 16
            cat = _category(v)
            st["ac_cat"] = max(st["ac_cat"], cat)
            bits.put(*ac[t][run * 16 + cat])
            bits.put(_magnitude(v, cat), cat)
            run = 0
        if run:
            bits.put(*ac[t][0x00])
    bits.flush()
    st["stuffed"] = bits.stuffed
    if stats is not None:
        for k, v in st.items():
            stats[k] = max(stats.get(k, 0), v) if k in ("dc_cat", "ac_cat") else stats.get(k, 0) + v
    return hdr + bytes(bits.out) + b"\xff\xd9"
