"""numpy restatement of `Image.open(f).convert("RGB")` for the baseline JPEGs the device decodes (csrc/jpeg.cu), written
from the JPEG standard (ITU-T T.81) and libjpeg-turbo's documented default decompression path, and checked byte for
byte against the installed Pillow (libjpeg-turbo) by tests/test_jpeg_cpu.py.

    header    SOI, then markers up to the first SOS: SOF0 / SOF1 with 8-bit samples, 8-bit DQT, DHT, DRI, APP0 (JFIF),
              APP14 (Adobe), other APPn and COM skipped.  Everything else, or anything malformed, is `Ineligible` (the
              host path decodes it).  The entropy-coded segment runs to the first marker that is neither a stuffed
              0xFF00 nor RSTn, and must be followed by EOI.
    entropy   canonical Huffman codes as libjpeg derives them (a table with an all-ones code is bogus); DC differences
              are summed per component from 0 at every restart interval (int32, stored as 16-bit JCOEF); AC (run,
              size) pairs fill the zig-zag order, (r, 0) with r != 15 is an end of block, (15, 0) sixteen zeros.
              Anomalies are flagged, never repaired: a code with no table entry, a DC category above 11 or an AC size
              above 10, a run past coefficient 63, bits needed past the end of an interval, and RSTn markers missing,
              extra or out of order.
    idct      jpeg_idct_islow: CONST_BITS 13, PASS1_BITS 2, columns then rows, JLONG (64-bit) intermediates, the
              pass-1 results truncated to int, outputs range-limited through the 1024-entry wrap-around table.  A block
              with a dequantised coefficient outside int16 or an output outside [-512, 512) is flagged too: there
              libjpeg-turbo's 16-bit SIMD IDCT and its C IDCT disagree, so no single answer is Pillow's.
    upsample  h2v1 / h2v2 "fancy" (triangle) filters with edge replication at the component's real size
              (downsampled_width, downsampled_height), rounding biases 1 / 2 (h2v1) and 8 / 7 (h2v2); a component at
              most 2 samples wide is box-upsampled instead, as libjpeg-turbo selects.
    colour    YCbCr -> RGB with libjpeg's 16-bit fixed-point tables; grayscale is replicated into three channels.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], dtype=np.int64)   # zig-zag index -> natural (row-major) index

# status bits of a decode (csrc/jpeg.cu uses the same values)
BAD_CODE, BAD_SIZE, BAD_RUN, SHORT_DATA, BAD_RST, IDCT_RANGE = 1, 2, 4, 8, 16, 32


class Ineligible(ValueError):
    """The file is not one the device decodes (or its header is malformed); the host path takes it."""


@dataclass
class Huff:
    maxcode: list          # [18]: largest code of each length, -1 if none (index 17: sentinel)
    valoffset: list        # [17]: value index = code + valoffset[length]
    values: list


@dataclass
class Header:
    width: int
    height: int
    ncomp: int
    samp: list             # [(h, v)] per component
    qt: list               # [64] int per component, natural order
    dc: list               # Huff per component
    ac: list
    restart: int           # restart interval in MCUs (0: none)
    ecs: tuple             # (start, end) byte offsets of the entropy-coded segment
    mcux: int = 0
    mcuy: int = 0
    blocks: list = field(default_factory=list)   # per MCU: [(component, bx, by)] block layout within the MCU
    planes: list = field(default_factory=list)   # per component: (blocks wide, blocks high)


def derive_huff(counts, values, is_dc):
    """libjpeg's derived decoding table (jpeg_make_d_derived_tbl); Ineligible for a bogus table."""
    sizes = [l for l in range(1, 17) for _ in range(counts[l - 1])]
    if len(sizes) > 256 or len(values) != len(sizes):
        raise Ineligible("bogus Huffman table")
    codes, code, p = [], 0, 0
    for si in range(1, 17):
        while p < len(sizes) and sizes[p] == si:
            codes.append(code)
            code += 1
            p += 1
        if code >= (1 << si):
            raise Ineligible("bogus Huffman table definition")
        code <<= 1
    maxcode, valoffset, p = [-1] * 18, [0] * 17, 0
    for l in range(1, 17):
        if counts[l - 1]:
            valoffset[l] = p - codes[p]
            p += counts[l - 1]
            maxcode[l] = codes[p - 1]
    maxcode[17] = 0xFFFFF
    if is_dc and any(v > 15 for v in values):
        raise Ineligible("DC Huffman symbol above 15")
    return Huff(maxcode, valoffset, list(values))


def _be16(d, i):
    return (d[i] << 8) | d[i + 1]


def parse(data: bytes) -> Header:
    """The header of a file the device decodes; `Ineligible` with the reason for any other file."""
    d, n = data, len(data)
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise Ineligible("not a JPEG")
    pos = 2
    sof = None
    dqt, dht = {}, {}
    restart = 0
    jfif = False
    adobe = None
    while True:
        if pos + 4 > n or d[pos] != 0xFF:
            raise Ineligible("no marker where one is expected")
        m = d[pos + 1]
        if m == 0xFF or m == 0x01 or 0xD0 <= m <= 0xD9:
            raise Ineligible(f"unexpected marker 0x{m:02x}")
        length = _be16(d, pos + 2)
        if length < 2 or pos + 2 + length > n:
            raise Ineligible("segment length past the end of the file")
        seg = d[pos + 4:pos + 2 + length]
        pos += 2 + length
        if m in (0xC0, 0xC1):
            if sof is not None or len(seg) < 6:
                raise Ineligible("duplicate or short SOF")
            prec, h, w, nf = seg[0], _be16(seg, 1), _be16(seg, 3), seg[5]
            if prec != 8 or h == 0 or w == 0 or nf not in (1, 3) or len(seg) != 6 + 3 * nf:
                raise Ineligible("not an 8-bit gray or 3-component frame")
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)]
            if len({c[0] for c in comps}) != nf or any(not (1 <= c[1] <= 4 and 1 <= c[2] <= 4) or c[3] > 3
                                                      for c in comps):
                raise Ineligible("bad component parameters")
            if nf == 3 and ((comps[0][1], comps[0][2]) not in ((1, 1), (2, 1), (2, 2))
                            or any((c[1], c[2]) != (1, 1) for c in comps[1:])):
                raise Ineligible("sampling other than 4:4:4, 4:2:2 or 4:2:0")
            sof = (w, h, comps)
        elif 0xC2 <= m <= 0xCF and m != 0xC4:
            raise Ineligible("not a baseline / extended sequential Huffman frame")
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                tc_th = seg[i]
                if tc_th & 0xEC:
                    raise Ineligible("bad DHT class or index")
                if i + 17 > len(seg):
                    raise Ineligible("truncated DHT")
                counts = list(seg[i + 1:i + 17])
                total = sum(counts)
                if total > 256 or i + 17 + total > len(seg):
                    raise Ineligible("bogus or truncated DHT")
                dht[(tc_th >> 4, tc_th & 3)] = (counts, list(seg[i + 17:i + 17 + total]))
                i += 17 + total
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                if pq != 0 or tq > 3:
                    raise Ineligible("16-bit or bad quantisation table")
                if i + 65 > len(seg):
                    raise Ineligible("truncated DQT")
                q = np.zeros(64, np.int64)
                q[ZIGZAG] = np.frombuffer(bytes(seg[i + 1:i + 65]), np.uint8)
                dqt[tq] = q
                i += 65
        elif m == 0xDD:
            if length != 4:
                raise Ineligible("bad DRI length")
            restart = _be16(seg, 0)
        elif m == 0xE0:
            if len(seg) >= 14 and bytes(seg[:5]) == b"JFIF\0":
                jfif = True
        elif m == 0xEE:
            if len(seg) >= 12 and bytes(seg[:5]) == b"Adobe":
                adobe = seg[11]
        elif 0xE1 <= m <= 0xEF or m == 0xFE:
            pass
        elif m == 0xDA:
            break
        else:
            raise Ineligible(f"marker 0x{m:02x} before the scan")
    if sof is None:
        raise Ineligible("SOS before SOF")
    w, h, comps = sof
    nf = len(comps)
    ns = seg[0] if seg else 0
    if ns != nf or len(seg) != 4 + 2 * ns:
        raise Ineligible("the scan does not hold every component")
    dc, ac, qt = [], [], []
    for i in range(ns):
        cid, td, ta = seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15
        if cid != comps[i][0] or td > 3 or ta > 3 or (0, td) not in dht or (1, ta) not in dht \
                or comps[i][3] not in dqt:
            raise Ineligible("scan component, Huffman or quantisation table missing")
        dc.append(derive_huff(*dht[(0, td)], True))
        ac.append(derive_huff(*dht[(1, ta)], False))
        qt.append(dqt[comps[i][3]])
    if (seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]) != (0, 63, 0):
        raise Ineligible("not a sequential scan")
    if nf == 3:
        ids = tuple(c[0] for c in comps)
        if jfif and adobe is not None and adobe != 1 or not jfif and adobe is not None and adobe != 1 \
                or not jfif and adobe is None and ids == (82, 71, 66):
            raise Ineligible("not YCbCr")
    # the entropy-coded segment: up to the first marker that is neither 0xFF00 nor RSTn, then EOI
    start, i = pos, pos
    while True:
        i = d.find(b"\xff", i) if isinstance(d, bytes) else bytes(d).find(b"\xff", i)
        if i < 0 or i + 1 >= n:
            raise Ineligible("no EOI after the scan")
        nx = d[i + 1]
        if nx == 0 or 0xD0 <= nx <= 0xD7:
            i += 2
            continue
        if nx != 0xD9:
            raise Ineligible("the scan is not followed by EOI")
        break
    hdr = Header(w, h, nf, [(c[1], c[2]) for c in comps], qt, dc, ac, restart, (start, i))
    layout(hdr)
    return hdr


def layout(hdr: Header) -> None:
    """MCU grid and block layout: one block per MCU over ceil(W/8) x ceil(H/8) for grayscale (a non-interleaved
    scan); an interleaved MCU of h x v luma blocks then one Cb and one Cr block for YCbCr."""
    if hdr.ncomp == 1:
        hdr.mcux, hdr.mcuy = -(-hdr.width // 8), -(-hdr.height // 8)
        hdr.blocks = [(0, 0, 0)]
        hdr.planes = [(hdr.mcux, hdr.mcuy)]
        return
    hm, vm = hdr.samp[0]
    hdr.mcux, hdr.mcuy = -(-hdr.width // (8 * hm)), -(-hdr.height // (8 * vm))
    hdr.blocks = [(c, bx, by) for c, (h, v) in enumerate(hdr.samp) for by in range(v) for bx in range(h)]
    hdr.planes = [(hdr.mcux * h, hdr.mcuy * v) for h, v in hdr.samp]


def info(data: bytes):
    """(width, height, components, luma (h, v), eligible) from the header alone; eligible is False (and the sizes
    are 0) for any file the device does not decode."""
    try:
        hdr = parse(data)
    except Ineligible:
        return 0, 0, 0, (0, 0), False
    return hdr.width, hdr.height, hdr.ncomp, tuple(hdr.samp[0]) if hdr.ncomp == 3 else (1, 1), True


# ---- entropy decoding ---------------------------------------------------------------------------------------------

def intervals(data: bytes, hdr: Header):
    """The destuffed bytes of each restart interval, and whether the RSTn markers are exactly the expected ones."""
    s, e = hdr.ecs
    raw = bytes(data[s:e])
    out, cur, ok, k, i = [], bytearray(), True, 0, 0
    while i < len(raw):
        b = raw[i]
        if b == 0xFF:
            nx = raw[i + 1]
            if nx == 0:
                cur.append(0xFF)
            else:
                ok &= nx == 0xD0 + (k & 7)
                k += 1
                out.append(bytes(cur))
                cur = bytearray()
            i += 2
            continue
        cur.append(b)
        i += 1
    out.append(bytes(cur))
    mcus = hdr.mcux * hdr.mcuy
    want = -(-mcus // hdr.restart) if hdr.restart else 1
    return out, ok and len(out) == want


class _Bits:
    def __init__(self, buf: bytes):
        self.buf, self.pos, self.n = buf + b"\0\0\0\0", 0, 8 * len(buf)

    def get(self, s):
        """s bits (zeros past the end, as libjpeg inserts them; the caller checks `pos <= n` afterwards)."""
        if s == 0:
            return 0
        p = self.pos
        v = int.from_bytes(self.buf[p >> 3:(p >> 3) + 4], "big")
        self.pos = p + s
        return (v >> (32 - (p & 7) - s)) & ((1 << s) - 1)

    def huff(self, t: Huff):
        code, l = self.get(1), 1
        while code > t.maxcode[l]:
            code = (code << 1) | self.get(1)
            l += 1
            if l > 16:
                return None
        return t.values[code + t.valoffset[l]]


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def decode_coefficients(data: bytes, hdr: Header):
    """(per component int16 [blocks high, blocks wide, 64] natural-order coefficients, status bits)."""
    coefs = [np.zeros((bh, bw, 64), np.int16) for bw, bh in hdr.planes]
    segs, rst_ok = intervals(data, hdr)
    status = 0 if rst_ok else BAD_RST
    mcus = hdr.mcux * hdr.mcuy
    per = hdr.restart if hdr.restart else mcus
    for iv in range(min(len(segs), -(-mcus // per))):
        br = _Bits(segs[iv])
        pred = [0] * hdr.ncomp
        for m in range(iv * per, min(mcus, (iv + 1) * per)):
            my, mx = divmod(m, hdr.mcux)
            for c, bx, by in hdr.blocks:
                h, v = (1, 1) if hdr.ncomp == 1 else hdr.samp[c]
                blk = coefs[c][my * v + by, mx * h + bx]
                s = br.huff(hdr.dc[c])
                if s is None:
                    return coefs, status | BAD_CODE
                if s > 11:
                    return coefs, status | BAD_SIZE
                pred[c] = (pred[c] + _extend(br.get(s), s) + 2 ** 31) % 2 ** 32 - 2 ** 31
                blk[0] = np.int16(((pred[c] + 32768) & 0xFFFF) - 32768)
                k = 1
                while k < 64:
                    rs = br.huff(hdr.ac[c])
                    if rs is None:
                        return coefs, status | BAD_CODE
                    r, s = rs >> 4, rs & 15
                    if s == 0:
                        if r != 15:
                            break
                        if k + 15 > 63:
                            return coefs, status | BAD_RUN
                        k += 16
                        continue
                    if s > 10:
                        return coefs, status | BAD_SIZE
                    k += r
                    if k > 63:
                        return coefs, status | BAD_RUN
                    blk[ZIGZAG[k]] = _extend(br.get(s), s)
                    k += 1
                if br.pos > br.n:
                    return coefs, status | SHORT_DATA
    return coefs, status


# ---- IDCT, upsampling, colour -------------------------------------------------------------------------------------

CONST_BITS, PASS1_BITS = 13, 2
F = dict(c0_298=2446, c0_390=3196, c0_541=4433, c0_765=6270, c0_899=7373, c1_175=9633, c1_501=12299, c1_847=15137,
         c1_961=16069, c2_053=16819, c2_562=20995, c3_072=25172)


def _idct_1d(x):
    """One islow butterfly over axis 1 of x [N, 8] (int64, already scaled inputs); returns the 8 unscaled sums."""
    z2, z3 = x[:, 2], x[:, 6]
    z1 = (z2 + z3) * F["c0_541"]
    tmp2 = z1 + z3 * -F["c1_847"]
    tmp3 = z1 + z2 * F["c0_765"]
    tmp0 = (x[:, 0] + x[:, 4]) << CONST_BITS
    tmp1 = (x[:, 0] - x[:, 4]) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = x[:, 7], x[:, 5], x[:, 3], x[:, 1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F["c1_175"]
    t0, t1, t2, t3 = t0 * F["c0_298"], t1 * F["c2_053"], t2 * F["c3_072"], t3 * F["c1_501"]
    z1, z2, z3, z4 = z1 * -F["c0_899"], z2 * -F["c2_562"], z3 * -F["c1_961"] + z5, z4 * -F["c0_390"] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    return np.stack([t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3], 1)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def idct_islow(coef, q):
    """coef int16 [N, 64] natural order, q [64] -> (uint8 [N, 8, 8], per-block out-of-range flag)."""
    deq = coef.astype(np.int64) * q.astype(np.int64)
    bad = np.abs(deq).max(1) > 32767
    cols = deq.reshape(-1, 8, 8).transpose(0, 2, 1).reshape(-1, 8)        # [N*8 columns, 8 rows]
    ws = _descale(_idct_1d(cols), CONST_BITS - PASS1_BITS)
    ws = ((ws + 2 ** 31) % 2 ** 32) - 2 ** 31                                # (int) of the JLONG result
    ws = ws.reshape(-1, 8, 8).transpose(0, 2, 1)                             # [N, row, col]
    bad |= np.abs(ws).reshape(len(coef), -1).max(1) > 32767
    out = _descale(_idct_1d(ws.reshape(-1, 8)), CONST_BITS + PASS1_BITS + 3).reshape(-1, 8, 8)
    bad |= ((out < -512) | (out > 511)).reshape(len(coef), -1).any(1)
    wrapped = ((out + 512) & 1023) - 512                                     # the range-limit table's wrap-around
    return np.clip(wrapped + 128, 0, 255).astype(np.uint8), bad


def _upsample(p, dw, dh, h, v, hm, vm):
    """Component samples p [>= dh, >= dw] (its real size dw x dh) -> full-resolution rows."""
    p = p[:dh, :dw].astype(np.int32)
    if (h, v) == (hm, vm):
        return p
    if dw <= 2:                                     # box upsampling for a component at most 2 samples wide
        return np.repeat(np.repeat(p, hm // h, 1), vm // v, 0)
    left = np.concatenate([p[:, :1], p[:, :-1]], 1)
    right = np.concatenate([p[:, 1:], p[:, -1:]], 1)
    if vm == v:                                     # h2v1
        out = np.empty((dh, 2 * dw), np.int32)
        out[:, 0::2] = (3 * p + left + 1) >> 2
        out[:, 1::2] = (3 * p + right + 2) >> 2
        out[:, 0] = p[:, 0]
        out[:, -1] = p[:, -1]
        return out
    above = np.concatenate([p[:1], p[:-1]], 0)      # h2v2: rows above / below, edges replicated
    below = np.concatenate([p[1:], p[-1:]], 0)
    out = np.empty((2 * dh, 2 * dw), np.int32)
    for r, nb in ((0, above), (1, below)):
        col = 3 * p + nb                            # vertical sums
        lcol = np.concatenate([col[:, :1], col[:, :-1]], 1)
        rcol = np.concatenate([col[:, 1:], col[:, -1:]], 1)
        even = (3 * col + lcol + 8) >> 4
        odd = (3 * col + rcol + 7) >> 4
        even[:, 0] = (4 * col[:, 0] + 8) >> 4
        odd[:, -1] = (4 * col[:, -1] + 7) >> 4
        out[r::2, 0::2] = even
        out[r::2, 1::2] = odd
    return out


def ycc_tables():
    """libjpeg's build_ycc_rgb_table: (Cr->R, Cb->B, Cr->G, Cb->G) over the 256 sample values, int64."""
    x = np.arange(256, dtype=np.int64) - 128
    fix = lambda v: int(v * 65536 + 0.5)   # noqa: E731
    half = 1 << 15
    return (fix(1.40200) * x + half) >> 16, (fix(1.77200) * x + half) >> 16, -fix(0.71414) * x, \
        -fix(0.34414) * x + half


def decode(data: bytes):
    """(uint8 [H, W, 3] RGB, status bits) of an eligible file; raises Ineligible for any other."""
    hdr = parse(data)
    coefs, status = decode_coefficients(data, hdr)
    hm = max(s[0] for s in hdr.samp) if hdr.ncomp == 3 else 1
    vm = max(s[1] for s in hdr.samp) if hdr.ncomp == 3 else 1
    full = []
    for c, (bw, bh) in enumerate(hdr.planes):
        px, bad = idct_islow(coefs[c].reshape(-1, 64), hdr.qt[c])
        if bad.any():
            status |= IDCT_RANGE
        plane = px.reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)
        h, v = (1, 1) if hdr.ncomp == 1 else hdr.samp[c]
        dw, dh = -(-hdr.width * h // hm), -(-hdr.height * v // vm)
        full.append(_upsample(plane, dw, dh, h, v, hm, vm)[:hdr.height, :hdr.width])
    if hdr.ncomp == 1:
        y = full[0].astype(np.uint8)
        return np.repeat(y[:, :, None], 3, 2), status
    y, cb, cr = full
    crr, cbb, crg, cbg = ycc_tables()
    rgb = np.stack([y + crr[cr], y + ((cbg[cb] + crg[cr]) >> 16), y + cbb[cb]], -1)
    return np.clip(rgb, 0, 255).astype(np.uint8), status
