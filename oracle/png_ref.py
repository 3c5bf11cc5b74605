"""numpy / Python restatement of the device PNG decoder (multi-hmr_b200/csrc/png.cu): the eligibility rules of the
host chunk walk, inflate as RFC 1950 / 1951 with zlib's validity rules, the chain of blocks the device follows, the
five scanline filters and the expansion to RGB.  The status bits are the device's, block for block: the device
measures each block without a window and then chains the measurements, so this decodes each block the same way
(`measure`) before it writes it (`emit`, with the window), and applies the same precedence of errors.

Pinned against Pillow (`Image.open(f).convert("RGB")`) and Python's zlib by tests/test_png_cpu.py and
tests/test_png_edges_cpu.py."""
from __future__ import annotations

import struct
import zlib

import numpy as np

BAD_CODE, BAD_DIST, BAD_CHAIN, BAD_LENGTH, BAD_FILTER, BAD_ADLER, BAD_HEADER = 1, 2, 4, 8, 16, 32, 64

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LENS = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
MAX_STREAM = 1 << 28
MAX_INFLATED = 1 << 30


def chain_cap(expect):
    """Blocks the device's chain holds for a photo of `expect` inflated bytes (more is BAD_CHAIN)."""
    return 1024 + expect // 64


class Bits:
    """The device's bit reader: 32 bits from any position, LSB first, zeros past the stream."""

    def __init__(self, data: bytes):
        self.n = len(data)
        self.buf = bytes(data) + bytes(16)
        self.nw = (self.n + 8) // 4

    def peek(self, pos: int) -> int:
        w = pos >> 5
        if w < 0 or w > self.nw - 2:
            return 0
        v = int.from_bytes(self.buf[4 * w:4 * w + 8], "little")
        return (v >> (pos & 31)) & 0xFFFFFFFF


def lengths_ok(lens, kind):
    """zlib's inflate_table verdict ('codes', 'lens' or 'dists'); see png.cu `lengths_ok`."""
    count = [0] * 16
    for v in lens:
        count[v] += 1
    mx = max((l for l in range(1, 16) if count[l]), default=0)
    if mx == 0:
        return kind == "dists"
    left = 1
    for l in range(1, 16):
        left = (left << 1) - count[l]
        if left < 0:
            return False
    return not (left > 0 and (kind == "codes" or mx != 1))


class Huff:
    """Canonical code -> a 15-bit stream-order lookup table of (symbol << 4 | length), -1 for no code."""

    def __init__(self, lens):
        lut = np.full(1 << 15, -1, dtype=np.int32)
        count = [0] * 16
        for v in lens:
            count[v] += 1
        count[0] = 0
        code, nxt = 0, [0] * 16
        for l in range(1, 16):
            code = (code + count[l - 1]) << 1
            nxt[l] = code
        for s, l in enumerate(lens):
            if l:
                c = nxt[l]
                nxt[l] += 1
                rev = int(format(c, f"0{l}b")[::-1], 2)
                lut[rev::1 << l] = s << 4 | l
        self.lut = lut.tolist()

    def decode(self, bits):
        e = self.lut[bits & 0x7FFF]
        return (-1, 0) if e < 0 else (e >> 4, e & 15)


def read_dynamic(bits: Bits, pos: int, end: int):
    """A dynamic block's header after its 3 type bits -> (error, pos, lens, nlit, ndist); png.cu `read_dynamic`."""
    b = bits.peek(pos)
    nlit, ndist, ncl = (b & 31) + 257, ((b >> 5) & 31) + 1, ((b >> 10) & 15) + 4
    pos += 14
    if nlit > 286 or ndist > 30:
        return BAD_CODE, pos, None, nlit, ndist
    cl = [0] * 19
    for i in range(ncl):
        cl[CL_ORDER[i]] = bits.peek(pos + 3 * i) & 7
    pos += 3 * ncl
    if pos > end:
        return BAD_CHAIN, pos, None, nlit, ndist
    if not lengths_ok(cl, "codes"):
        return BAD_CODE, pos, None, nlit, ndist
    h = Huff(cl)
    total, lens = nlit + ndist, []
    while len(lens) < total:
        b = bits.peek(pos)
        s, l = h.decode(b)
        pos += l
        b >>= l
        if s < 16:
            lens.append(s)
        else:
            if s == 16:
                if not lens:
                    return BAD_CODE, pos, None, nlit, ndist
                v, rep = lens[-1], 3 + (b & 3)
                pos += 2
            elif s == 17:
                v, rep = 0, 3 + (b & 7)
                pos += 3
            else:
                v, rep = 0, 11 + (b & 127)
                pos += 7
            if len(lens) + rep > total:
                return BAD_CODE, pos, None, nlit, ndist
            lens += [v] * rep
        if pos > end:
            return BAD_CHAIN, pos, None, nlit, ndist
    if lens[256] == 0:
        return BAD_CODE, pos, None, nlit, ndist
    if not lengths_ok(lens[:nlit], "lens") or not lengths_ok(lens[nlit:], "dists"):
        return BAD_CODE, pos, None, nlit, ndist
    return 0, pos, lens, nlit, ndist


def decode_block(bits: Bits, start: int, cap: int, out: bytearray | None = None):
    """The block at bit `start` -> dict(end, len, far, err, final), png.cu `decode_block`.  With `out` (the bytes
    before the block) the block's bytes are appended to it; the caller does so only after the chain accepted the
    measurement, so every copy source then exists."""
    end = 8 * bits.n
    m = dict(end=start, len=0, far=0, err=0, final=0)
    b = bits.peek(start)
    m["final"] = b & 1
    kind = (b >> 1) & 3
    pos = start + 3
    if kind == 3:
        m["err"] = BAD_CODE
        return m
    if kind == 0:
        pos = (pos + 7) & ~7
        b = bits.peek(pos)
        n = b & 0xFFFF
        if (b >> 16) != (~b & 0xFFFF):
            m["err"] = BAD_CHAIN if pos + 32 > end else BAD_CODE
            return m
        pos += 32
        if pos + 8 * n > end:
            m["err"] = BAD_CHAIN
            return m
        if n > cap:
            m["err"] = BAD_LENGTH
            return m
        if out is not None:
            out += bits.buf[pos // 8:pos // 8 + n]
        m["len"], m["end"] = n, pos + 8 * n
        return m
    if kind == 1:
        lit, dist, nlit, ndist = Huff(FIXED_LENS), Huff([5] * 32), 286, 30
    else:
        err, pos, lens, nlit, ndist = read_dynamic(bits, pos, end)
        if err:
            m["err"] = err
            return m
        lit = Huff(lens[:nlit])
        dl = lens[nlit:]
        if not any(dl):
            ndist = 0
        dist = Huff(dl) if ndist else None
    n, base = 0, 0 if out is None else len(out)
    while True:
        if pos > end:
            m["err"] = BAD_CHAIN
            break
        b = bits.peek(pos)
        s, l = lit.decode(b)
        if s < 0 or s >= nlit:
            m["err"] = BAD_CODE
            break
        pos += l
        if s < 256:
            if n >= cap:
                m["err"] = BAD_LENGTH
                break
            if out is not None:
                out.append(s)
            n += 1
            continue
        if s == 256:
            if pos > end:
                m["err"] = BAD_CHAIN
            break
        li = s - 257
        ln = LEN_BASE[li] + ((b >> l) & ((1 << LEN_EXTRA[li]) - 1))
        pos += LEN_EXTRA[li]
        b = bits.peek(pos)
        ds, l = dist.decode(b) if ndist else (-1, 0)
        if ds < 0 or ds >= ndist:
            m["err"] = BAD_CODE
            break
        d = DIST_BASE[ds] + ((b >> l) & ((1 << DIST_EXTRA[ds]) - 1))
        pos += l + DIST_EXTRA[ds]
        m["far"] = max(m["far"], d - n)
        if n + ln > cap:
            m["err"] = BAD_LENGTH
            break
        if out is not None:
            src = base + n - d
            for i in range(ln):
                out.append(out[src + i])
        n += ln
    m["len"], m["end"] = n, pos
    return m


def inflate(stream: bytes, expect: int):
    """zlib stream -> (status, inflated bytes or None, chain blocks), the device's verdict: status 0 exactly when
    the stream inflates, as zlib does it, to `expect` bytes with a matching Adler-32."""
    bits = Bits(stream)
    h = bits.peek(0)
    cmf, flg = h & 255, (h >> 8) & 255
    if len(stream) < 2 or (cmf * 256 + flg) % 31 or (cmf & 15) != 8 or (cmf >> 4) > 7 or (flg & 32):
        return BAD_HEADER, None, 0
    out, pos, nblocks, err, final = bytearray(), 16, 0, 0, False
    cap = chain_cap(expect)
    while True:
        if nblocks >= cap:
            err = BAD_CHAIN
            break
        total = len(out)
        m = decode_block(bits, pos, expect)
        if m["far"] > total:
            err = BAD_DIST
        elif m["err"]:
            err = m["err"]
        elif total + m["len"] > expect:
            err = BAD_LENGTH
        if err:
            break
        decode_block(bits, pos, expect, out)
        nblocks += 1
        pos = m["end"]
        if m["final"]:
            final = True
            break
    if not err and len(out) != expect:
        err = BAD_LENGTH
    if not err:
        q = (pos + 7) >> 3
        if q + 4 > len(stream):
            err = BAD_ADLER
        elif struct.unpack(">I", stream[q:q + 4])[0] != zlib.adler32(bytes(out)):
            err = BAD_ADLER
    assert err or final
    return err, (None if err else bytes(out)), nblocks


def parse(data: bytes):
    """The chunk walk of png.cu `parse`: dict(W, H, ctype, palette, stream) for an eligible file, else None."""
    data = bytes(data)
    if len(data) < 8 or data[:8] != b"\x89PNG\r\n\x1a\n":
        return None
    pos, hdr, plte, trns, text, stream, in_idat = 8, None, None, False, 0, [], False
    passive = {b"gAMA": 4, b"cHRM": 32, b"sRGB": 1, b"pHYs": 9}
    refused = {b"IHDR", b"IEND", b"iCCP", b"zTXt", b"iTXt", b"eXIf", b"acTL", b"fcTL", b"fdAT"}
    while True:
        if pos + 12 > len(data):
            return None
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        t = data[pos + 4:pos + 8]
        if n > 0x7FFFFFFF or pos + 12 + n > len(data) or not all(chr(c).isascii() and chr(c).isalpha() for c in t):
            return None
        c = data[pos + 8:pos + 8 + n]
        if hdr is None:
            if t != b"IHDR" or n != 13:
                return None
            W, H, depth, ct, comp, filt, inter = struct.unpack(">IIBBBBB", c)
            if not (1 <= W <= 0x7FFFFFFF and 1 <= H <= 0x7FFFFFFF) or depth != 8 or ct not in CHANNELS \
                    or comp or filt or inter:
                return None
            hdr = dict(W=W, H=H, ctype=ct)
        elif t == b"IDAT":
            if ct == 3 and plte is None:
                return None
            in_idat = True
            stream.append(c)
        elif in_idat:
            if t != b"IEND":
                return None
            pal = np.zeros(768, dtype=np.uint8)
            if plte is not None:
                pal[:len(plte)] = np.frombuffer(plte, dtype=np.uint8)
            return dict(hdr, palette=pal.reshape(256, 3), stream=b"".join(stream))
        elif t == b"PLTE":
            if plte is not None or n % 3 or not 3 <= n <= 768 or ct in (0, 4):
                return None
            plte = c
        elif t == b"tRNS":
            if trns:
                return None
            trns = True
            if ct == 0 and n != 2 or ct == 2 and n != 6 or ct in (4, 6):
                return None
            if ct == 3 and (plte is None or not 1 <= n <= len(plte) // 3 or c.count(0) != 1
                            or c.count(0) + c.count(255) != n):
                return None
        elif t in passive:
            if n != passive[t]:
                return None
        elif t == b"tEXt":
            text += n
            if text > 1 << 20:
                return None
        elif t in refused:
            return None
        if t != b"IDAT" and zlib.crc32(t + c) != struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0]:
            return None
        pos += 12 + n


def unfilter(inf: bytes, W: int, H: int, bpp: int):
    """Inflated scanlines -> (status, uint8 [H, W * bpp] reconstructed bytes)."""
    stride = 1 + W * bpp
    a = np.frombuffer(inf, dtype=np.uint8).reshape(H, stride)
    out = np.zeros((H, W * bpp), dtype=np.int32)
    prev = np.zeros(W * bpp, dtype=np.int32)
    status = 0
    for y in range(H):
        ft, f = int(a[y, 0]), a[y, 1:].astype(np.int32)
        if ft > 4:
            status = BAD_FILTER
        if ft == 2:
            row = (f + prev) & 255
        elif ft in (1, 3, 4):
            row = np.zeros_like(f)
            for x in range(0, W * bpp, bpp):
                left = row[x - bpp:x] if x else np.zeros(bpp, dtype=np.int32)
                up = prev[x:x + bpp]
                ul = prev[x - bpp:x] if x else np.zeros(bpp, dtype=np.int32)
                if ft == 1:
                    pred = left
                elif ft == 3:
                    pred = (left + up) >> 1
                else:
                    p = left + up - ul
                    pa, pb, pc = np.abs(p - left), np.abs(p - up), np.abs(p - ul)
                    pred = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, ul))
                row[x:x + bpp] = (f[x:x + bpp] + pred) & 255
        else:
            row = f
        out[y] = row
        prev = row
    return status, out.astype(np.uint8)


def expand(raw: np.ndarray, W: int, H: int, ctype: int, palette: np.ndarray) -> np.ndarray:
    """Reconstructed bytes -> uint8 [H, W, 3] RGB, as Pillow's convert("RGB"): gray replicated, alpha dropped,
    palette looked up (entries past the PLTE's are black)."""
    px = raw.reshape(H, W, CHANNELS[ctype])
    if ctype == 3:
        return palette[px[..., 0]]
    if ctype in (0, 4):
        return np.repeat(px[..., :1], 3, axis=2)
    return np.ascontiguousarray(px[..., :3])


def decode(data: bytes):
    """A PNG file -> (status, uint8 [H, W, 3] RGB or None); None, None for an ineligible file."""
    h = parse(data)
    if h is None:
        return None, None
    W, H, ct = h["W"], h["H"], h["ctype"]
    bpp = CHANNELS[ct]
    status, inf, _ = inflate(h["stream"], H * (1 + W * bpp))
    if status:
        return status, None
    status, raw = unfilter(inf, W, H, bpp)
    if status:
        return status, None
    return 0, expand(raw, W, H, ct, h["palette"])
