"""Test-only zlib / PNG writer that follows RFC 1950, RFC 1951 and the PNG specification directly, so that tests can
make the streams no PNG encoder writes: stored blocks anywhere (empty, final, straddling IDAT chunks), fixed and
dynamic blocks with explicit code lengths (15-bit codes, one distance code, repeat codes across the literal / length
-> distance boundary), copies of any length and distance, one-symbol blocks, and IDAT split at any sizes.

A deflate stream is a list of blocks; a block's content is a list of tokens: an int (a literal byte) or a tuple
(length, distance).  `expand` gives the bytes any inflater must produce."""
from __future__ import annotations

import heapq
import struct
import zlib

import numpy as np

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


class BitWriter:
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value: int, nbits: int):
        self.v |= (value & ((1 << nbits) - 1)) << self.n
        self.n += nbits

    def put_code(self, code: int, length: int):
        """A Huffman code: most significant bit first."""
        self.put(int(format(code, f"0{length}b")[::-1], 2) if length else 0, length)

    def align(self):
        self.n = (self.n + 7) & ~7

    def bytes(self) -> bytes:
        return (self.v).to_bytes((self.n + 7) // 8, "little")


def canonical(lens):
    """Code of each symbol (canonical Huffman, RFC 1951 3.2.2)."""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    codes = [0] * len(lens)
    for s, l in enumerate(lens):
        if l:
            codes[s] = nxt[l]
            nxt[l] += 1
    return codes


def huffman_lengths(freq, limit):
    """Code lengths <= limit for the symbols of nonzero frequency (Huffman, then JPEG Annex K.3's length limiting)."""
    used = [s for s, f in enumerate(freq) if f]
    lens = [0] * len(freq)
    if len(used) == 1:
        lens[used[0]] = 1
        return lens
    if not used:
        return lens
    heap = [(freq[s], i, [s]) for i, s in enumerate(used)]
    heapq.heapify(heap)
    depth = {s: 0 for s in used}
    k = len(heap)
    while len(heap) > 1:
        f1, _, a = heapq.heappop(heap)
        f2, _, b = heapq.heappop(heap)
        for s in a + b:
            depth[s] += 1
        heapq.heappush(heap, (f1 + f2, k, a + b))
        k += 1
    mx = max(depth.values())
    counts = [0] * (max(mx, limit) + 1)
    for d in depth.values():
        counts[d] += 1
    for i in range(mx, limit, -1):
        while counts[i] > 0:
            j = i - 2
            while counts[j] == 0:
                j -= 1
            counts[i] -= 2
            counts[i - 1] += 1
            counts[j + 1] += 2
            counts[j] -= 1
    order = sorted(used, key=lambda s: (-freq[s], s))
    lengths = [l for l in range(1, limit + 1) for _ in range(counts[l])]
    for s, l in zip(order, lengths):
        lens[s] = l
    return lens


def _len_sym(n):
    for i in range(28, -1, -1):
        if n >= LEN_BASE[i] and (i != 28 or n == 258):
            if i == 27 and n == 258:
                continue
            return i, n - LEN_BASE[i]
    raise ValueError(n)


def _dist_sym(d):
    for i in range(29, -1, -1):
        if d >= DIST_BASE[i]:
            return i, d - DIST_BASE[i]
    raise ValueError(d)


def _symbols(tokens):
    lit, dist = [0] * 286, [0] * 30
    for t in tokens:
        if isinstance(t, int):
            lit[t] += 1
        else:
            lit[257 + _len_sym(t[0])[0]] += 1
            dist[_dist_sym(t[1])[0]] += 1
    lit[256] += 1
    return lit, dist


def _write_tokens(w, tokens, lit_lens, dist_lens):
    lc, dc = canonical(lit_lens), canonical(dist_lens)
    for t in tokens:
        if isinstance(t, int):
            w.put_code(lc[t], lit_lens[t])
        else:
            i, e = _len_sym(t[0])
            w.put_code(lc[257 + i], lit_lens[257 + i])
            w.put(e, LEN_EXTRA[i])
            i, e = _dist_sym(t[1])
            w.put_code(dc[i], dist_lens[i])
            w.put(e, DIST_EXTRA[i])
    w.put_code(lc[256], lit_lens[256])


def _rle(lens, rle=True):
    """Code-length symbols: (symbol, extra value, extra bits)."""
    out, i = [], 0
    while i < len(lens):
        v, j = lens[i], i
        while j < len(lens) and lens[j] == v:
            j += 1
        run = j - i
        if rle and v == 0 and run >= 3:
            while run >= 11:
                k = min(run, 138)
                out.append((18, k - 11, 7))
                run -= k
                i += k
            if run >= 3:
                out.append((17, run - 3, 3))
                i += run
                run = 0
        elif rle and run >= 4:
            out.append((v, 0, 0))
            i += 1
            run -= 1
            while run >= 3:
                k = min(run, 6)
                out.append((16, k - 3, 2))
                run -= k
                i += k
        for _ in range(run):
            out.append((v, 0, 0))
            i += 1
    return out


def stored_block(w, data: bytes, final: bool):
    w.put(int(final), 1)
    w.put(0, 2)
    w.align()
    w.put(len(data), 16)
    w.put(~len(data) & 0xFFFF, 16)
    for b in data:
        w.put(b, 8)


def fixed_block(w, tokens, final: bool):
    w.put(int(final), 1)
    w.put(1, 2)
    _write_tokens(w, tokens, FIXED_LIT, [5] * 30)


def dynamic_block(w, tokens, final: bool, lit_lens=None, dist_lens=None, rle=True, nlit=None, ndist=None):
    """A dynamic block; code lengths from the tokens' frequencies unless given (lists of 286 / 30 or fewer)."""
    lf, df = _symbols(tokens)
    if lit_lens is None:
        lit_lens = huffman_lengths(lf, 15)
    if dist_lens is None:
        dist_lens = huffman_lengths(df, 15)
    lit_lens = list(lit_lens) + [0] * (286 - len(lit_lens))
    dist_lens = list(dist_lens) + [0] * (30 - len(dist_lens))
    if nlit is None:
        nlit = max(257, max(i for i, l in enumerate(lit_lens) if l) + 1)
    if ndist is None:
        ndist = max([1] + [i + 1 for i, l in enumerate(dist_lens) if l])
    cl_syms = _rle(lit_lens[:nlit] + dist_lens[:ndist], rle)
    cf = [0] * 19
    for s, _, _ in cl_syms:
        cf[s] += 1
    if sum(1 for f in cf if f) == 1:   # the code-length code must be complete
        cf[18 if cl_syms[0][0] != 18 else 0] += 1
    cl_lens = huffman_lengths(cf, 7)
    ncl = max(4, max(i for i, s in enumerate(CL_ORDER) if cl_lens[s]) + 1)
    w.put(int(final), 1)
    w.put(2, 2)
    w.put(nlit - 257, 5)
    w.put(ndist - 1, 5)
    w.put(ncl - 4, 4)
    for i in range(ncl):
        w.put(cl_lens[CL_ORDER[i]], 3)
    cc = canonical(cl_lens)
    for s, e, nb in cl_syms:
        w.put_code(cc[s], cl_lens[s])
        w.put(e, nb)
    _write_tokens(w, tokens, lit_lens[:nlit], dist_lens[:ndist])


def expand(blocks):
    """The bytes of a list of ('stored', data) / ('fixed' | 'dynamic', tokens, ...) blocks."""
    out = bytearray()
    for b in blocks:
        if b[0] == "stored":
            out += b[1]
            continue
        for t in b[1]:
            if isinstance(t, int):
                out.append(t)
            else:
                n, d = t
                for _ in range(n):
                    out.append(out[-d])
    return bytes(out)


def deflate(blocks):
    """Raw deflate bytes of the blocks: ('stored', data), ('fixed', tokens), ('dynamic', tokens, {options}); the last
    block is final unless a block says {'final': ...} itself."""
    w = BitWriter()
    for i, b in enumerate(blocks):
        opts = b[2] if len(b) > 2 else {}
        final = opts.get("final", i == len(blocks) - 1)
        if b[0] == "stored":
            stored_block(w, b[1], final)
        elif b[0] == "fixed":
            fixed_block(w, b[1], final)
        else:
            dynamic_block(w, b[1], final, **{k: v for k, v in opts.items() if k != "final"})
    return w.bytes()


def zlib_wrap(raw_deflate: bytes, data: bytes, level_bits: int = 2) -> bytes:
    cmf = 0x78
    flg = level_bits << 6
    flg += 31 - (cmf * 256 + flg) % 31
    return bytes([cmf, flg]) + raw_deflate + struct.pack(">I", zlib.adler32(data))


def zstream(blocks) -> tuple[bytes, bytes]:
    """(zlib stream, its inflated bytes)."""
    data = expand(blocks)
    return zlib_wrap(deflate(blocks), data), data


# ---- PNG ----------------------------------------------------------------------------------------------------------
def chunk(kind: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data))


def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def filter_rows(px: np.ndarray, bpp: int, filters) -> bytes:
    """uint8 [H, W * bpp] pixels -> scanlines with the filter types `filters` (one per row)."""
    H, n = px.shape
    if not any(filters):
        return np.concatenate([np.zeros((H, 1), np.uint8), px], axis=1).tobytes()
    out, prev = bytearray(), [0] * n
    for y in range(H):
        row, ft = [int(v) for v in px[y]], filters[y]
        out.append(ft)
        for x in range(n):
            a = row[x - bpp] if x >= bpp else 0
            b = prev[x]
            c = prev[x - bpp] if x >= bpp else 0
            pred = [0, a, b, (a + b) >> 1, paeth(a, b, c)][ft]
            out.append((row[x] - pred) & 255)
        prev = row
    return bytes(out)


def png_file(W, H, ctype, stream: bytes, palette: bytes | None = None, before=(), idat_sizes=None,
             after=(), interlace=0, depth=8) -> bytes:
    """A PNG file around a zlib stream; `idat_sizes` splits it into IDAT chunks of those sizes (the rest in one)."""
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, ctype, 0, 0, interlace))
    if palette is not None:
        out += chunk(b"PLTE", palette)
    for c in before:
        out += c
    pos = 0
    for n in idat_sizes or []:
        out += chunk(b"IDAT", stream[pos:pos + n])
        pos += n
    if pos < len(stream) or not idat_sizes:
        out += chunk(b"IDAT", stream[pos:])
    for c in after:
        out += c
    return out + chunk(b"IEND", b"")


def make_png(px: np.ndarray, ctype: int, filters=None, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, palette=None,
             idat_sizes=None, before=()) -> bytes:
    """uint8 [H, W, channels] -> a PNG with the given per-row filter types (None: all 0) and zlib settings."""
    H, W = px.shape[:2]
    bpp = CHANNELS[ctype]
    raw = filter_rows(px.reshape(H, W * bpp), bpp, filters if filters is not None else [0] * H)
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    return png_file(W, H, ctype, c.compress(raw) + c.flush(), palette=palette, idat_sizes=idat_sizes, before=before)
