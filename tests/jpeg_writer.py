"""A baseline JPEG writer that takes quantised coefficients, for the JPEG decode tests (oracle/jpeg_ref.py, csrc/jpeg.cu).

Pillow's encoder only writes its standard or optimised tables in slots 0 / 1, ends every block with EOB and gives the
parallel Huffman decoder streams it synchronises on quickly.  This writer follows ITU-T T.81 directly: the caller
chooses every coefficient, every table, its slot and each component's selectors, the restart interval and how a block
ends, so the decoder's slow Huffman path, its worst-case synchronisation, DC-prediction wrap-around and marker
placement can be reached on purpose.  It returns the exact coefficient planes libjpeg decodes from the file and a log of
the symbols it emitted, so a test can assert what its stream covers.
"""
from dataclasses import dataclass

import numpy as np

ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], dtype=np.int64)   # zig-zag index -> natural index
SAMPLING = {"L": [(1, 1)], "444": [(1, 1)] * 3, "422": [(2, 1), (1, 1), (1, 1)], "420": [(2, 2), (1, 1), (1, 1)]}
EOB, ZRL = 0x00, 0xF0


def table(lengths: dict):
    """(counts, values) of a DHT table from {symbol: code length}; values ordered by length, then symbol."""
    counts = [0] * 16
    for l in lengths.values():
        counts[l - 1] += 1
    assert sum(c / 2 ** (l + 1) for l, c in enumerate(counts)) < 1, "the all-ones code must stay unused"
    return counts, sorted(lengths, key=lambda s: (lengths[s], s))


def flat_tables():
    """DC categories 0-11 at 4 bits and all 162 AC symbols at 8 bits: every coefficient is codable."""
    ac = {EOB: 8, ZRL: 8}
    ac.update({(r << 4) | s: 8 for r in range(16) for s in range(1, 11)})
    return table({s: 4 for s in range(12)}), table(ac)


def codes(counts):
    """Canonical codes (code, length) in value order, as T.81 Annex C assigns them."""
    out, code = [], 0
    for l in range(1, 17):
        for _ in range(counts[l - 1]):
            out.append((code, l))
            code += 1
        code <<= 1
    return out


def segment(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker, (len(payload) + 2) >> 8, (len(payload) + 2) & 255]) + payload


def dqt(slot: int, q) -> bytes:
    """DQT of 64 8-bit quantisers given in natural order."""
    q = np.asarray(q, np.int64)
    return segment(0xDB, bytes([slot]) + bytes(int(v) for v in q[ZIGZAG]))


def dht(cls: int, slot: int, counts, values) -> bytes:
    return segment(0xC4, bytes([cls << 4 | slot]) + bytes(counts) + bytes(values))


def planes_shape(width, height, mode):
    """[(blocks high, blocks wide)] of each component's plane: the padded MCU grid."""
    samp = SAMPLING[mode]
    hm, vm = samp[0] if mode != "L" else (1, 1)
    mx, my = -(-width // (8 * hm)), -(-height // (8 * vm))
    return [(my * v, mx * h) for h, v in samp] if mode != "L" else [(my, mx)]


@dataclass
class Stream:
    data: bytes
    planes: list           # per component int16 [blocks high, blocks wide, 64], natural order: what libjpeg decodes
    log: np.ndarray        # [symbols, 4] int64: class (0 DC, 1 AC), component, code length, bit offset of the code
    ecs: tuple             # (start, end) byte offsets of the entropy-coded segment in `data`
    markers: list          # RSTn offsets inside the entropy-coded segment (raw, stuffed bytes)
    interval_bytes: list   # destuffed bytes of each restart interval, padding included

    @property
    def raw(self) -> bytes:
        return self.data[self.ecs[0]:self.ecs[1]]


def _pack(vals, nbits):
    """Bits of (value, width) pairs, MSB first, 1-padded to a byte; bytes before stuffing."""
    if len(vals) == 0:
        return b""
    v = (np.asarray(vals, np.uint64) << (np.uint64(32) - np.asarray(nbits, np.uint64))).astype(">u4")
    bits = np.unpackbits(v.view(np.uint8)).reshape(-1, 32)
    bits = bits[np.arange(32)[None, :] < np.asarray(nbits)[:, None]]
    bits = np.concatenate([bits, np.ones(-len(bits) % 8, np.uint8)])
    return np.packbits(bits).tobytes()


def write(width, height, mode, coefs, *, dc=None, ac=None, sel=None, qt=None, tq=None, restart=0, zrl_end=None,
          before=b"", scan_order=None) -> Stream:
    """A baseline (SOF0) file of `coefs`: per component int64 [blocks high, blocks wide, 64] in zig-zag order over the
    padded MCU grid, index 0 the absolute DC (libjpeg's running sum from 0 at every restart; any int, its 16-bit wrap
    is what libjpeg stores).  AC values must fit category 10, DC differences category 11.

    dc / ac: {slot 0-3: (counts, values)} (default: `flat_tables` in slot 0); sel: per component (DC slot, AC slot);
    qt: {slot: 64 natural-order quantisers} (default all 1 in slot 0); tq: per component quantisation slot; restart:
    DRI in MCUs (0: none); zrl_end: per component bool [blocks high, blocks wide], blocks whose trailing zeros are
    coded as ZRLs up to coefficient 64 instead of EOB (their last nonzero zig-zag index + 1 must be a multiple of 16
    below 64); before: segments written right after SOI (decoy tables, ...); scan_order: SOS component order."""
    samp = SAMPLING[mode]
    nc = len(samp)
    shapes = planes_shape(width, height, mode)
    assert [tuple(c.shape) for c in coefs] == [s + (64,) for s in shapes], "planes must cover the padded MCU grid"
    if dc is None or ac is None:
        fdc, fac = flat_tables()
        dc, ac = dc or {0: fdc}, ac or {0: fac}
    sel = sel or [(0, 0)] * nc
    qt = qt or {0: [1] * 64}
    tq = tq or [0] * nc
    dcode = {t: dict(zip(v, codes(c))) for t, (c, v) in dc.items()}
    acode = {t: dict(zip(v, codes(c))) for t, (c, v) in ac.items()}
    hm, vm = samp[0] if nc == 3 else (1, 1)
    mcux, mcuy = shapes[0][1] // hm, shapes[0][0] // vm
    layout = [(c, bx, by) for c, (h, v) in enumerate(samp) for by in range(v if nc == 3 else 1)
              for bx in range(h if nc == 3 else 1)]
    mcus = mcux * mcuy
    per = restart if restart else mcus
    planes = [np.zeros(s + (64,), np.int16) for s in shapes]
    log, chunks, ibytes, bit0 = [], [], [], 0
    for m0 in range(0, mcus, per):
        vals, nbits, pred, pos = [], [], [0] * nc, 0

        def put(v, n, cls=None, comp=None, length=None):
            nonlocal pos
            if cls is not None:
                log.append((cls, comp, length, bit0 + pos))
            vals.append(v)
            nbits.append(n)
            pos += n

        for m in range(m0, min(mcus, m0 + per)):
            my, mx = divmod(m, mcux)
            for c, bx, by in layout:
                h, v = samp[c] if nc == 3 else (1, 1)
                r, col = my * v + by, mx * h + bx
                z = [int(x) for x in coefs[c][r, col]]
                planes[c][r, col, 0] = ((z[0] + 32768) & 0xFFFF) - 32768
                diff, pred[c] = z[0] - pred[c], z[0]
                s = abs(diff).bit_length()
                assert s <= 11, f"DC difference {diff} beyond category 11"
                code, l = dcode[sel[c][0]][s]
                put(code << s | (diff if diff >= 0 else diff + (1 << s) - 1) & ((1 << s) - 1), l + s, 0, c, l)
                table_ac = acode[sel[c][1]]
                last = max([k for k in range(1, 64) if z[k]], default=0)
                run = 0
                for k in range(1, last + 1):
                    if z[k] == 0:
                        run += 1
                        continue
                    planes[c][r, col, ZIGZAG[k]] = z[k]
                    while run >= 16:
                        code, l = table_ac[ZRL]
                        put(code, l, 1, c, l)
                        run -= 16
                    s = abs(z[k]).bit_length()
                    assert s <= 10, f"AC value {z[k]} beyond category 10"
                    code, l = table_ac[run << 4 | s]
                    put(code << s | (z[k] if z[k] > 0 else z[k] + (1 << s) - 1) & ((1 << s) - 1), l + s, 1, c, l)
                    run = 0
                if last < 63:
                    if zrl_end is not None and zrl_end[c][r, col]:
                        assert (last + 1) % 16 == 0, "a ZRL ending needs a multiple of 16 trailing zeros"
                        for _ in range((63 - last) // 16):
                            code, l = table_ac[ZRL]
                            put(code, l, 1, c, l)
                    else:
                        code, l = table_ac[EOB]
                        put(code, l, 1, c, l)
        packed = _pack(vals, nbits)
        ibytes.append(len(packed))
        bit0 += 8 * len(packed)
        chunks.append(packed.replace(b"\xff", b"\xff\x00"))
    raw, markers = bytearray(), []
    for i, ch in enumerate(chunks):
        if i:
            markers.append(len(raw))
            raw += bytes([0xFF, 0xD0 + (i - 1) % 8])
        raw += ch
    head = b"\xff\xd8" + before + segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for slot in sorted(qt):
        head += dqt(slot, qt[slot])
    ids = [1, 2, 3][:nc]
    sof = bytes([8, height >> 8, height & 255, width >> 8, width & 255, nc])
    for c in range(nc):
        h, v = samp[c] if nc == 3 else (1, 1)
        sof += bytes([ids[c], h << 4 | v, tq[c]])
    head += segment(0xC0, sof)
    for slot in sorted(dc):
        head += dht(0, slot, *dc[slot])
    for slot in sorted(ac):
        head += dht(1, slot, *ac[slot])
    if restart:
        head += segment(0xDD, bytes([restart >> 8, restart & 255]))
    order = scan_order or list(range(nc))
    head += segment(0xDA, bytes([nc]) + b"".join(bytes([ids[c], sel[c][0] << 4 | sel[c][1]]) for c in order)
                    + bytes([0, 63, 0]))
    data = head + bytes(raw) + b"\xff\xd9"
    return Stream(data, planes, np.array(log, np.int64).reshape(-1, 4), (len(head), len(head) + len(raw)), markers,
                  ibytes)


# ---- coefficient generators ---------------------------------------------------------------------------------------

def zeros(width, height, mode):
    return [np.zeros(s + (64,), np.int64) for s in planes_shape(width, height, mode)]


def value(rng, s):
    """A random value of magnitude category s >= 1."""
    m = int(rng.integers(1 << (s - 1), 1 << s))
    return m if rng.integers(0, 2) else -m


def fill_symbols(rng, block, symbols, n, zrl_every=0):
    """Puts up to n random AC (run, size) symbols from `symbols` into a zig-zag block from k = 1; every
    `zrl_every`-th symbol gets 16 more zeros before it (a ZRL).  Returns the next free index."""
    k = 1
    for i in range(n):
        rs = symbols[int(rng.integers(0, len(symbols)))]
        r = (rs >> 4) + (16 if zrl_every and i % zrl_every == zrl_every - 1 else 0)
        if k + r > 63:
            break
        k += r
        block[k] = value(rng, rs & 15)
        k += 1
    return k


def dc_walk(rng, n, categories=range(12)):
    """n absolute DC values whose differences take categories from `categories` at random; each step goes towards 0,
    so the values stay within +-2047 (a mean of at most 256 for a DC quantiser of 1: inside the IDCT's range)."""
    out, cur = [], 0
    for _ in range(n):
        s = int(rng.choice(list(categories)))
        d = abs(value(rng, s)) if s else 0
        cur = cur - d if cur > 0 or (cur == 0 and rng.integers(0, 2)) else cur + d
        out.append(cur)
    return out


def encoding_order(mode, plane, c):
    """(row, column) of component c's blocks of `plane` [blocks high, blocks wide, ...] in the order the scan codes
    them (MCU by MCU), so that DC differences are taken between neighbours in that order."""
    h, v = SAMPLING[mode][c] if mode != "L" else (1, 1)
    my, mx = plane.shape[0] // v, plane.shape[1] // h
    return [(m // mx * v + by, m % mx * h + bx) for m in range(mx * my) for by in range(v) for bx in range(h)]


def dc_fill(rng, co, mode, categories=range(12)):
    """Every block's DC from `dc_walk`, walked in encoding order per component."""
    for c, plane in enumerate(co):
        order = encoding_order(mode, plane, c)
        for (r, col), d in zip(order, dc_walk(rng, len(order), categories)):
            plane[r, col, 0] = d


# ---- the stream families of tests/test_jpeg_edges_*.py ------------------------------------------------------------

# AC symbols of the one-code-per-length table: sizes up to 3 keep every block inside the IDCT's range
LENGTH_SYMBOLS = [0x01, 0x02, 0x03, 0x11, 0x12, 0x21, 0x22, 0x31, 0x41, 0x51, 0x62, 0x81, 0xA3, 0xF1]


def code_length_stream(mode, w, h, seed):
    """One DC and one AC table with exactly one code of every length 1-16 (counts all 1; the all-ones 16-bit code
    unused).  AC: a seeded permutation of EOB, ZRL and LENGTH_SYMBOLS over the lengths, and every symbol drawn
    uniformly, so nearly half the AC codes take libjpeg's slow path (10-16 bits).  DC: categories 0-11 at lengths
    1-4 and 9-16 (the unusable categories 12-15 fill lengths 5-8)."""
    rng = np.random.default_rng(seed)
    acs = [EOB, ZRL] + LENGTH_SYMBOLS
    ac = table({s: l + 1 for l, s in enumerate(rng.permutation(acs).tolist())})
    dcl = [1, 2, 3, 4] + list(range(9, 17))
    dc = table({**{c: dcl[i] for i, c in enumerate(rng.permutation(12).tolist())}, 12: 5, 13: 6, 14: 7, 15: 8})
    co = zeros(w, h, mode)
    dc_fill(rng, co, mode)
    for c in co:
        for b in c.reshape(-1, 64):
            fill_symbols(rng, b, LENGTH_SYMBOLS, int(rng.integers(0, 12)), zrl_every=4)
    return write(w, h, mode, co, dc={0: dc}, ac={0: ac})


def sync_stream(mcux, mcuy, restart=0, split_tables=False):
    """4:4:4 where every block has the same code lengths: DC difference +1 / -1 alternating (category 1), five AC
    coefficients of +-1 at k = 1..5 and EOB, 58 bits with the flat tables.  With all three components on one table
    pair the code lengths repeat every block, so nothing in the bits tells which component a block belongs to.
    split_tables puts the chroma components on tables with other code lengths (a 65-bit block)."""
    rng = np.random.default_rng(mcux * 7 + mcuy)
    co = zeros(8 * mcux, 8 * mcuy, "444")
    per = restart or mcux * mcuy
    for m0 in range(0, mcux * mcuy, per):
        dcs = [0, 0, 0]
        for m in range(m0, min(m0 + per, mcux * mcuy)):
            for c in range(3):
                dcs[c] += 1 if (3 * (m - m0) + c) % 2 == 0 else -1
                blk = co[c][m // mcux, m % mcux]
                blk[0] = dcs[c]
                blk[1:6] = rng.choice([-1, 1], 5)
    fdc, fac = flat_tables()
    if not split_tables:
        return write(8 * mcux, 8 * mcuy, "444", co, restart=restart)
    cac = table({EOB: 9, ZRL: 9, **{(r << 4) | s: 9 for r in range(16) for s in range(1, 11)}})
    return write(8 * mcux, 8 * mcuy, "444", co, restart=restart, dc={0: fdc, 1: table({s: 5 for s in range(12)})},
                 ac={0: fac, 1: cac}, sel=[(0, 0), (1, 1), (1, 1)])


def dc_wrap_stream(mode, w, h, restart):
    """DC differences of +2047 for 40 blocks, -2047 for 80, +2047 for 40 (per component, counted from each
    restart): the prediction runs to +-81880, through +-32767 several times; only its 16-bit wrap is stored."""
    co = zeros(w, h, mode)
    samp = SAMPLING[mode]
    hm, vm = samp[0] if mode != "L" else (1, 1)
    mcux, mcuy = co[0].shape[1] // hm, co[0].shape[0] // vm
    per = restart or mcux * mcuy
    for c, (hc, vc) in enumerate(samp if mode != "L" else [(1, 1)]):
        for m0 in range(0, mcux * mcuy, per):
            n, dcv = 0, 0
            for m in range(m0, min(m0 + per, mcux * mcuy)):
                for by in range(vc):
                    for bx in range(hc):
                        dcv += 2047 if (n % 160) < 40 or (n % 160) >= 120 else -2047
                        co[c][(m // mcux) * vc + by, (m % mcux) * hc + bx, 0] = dcv
                        n += 1
    return write(w, h, mode, co, restart=restart)


def endings_stream(mode, w, h, seed):
    """Blocks ended by ZRL at k = 48 (no EOB), blocks whose coefficient 63 is nonzero (no EOB), DC-only blocks (EOB
    right after DC), and distinctive values (DC 777 - component, coefficient 63 = -3) in every block of the padded
    MCU grid outside the image."""
    rng = np.random.default_rng(seed)
    co = zeros(w, h, mode)
    samp = SAMPLING[mode]
    hm, vm = samp[0] if mode != "L" else (1, 1)
    zrl = []
    dc_fill(rng, co, mode, range(10))
    for c, plane in enumerate(co):
        hc, vc = samp[c] if mode != "L" else (1, 1)
        bw, bh = -(-(-(-w * hc // hm)) // 8), -(-(-(-h * vc // vm)) // 8)   # blocks holding real samples
        z = np.zeros(plane.shape[:2], bool)
        for i in range(plane.shape[0]):
            for j in range(plane.shape[1]):
                b, n = plane[i, j], i * plane.shape[1] + j
                if i >= bh or j >= bw:
                    b[0], b[63] = 777 - c, -3
                elif n % 3 == 1:
                    b[1:48] = rng.integers(-2, 3, 47)
                    b[47] = value(rng, 2)
                    z[i, j] = True
                elif n % 3 == 2:
                    fill_symbols(rng, b, [0x01, 0x11, 0x32], 5)
                    b[63] = value(rng, 1)
        zrl.append(z)
    return write(w, h, mode, co, zrl_end=zrl)


def per_component_stream(mode, w, h, seed):
    """Tables in slots 2 and 3, selectors swapped between the components, three quantisation tables (Tq 3 / 0 / 1)."""
    rng = np.random.default_rng(seed)
    fdc, fac = flat_tables()
    dc2 = table({c: [2, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12][c] for c in range(12)})
    ac2 = table({EOB: 2, 0x01: 3, 0x02: 4, **{(r << 4) | s: 10 for r in range(16) for s in range(1, 11)
                                            if (r << 4) | s not in (0x01, 0x02)}, ZRL: 10})
    q = np.arange(64)
    co = zeros(w, h, mode)
    dc_fill(rng, co, mode, range(10))
    for c in co:
        for b in c.reshape(-1, 64):
            fill_symbols(rng, b, [0x01, 0x02, 0x11, 0x21, 0x12], int(rng.integers(0, 8)), zrl_every=3)
    return write(w, h, mode, co, dc={2: dc2, 3: fdc}, ac={0: fac, 2: ac2}, sel=[(3, 2), (2, 0), (3, 0)][:len(co)],
                 qt={0: 1 + q % 3, 1: 2 + q % 2, 3: 1 + (q // 8) % 3}, tq=[3, 0, 1][:len(co)])


DENSE_AC = table({**{s: l + 1 for l, s in enumerate([0x11, 0x21, 0x31, 0x41, 0x51, 0x61, 0x71, 0x81])},
                  0x01: 9, 0x02: 10, 0x03: 11, 0x06: 12, EOB: 13, ZRL: 14, 0x04: 15, 0x05: 16})
DENSE_DC = table({**{c: c for c in range(1, 12)}, 0: 12, 12: 13, 13: 14, 14: 15, 15: 16})


def dense_stream(mcus, restart=0, extra=(0, 0, 0)):
    """Gray, mostly 1-bits, so 0xFF bytes (and their stuffing) are frequent: DC difference 0 on an 11-ones code, three
    AC values of 63 on 11-ones codes with 6 one-bits each, EOB of 12 ones.  `extra` adds (+1, +3, +7) values to the
    first block (10, 12 and 14 bits each) to move every later byte by a few bits."""
    co = zeros(8 * mcus, 8, "L")
    co[0][:, :, 1:4] = 63
    k = 4
    for n, v in zip(extra, (1, 3, 7)):
        co[0][0, 0, k:k + n] = v
        k += n
    return write(8 * mcus, 8, "L", co, dc={0: DENSE_DC}, ac={0: DENSE_AC}, restart=restart)


def idct_boundary_streams():
    """(name, 8 x 8 gray stream, status) on both sides of the IDCT-range flag: a DC-only block with a DC quantiser of
    4 (mean DC * 4 / 8: outputs 511 / 512 and -512 / -513), and one AC coefficient at zig-zag 1 with a quantiser of
    4, whose largest outputs leave [-512, 512) between 737 and 738."""
    rows = []
    for name, k, v, q, status in (("dc 1022", 0, 1022, 4, 0), ("dc 1023", 0, 1023, 4, 32),
                                  ("dc -1025", 0, -1025, 4, 0), ("dc -1026", 0, -1026, 4, 32),
                                  ("ac 737", 1, 737, 4, 0), ("ac 738", 1, 738, 4, 32),
                                  ("ac -737", 1, -737, 4, 0), ("ac -738", 1, -738, 4, 32)):
        co = zeros(8, 8, "L")
        co[0][0, 0, k] = v
        qt = np.ones(64, np.int64)
        qt[ZIGZAG[k]] = q
        rows.append((name, write(8, 8, "L", co, qt={0: qt}), status))
    return rows
