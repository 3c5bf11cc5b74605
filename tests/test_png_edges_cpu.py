"""CPU: the restatement's inflate (oracle/png_ref.py) against Python's zlib on the stream families of
tests/png_writer.py, written straight from RFC 1950 / 1951 (stored, fixed and dynamic blocks, 15-bit codes, one
distance code, repeats across the literal / length -> distance boundary, every length and distance class, overlapping
copies, copies of copies across blocks, one-symbol blocks, a valid header planted inside stored data, a distance one
byte too far back), the same streams as PNG files with IDAT split into 1-byte and empty chunks against Pillow, and a
seeded fuzz: the restatement never returns bytes where Pillow raises, and where it does not flag it returns Pillow's."""
import random
import zlib

import numpy as np
import pytest

import png_util as U
import png_writer as pw
from oracle import png_ref as R

FAMILIES = U.stream_families()


@pytest.mark.parametrize("name, stream, data", FAMILIES, ids=[n for n, _, _ in FAMILIES])
def test_inflate_equals_zlib(name, stream, data):
    if data is None:
        with pytest.raises(zlib.error):
            zlib.decompress(stream)
        assert R.inflate(stream, 100)[0] == R.BAD_DIST
        return
    assert zlib.decompress(stream) == data
    status, out, nblocks = R.inflate(stream, len(data))
    assert status == 0 and out == data and nblocks >= 1
    assert R.inflate(stream, len(data) + 1)[0] == R.BAD_LENGTH
    if len(data) > 1:
        assert R.inflate(stream, len(data) - 1)[0] == R.BAD_LENGTH


@pytest.mark.parametrize("name, stream, data", [f for f in FAMILIES if f[2]], ids=[n for n, _, d in FAMILIES if d])
def test_families_as_png_files_equal_pillow(name, stream, data):
    """The family's bytes as a gray image of one row (filter 0 plus the bytes), IDAT in 1-byte and empty chunks."""
    raw = b"\0" + data
    s, _ = pw.zstream([("stored", raw[:1]), ("dynamic", list(raw[1:]) if len(raw) < 4000 else [])]
                      if len(raw) < 4000 else [("stored", raw)])
    sizes = [1, 0, 2, 0, 0] * (len(s) // 3 + 1)
    f = pw.png_file(len(data), 1, 0, s, idat_sizes=sizes[:len(s)])
    status, rgb = R.decode(f)
    assert status == 0 and np.array_equal(rgb, U.pillow(f))


def _fuzz_bases():
    rng = np.random.default_rng(4)
    bases = [U.pillow_png(U.photo(rng, 9 + i, 13 + 2 * i, pw.CHANNELS[ct]), ct)
             for i, ct in enumerate([0, 2, 3, 4, 6, 2])]
    bases.append(pw.make_png(U.photo(rng, 8, 8, 3), 2, strategy=zlib.Z_FIXED))
    bases.append(pw.make_png(U.photo(rng, 6, 7, 3), 2, level=0))
    return bases


def test_fuzz_never_returns_bytes_where_pillow_raises():
    rng = random.Random(99)
    bases = _fuzz_bases()
    counts = {"exact": 0, "flagged_pillow_raises": 0, "flagged_pillow_decodes": 0}
    kinds = {}
    for i in range(600):
        b = bases[i % len(bases)]
        h = R.parse(b)
        s, kind = U.corrupt(h["stream"], rng)
        f = pw.png_file(h["W"], h["H"], h["ctype"], s,
                        palette=bytes(h["palette"].reshape(-1)) if h["ctype"] == 3 else None)
        status, rgb = R.decode(f)
        ref = U.pillow(f)
        if status == 0:
            assert isinstance(ref, np.ndarray) and np.array_equal(rgb, ref), (i, kind)
            counts["exact"] += 1
        elif isinstance(ref, np.ndarray):
            counts["flagged_pillow_decodes"] += 1
            kinds[(kind, status)] = kinds.get((kind, status), 0) + 1
        else:
            counts["flagged_pillow_raises"] += 1
    # Flagged files Pillow still decodes are the ones whose damage Pillow never reads: zlib stops once the last row
    # is out (trailing blocks, a damaged or missing Adler-32 in input it is not given), or the stream ends early with
    # Z_STREAM_END (Pillow keeps the rows it has).  They go to Pillow, which decodes them as before.
    print(counts, kinds)
    assert counts["flagged_pillow_raises"] > 0
