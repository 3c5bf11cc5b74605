"""GPU: the device inflate (`mhmr_op_png_inflate`) equals Python's zlib on every stream family of tests/png_writer.py,
flags the streams zlib refuses, follows the worst case (a stream of fixed-Huffman blocks) to the exact bytes, and
matches oracle/png_ref.py's status file for file on a seeded fuzz of PNG files."""
import random
import zlib

import numpy as np
import pytest
import torch

import png_util as U
import png_writer as pw
from oracle import png_ref as R

pytestmark = pytest.mark.gpu


def _inflate(streams, lengths, cuda_device):
    from multihmr_b200 import ops, preprocess

    _, dev, spans = preprocess.upload_bytes(streams, cuda_device)
    outs, status, counts = ops.png_inflate(dev, spans, lengths)
    return [o.cpu().numpy().tobytes() for o in outs], status.cpu().tolist(), counts.cpu().tolist()


def test_writer_streams_equal_zlib(cuda_device):
    fam = U.stream_families()
    lengths = [len(d) if d is not None else 100 for _, _, d in fam]
    outs, status, counts = _inflate([s for _, s, _ in fam], lengths, cuda_device)
    for (name, s, d), o, st, c, n in zip(fam, outs, status, counts, lengths):
        want = R.inflate(s, n)[0]
        assert st == want, name
        if d is None:
            with pytest.raises(zlib.error):
                zlib.decompress(s)
            assert st != 0, name
        else:
            assert st == 0 and o == d == zlib.decompress(s), name
            assert c[3] == len(d) and c[0] == R.inflate(s, n)[2], name
    planted = [c for (name, _, _), c in zip(fam, counts) if name == "planted-header"][0]
    assert planted[1] > planted[0] - planted[2], "the planted header is a candidate the chain never uses"


def test_zlib_levels_strategies_and_idat_splits(cuda_device):
    rng = np.random.default_rng(9)
    raw = U.photo(rng, 300, 400, 3).tobytes()
    streams = []
    for lvl in range(10):
        streams.append(zlib.compress(raw, lvl))
    for st in (zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED):
        c = zlib.compressobj(6, zlib.DEFLATED, 15, 9, st)
        streams.append(c.compress(raw) + c.flush())
    outs, status, counts = _inflate(streams, [len(raw)] * len(streams), cuda_device)
    assert status == [0] * len(streams)
    assert all(o == raw for o in outs)


def test_fixed_huffman_worst_case(cuda_device):
    """Z_FIXED at 1280 x 720 RGB: every block is on the slow path of the chain, the bytes stay exact."""
    rng = np.random.default_rng(1)
    raw = U.photo(rng, 720, 1280 * 3 + 1, 1).tobytes()[:720 * (1 + 1280 * 3)]
    c = zlib.compressobj(6, zlib.DEFLATED, 15, 8, zlib.Z_FIXED)
    s = c.compress(raw) + c.flush()
    outs, status, counts = _inflate([s], [len(raw)], cuda_device)
    assert status == [0] and outs[0] == raw
    assert counts[0][2] == counts[0][0] > 1


def test_idat_split_into_tiny_and_empty_chunks(cuda_device):
    rng = np.random.default_rng(2)
    px = U.photo(rng, 12, 9, 3)
    base = pw.make_png(px, 2, filters=[y % 5 for y in range(12)])
    z = R.parse(base)["stream"]
    stored, _ = pw.zstream([("stored", pw.filter_rows(px.reshape(12, 27), 3, [1] * 12))])
    files = [pw.png_file(9, 12, 2, z, idat_sizes=[1] * len(z)),
             pw.png_file(9, 12, 2, z, idat_sizes=[0, 3, 0, 0, 5, 1, 0]),
             pw.png_file(9, 12, 2, stored, idat_sizes=[7, 50, 1])]   # a stored block straddling IDAT chunks
    from multihmr_b200 import preprocess

    photos, ok = preprocess.decode_png(files, cuda_device)
    for f, p, good in zip(files, photos, ok):
        assert good and np.array_equal(p.cpu().numpy(), U.pillow(f))


def test_fuzz_device_status_equals_the_restatement(cuda_device):
    """Corrupt files are data: the device flags them exactly as the restatement does, and where it does not flag,
    its photo is Pillow's (which then never raised)."""
    from multihmr_b200 import ops, preprocess

    rng = random.Random(1234)
    nrng = np.random.default_rng(4)
    bases = [U.pillow_png(U.photo(nrng, 9 + i, 13 + 2 * i, pw.CHANNELS[ct]), ct) for i, ct in
             enumerate([0, 2, 3, 4, 6, 2, 2, 6])]
    bases.append(pw.make_png(U.photo(nrng, 8, 8, 3), 2, strategy=zlib.Z_FIXED))
    files = []
    for i in range(400):
        b = bases[i % len(bases)]
        h = R.parse(b)
        s, _ = U.corrupt(h["stream"], rng)
        files.append(pw.png_file(h["W"], h["H"], h["ctype"], s, palette=bytes(h["palette"].reshape(-1))
                                 if h["ctype"] == 3 else None))
    photos, ok = preprocess.decode_png(files, cuda_device)
    host, dev, spans = preprocess.upload_bytes([ops.png_idat(f) for f in files], cuda_device)
    outs = [torch.empty((ops.png_info(f)[1], ops.png_info(f)[0], 3), dtype=torch.uint8, device=cuda_device)
            for f in files]
    status = ops.png_decode(files, host, dev, spans, outs).cpu().tolist()
    flagged_but_accepted = 0
    for f, p, good, st in zip(files, photos, ok, status):
        want, rgb = R.decode(f)
        assert st == want
        ref = U.pillow(f)
        if good:
            assert isinstance(ref, np.ndarray) and np.array_equal(p.cpu().numpy(), ref)
        elif isinstance(ref, np.ndarray):
            flagged_but_accepted += 1
    print(f"fuzz: {sum(ok)} exact, {len(files) - sum(ok)} flagged, of which Pillow decoded {flagged_but_accepted}")
