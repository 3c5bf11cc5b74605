"""GPU: the device JPEG decode (csrc/jpeg.cu) where parallel Huffman decoders go wrong, on streams written coefficient by
coefficient (tests/jpeg_writer.py): codes of every length 1-16 at odd subsequence lengths, the synchronisation's worst
case, more than 1,024 scan tiles, DC predictions past +-32767, blocks ended without EOB, per-component tables in any
slot, stuffing and markers across the segment kernels' chunk and thread-slice edges, both sides of the IDCT-range flag,
and seeded corrupt streams.

"Coefficients" is `mhmr_op_jpeg_coefficients` called directly into a sentinel-filled buffer with a guard band past the
last plane (the op clears exactly its own planes): they must equal the writer's planes with status 0 and the guard
intact.  "Pixels" is `mhmr_op_jpeg_decode` into guard-banded frames: they must equal Pillow's."""
import io
import itertools
import time

import numpy as np
import pytest
import torch

import jpeg_util as ju
import jpeg_writer as jw
from oracle import jpeg_ref as jr

pytestmark = pytest.mark.gpu

SENTINEL, GUARD = -21846, 4096


def _coefficients(blobs, subseq_bits, device):
    """(per photo, per component int16 [blocks high, blocks wide, 64] numpy planes, statuses, sync passes)."""
    from multihmr_b200 import ops, preprocess
    from multihmr_b200._lib import call, stream

    host, dev, spans = preprocess.upload_bytes(blobs, device)
    infos = [ops.jpeg_info(b) for b in blobs]
    assert all(i[5] for i in infos)
    shapes = [ops.jpeg_plane_blocks(*i[:5]) for i in infos]
    total = sum(bw * bh * 64 for p in shapes for bw, bh in p)
    buf = torch.full((total + GUARD,), SENTINEL, dtype=torch.int16, device=device)
    status = torch.full((len(blobs),), -1, dtype=torch.int32, device=device)
    passes = torch.zeros(1, dtype=torch.int32, device=device)
    desc = ops._jpeg_desc(host, dev, spans, [(i[1], i[0]) for i in infos], None)
    with torch.cuda.device(device):
        call("mhmr_op_jpeg_coefficients", desc, len(spans), subseq_bits, buf, status, passes, stream())
    out = buf.cpu().numpy()
    assert (out[total:] == SENTINEL).all(), "a coefficient write left the planes"
    planes, pos = [], 0
    for p in shapes:
        planes.append([])
        for bw, bh in p:
            planes[-1].append(out[pos:pos + bw * bh * 64].reshape(bh, bw, 64))
            pos += bw * bh * 64
    return planes, status.cpu().tolist(), int(passes.item())


def _check_coefficients(streams, subseq_bits, device, what):
    planes, status, passes = _coefficients([s.data for s in streams], subseq_bits, device)
    assert status == [0] * len(streams), (what, subseq_bits, status)
    for i, (s, got) in enumerate(zip(streams, planes)):
        for c, (g, want) in enumerate(zip(got, s.planes)):
            assert np.array_equal(g, want), (what, subseq_bits, i, c, int((g != want).sum()))
    return passes


def _pixels(blobs, device):
    """(device RGB of every file as numpy, statuses) from one `ops.jpeg_decode` into guard-banded frames."""
    from multihmr_b200 import ops, preprocess

    host, dev, spans = preprocess.upload_bytes(blobs, device)
    frames, outs = [], []
    for b in blobs:
        w, h = ops.jpeg_info(b)[:2]
        frame = torch.full((h + 2, w + 5, 3), 0x5A, dtype=torch.uint8, device=device)
        frames.append(frame)
        outs.append(frame[1:h + 1, 2:w + 2])
    status = ops.jpeg_decode(host, dev, spans, outs).cpu().tolist()
    got = []
    for frame, out in zip(frames, outs):
        h, w = out.shape[:2]
        guard = frame.clone()
        guard[1:h + 1, 2:w + 2] = 0x5A
        assert bool((guard == 0x5A).all()), "a pixel write left the photo's box"
        got.append(out.cpu().numpy())
    return got, status


def _check_pixels(blobs, device, what):
    got, status = _pixels(blobs, device)
    assert status == [0] * len(blobs), (what, status)
    for i, (g, b) in enumerate(zip(got, blobs)):
        assert np.array_equal(g, ju.pillow_rgb(b)), (what, i)


def _subsequences(stream, subseq_bits):
    """The device's subsequence count: every restart interval cut into subsequence_bits pieces, at least one."""
    return sum(max(1, -(-8 * n // subseq_bits)) for n in stream.interval_bytes)


def test_codes_of_every_length_at_odd_subsequence_lengths(cuda_device):
    streams = [jw.code_length_stream(m, 192, 128, 10 + i) for i, m in enumerate(ju.MODES)]
    for m, s in zip(ju.MODES, streams):
        ac, dc = s.log[s.log[:, 0] == 1], s.log[s.log[:, 0] == 0]
        assert set(ac[:, 2].tolist()) == set(range(1, 17)), m
        assert set(dc[:, 2].tolist()) == set(range(1, 5)) | set(range(9, 17)), m
        assert (s.log[:, 2] >= 10).sum() >= 1000, m
        assert set((s.log[:, 3] % 32).tolist()) == set(range(32)), m
        assert set((s.log[s.log[:, 2] >= 10, 3] % 32).tolist()) == set(range(32)), m
        print(f"{m}: {len(s.log)} codes, {(s.log[:, 2] >= 10).sum()} of 10-16 bits, every bit offset mod 32")
    for bits in (1, 3, 7, 31, 32, 33, 257, 1024):
        passes = _check_coefficients(streams, bits, cuda_device, "code lengths")
        print(f"subsequence {bits} bits: {sum(_subsequences(s, bits) for s in streams)} subsequences, {passes} passes")
    _check_pixels([s.data for s in streams], cuda_device, "code lengths")


def test_worst_case_synchronisation(cuda_device):
    """4:4:4 on one table pair, every block 58 bits (jw.sync_stream), cut into 58-bit subsequences.  Subsequence j
    starts on block j's DC code, where pass 0 guesses the MCU's first block: wrong unless j = 0 mod 3, and nothing
    in the bits corrects it, since all blocks have the same code lengths.  A chain of guessed states advances its block
    of the MCU by one per subsequence, as the true state does, so it never meets the true state; and at a fixed
    subsequence it comes from one subsequence further left each pass, so its block of the MCU changes every pass.
    Only the chain from the interval's exact first subsequence is right, and it reaches subsequence p at pass p.  So
    pass p changes a start state for every p < nsub, and pass nsub is the first that changes none: passes == nsub
    exactly (per restart interval: the largest interval's subsequence count).  The DC sums must still land on the
    right component.  With chroma tables of other code lengths, the guesses lock on far sooner."""
    timings = {}

    def run(s, bits):
        torch.cuda.synchronize()
        t = time.perf_counter()
        passes = _check_coefficients([s], bits, cuda_device, "sync")
        timings[len(timings)] = time.perf_counter() - t
        return passes

    s = jw.sync_stream(40, 25)
    nsub = _subsequences(s, 58)
    assert nsub == 3000 and s.interval_bytes == [3000 * 58 // 8]
    run(s, 58)   # warm-up of the module and the allocator
    passes = run(s, 58)
    print(f"one interval: {nsub} subsequences, {passes} passes ({passes / nsub:.3f} nsub), {timings[1] * 1e3:.1f} ms")
    assert passes == nsub
    r = jw.sync_stream(40, 25, restart=100)
    per = max(max(1, -(-8 * n // 58)) for n in r.interval_bytes)
    rp = run(r, 58)
    print(f"restart every 100 MCUs: {len(r.interval_bytes)} intervals of {per} subsequences, {rp} passes")
    assert rp == per
    split = jw.sync_stream(40, 25, split_tables=True)
    sp = run(split, 58)
    print(f"chroma tables of other code lengths: {_subsequences(split, 58)} subsequences, {sp} passes "
          f"(against {passes} on one table pair)")
    assert sp < passes
    for bits in (57, 59, 1024):
        print(f"one table pair at {bits} bits: {_subsequences(s, bits)} subsequences, "
              f"{_check_coefficients([s], bits, cuda_device, 'sync')} passes")


def _scale_stream(seed):
    """2048 x 1024 gray, a restart marker after every MCU: 32,768 intervals of 21 destuffed bytes (DC of category
    11, eight AC values of category 10, EOB)."""
    rng = np.random.default_rng(seed)
    co = jw.zeros(2048, 1024, "L")
    mag = rng.integers(1024, 2048, co[0].shape[:2])
    co[0][:, :, 0] = np.where(rng.integers(0, 2, mag.shape) == 1, mag, -mag)
    ac = rng.integers(512, 1024, co[0].shape[:2] + (8,))
    co[0][:, :, 1:9] = np.where(rng.integers(0, 2, ac.shape) == 1, ac, -ac)
    return jw.write(2048, 1024, "L", co, restart=1)


def test_more_subsequences_than_scan_tiles_and_sync_threads(cuda_device):
    """More than 1,024 tiles of 1,024 subsequences (the tile scan's outer loop) and more than the 270,336 threads a
    132-SM cooperative grid holds (the sync kernel's grid-stride loop); short intervals bound the passes."""
    streams = [_scale_stream(0), _scale_stream(1)]
    for bits in (8, 1):
        nsub = sum(_subsequences(s, bits) for s in streams)
        bound = sum(-(-8 * (s.ecs[1] - s.ecs[0]) // bits) + len(s.interval_bytes) for s in streams)
        per = max(-(-8 * n // bits) for s in streams for n in s.interval_bytes)
        assert nsub > 1024 * 1024 and nsub > 132 * 2048 and nsub <= bound
        passes = _check_coefficients(streams, bits, cuda_device, "scale")
        print(f"{bits} bits: {nsub} subsequences (host bound {bound}), {-(-nsub // 1024)} tiles, {passes} passes, "
              f"{per} subsequences in the longest interval")
        assert passes <= per + 1


@pytest.mark.parametrize("mode", ["L", "420"])
def test_dc_predictions_past_int16(mode, cuda_device):
    """DC sums through +-32767 several times, restarts 37 MCUs apart (inside the runs), subsequences cut inside the
    runs; the pixels are IDCT-flagged."""
    streams = [jw.dc_wrap_stream(mode, 256, 64, r) for r in (0, 37)]
    for s in streams:
        for plane in s.planes:
            assert {32752, -30737} <= set(plane[:, :, 0].ravel().tolist())
    for bits in (1, 13, 1024):
        print(f"{mode}, {bits} bits: {_check_coefficients(streams, bits, cuda_device, 'dc wrap')} passes")
    _, status = _pixels([s.data for s in streams], cuda_device)
    assert status == [jr.IDCT_RANGE] * 2


def test_blocks_without_eob_and_padded_mcus(cuda_device):
    """ZRL to coefficient 64, coefficient 63 nonzero, EOB right after DC; distinctive padding blocks; 257 and 2049
    also cross the colour kernel's 256-wide x-blocks and 1,024-row grid."""
    streams = [jw.endings_stream(m, w, h, i) for i, m in enumerate(ju.MODES)
               for w, h in ((17, 9), (31, 1025), (257, 2049))]
    _check_coefficients(streams, 1024, cuda_device, "endings")
    _check_coefficients(streams[:3], 33, cuda_device, "endings")
    _check_pixels([s.data for s in streams], cuda_device, "endings")
    print(f"{len(streams)} streams, {sum(len(s.log) for s in streams)} codes")


def test_per_component_tables(cuda_device):
    streams = [jw.per_component_stream(m, 301, 199, i) for i, m in enumerate(["444", "422", "420"])]
    _check_coefficients(streams, 1024, cuda_device, "tables")
    _check_pixels([s.data for s in streams], cuda_device, "tables")


def _first(pred, **kw):
    """The first dense stream, over the first block's extra values, that satisfies pred (None if none does)."""
    for extra in itertools.product(range(6), repeat=3):
        s = jw.dense_stream(extra=extra, **kw)
        if pred(s):
            return s
    return None


def test_stuffing_and_markers_across_chunk_and_slice_edges(cuda_device):
    """Mostly-ones streams whose first interval is tuned so that a stuffed FF|00 and an FF|RSTn straddle raw offsets
    4095|4096 (two 4 KB segment chunks), and an FF|00 straddles a 16-byte thread slice inside a chunk; plus a Pillow
    photo of more than 1,024 chunks."""
    ff00 = _first(lambda s: s.raw[4095:4097] == b"\xff\x00", mcus=500)
    lo, hi = 1, 600   # the largest restart interval whose first interval ends at or before 4095
    while lo < hi:
        r = (lo + hi + 1) // 2
        lo, hi = (r, hi) if jw.dense_stream(2 * r, r).markers[0] <= 4095 else (lo, r - 1)
    for r in (lo, lo - 1, lo - 2):
        marker = _first(lambda s: s.markers[0] == 4095, mcus=2 * r, restart=r)
        if marker is not None:
            break
    assert ff00 is not None and marker is not None
    assert marker.raw[4095] == 0xFF and 0xD0 <= marker.raw[4096] <= 0xD7
    slices = [i for i in range(15, len(ff00.raw) - 1, 16) if ff00.raw[i:i + 2] == b"\xff\x00" and (i + 1) % 4096]
    assert slices
    big = ju.encode(ju.photo(2048, 1024, 5), "444", quality=100)
    s, e = ju.ecs_span(big)
    assert e - s > 4 << 20 and -(-(e - s) // 4096) > 1024
    print(f"FF|00 at 4095|4096, FF|{marker.raw[4096]:02X} at 4095|4096, FF|00 across {len(slices)} slice edges, "
          f"{-(-(e - s) // 4096)} chunks of {(e - s) / 2 ** 20:.1f} MiB")
    for bits in (1, 1024):
        _check_coefficients([ff00, marker], bits, cuda_device, "dense")
    _check_pixels([ff00.data, marker.data, big], cuda_device, "dense")


def test_idct_range_flag_boundary(cuda_device):
    rows = jw.idct_boundary_streams()
    got, status = _pixels([s.data for _, s, _ in rows], cuda_device)
    for (name, s, want), g, st in zip(rows, got, status):
        assert st == want == jr.decode(s.data)[1], (name, st)
        if st == 0:
            assert np.array_equal(g, ju.pillow_rgb(s.data)), name
    print(f"{sum(map(bool, status))} flagged, {status.count(0)} exact")


def _first_bit(data, status):
    """The first anomaly the restatement finds, as the device must report it.  RSTn markers are checked before any
    entropy data is decoded: past a wrong marker the two split the data differently (the restatement at every marker,
    the device at the first intervals - 1), so only that bit is common.  The restatement then stops at the first entropy
    anomaly; if its bit reader had passed the interval's data there, it was decoding zeros where the device decodes the
    next interval's bytes, and the device's bit is SHORT_DATA (its last block cannot end inside the data)."""
    if status & jr.BAD_RST:
        return jr.BAD_RST
    if status & (jr.BAD_CODE | jr.BAD_SIZE | jr.BAD_RUN):
        last = ju.bit_readers(data)[-1]
        if last.pos > last.n:
            return jr.SHORT_DATA
    return status & -status


def test_corrupt_streams_on_the_device(cuda_device):
    """The shared seeded corruptions over four samplings and restart intervals 0 / 1 / 2 / 7, in one call: the
    device flags a file exactly when the restatement does, with the restatement's first anomaly (`_first_bit`);
    unflagged files equal Pillow's pixels and the restatement's coefficients; no write leaves a photo's box."""
    from PIL import Image

    from multihmr_b200 import ops

    files = []
    for i, (mode, restart) in enumerate(itertools.product(ju.MODES, (0, 1, 2, 7))):
        data = ju.encode(ju.photo(48, 40, i), mode, quality=75, **({"restart_marker_blocks": restart} if restart else {}))
        for what, bad in ju.corruptions(np.random.default_rng(100 + i), data):
            if ops.jpeg_info(bad)[5]:
                files.append((mode, restart, what, bad, jr.decode(bad)[1]))
    got, status = _pixels([f[3] for f in files], cuda_device)
    exact, flagged, needed, overrun = [], 0, 0, 0
    for (mode, restart, what, bad, want), g, st in zip(files, got, status):
        assert (st != 0) == (want != 0), (mode, restart, what, st, want)
        if want:
            flagged += 1
            first = _first_bit(bad, want)
            overrun += first != want & -want
            assert st & first, (mode, restart, what, st, want)
            try:
                pil = np.asarray(Image.open(io.BytesIO(bad)).convert("RGB"))
            except Exception:
                continue
            needed += not np.array_equal(g, pil)
            continue
        assert np.array_equal(g, ju.pillow_rgb(bad)), (mode, restart, what)
        exact.append(bad)
    planes, cstatus, _ = _coefficients(exact, 1024, cuda_device)
    assert cstatus == [0] * len(exact)
    for b, p in zip(exact, planes):
        want, _ = jr.decode_coefficients(b, jr.parse(b))
        assert all(np.array_equal(x, y) for x, y in zip(p, want))
    print(f"{len(files)} eligible files: {flagged} flagged ({needed} whose raw device pixels differ from Pillow's, "
          f"{overrun} whose first bit is not the restatement's lowest), {len(exact)} exact")
    assert flagged and exact and needed
