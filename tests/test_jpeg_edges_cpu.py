"""CPU: streams written coefficient by coefficient (tests/jpeg_writer.py) reach what Pillow-encoded photos reach only
by chance: Huffman codes of every length 1-16 in any table slot, swapped selectors, DC predictions past +-32767, blocks
ended without EOB, and the IDCT-range flag on both sides of its boundary.  Each one is eligible to the device's header
parser and the restatement (oracle/jpeg_ref.py), decodes to exactly the writer's coefficients, and to Pillow's pixels."""
import numpy as np
import pytest

import jpeg_util as ju
import jpeg_writer as jw
from oracle import jpeg_ref as jr


@pytest.fixture(scope="module", autouse=True)
def _libjpeg_turbo():
    from PIL import features

    if not features.check_feature("libjpeg_turbo"):
        pytest.skip("Pillow's JPEG backend is not libjpeg-turbo: the restatement pins libjpeg-turbo's arithmetic")


def _check(stream, what, status=0):
    """Eligible to both parsers, the writer's coefficients exactly, and Pillow's pixels unless flagged."""
    from multihmr_b200 import ops

    data = stream.data
    info = ops.jpeg_info(data)
    assert info[5] == 1 and jr.info(data)[4], what
    assert info[:5] == jr.info(data)[:3] + jr.info(data)[3], what
    coefs, st = jr.decode_coefficients(data, jr.parse(data))
    assert st == 0, (what, st)
    for c, (got, want) in enumerate(zip(coefs, stream.planes)):
        assert np.array_equal(got, want), (what, c)
    px, st = jr.decode(data)
    assert st == status, (what, st)
    if status == 0:
        assert np.array_equal(px, ju.pillow_rgb(data)), what


def _lengths(stream, cls):
    return set(stream.log[stream.log[:, 0] == cls, 2].tolist())


@pytest.mark.parametrize("mode", ju.MODES)
def test_codes_of_every_length_decode_exactly(mode):
    s = jw.code_length_stream(mode, 64, 48, ju.MODES.index(mode))
    _check(s, mode)
    assert _lengths(s, 1) == set(range(1, 17)), "every AC code length"
    assert _lengths(s, 0) == set(range(1, 5)) | set(range(9, 17)), "every usable DC code length"
    print(f"{mode}: {len(s.log)} codes, {(s.log[:, 2] >= 10).sum()} of 10-16 bits")


@pytest.mark.parametrize("mode", ju.MODES)
@pytest.mark.parametrize("restart", [0, 23])
def test_dc_predictions_past_int16_are_stored_wrapped(mode, restart):
    """The DC sum runs past 32767 in every component (16 and 17 times 2047 are stored as 32752 and -30737), also
    between restarts 23 MCUs apart; the blocks' pixels are IDCT-flagged."""
    s = jw.dc_wrap_stream(mode, 128, 48, restart)
    _check(s, (mode, restart), status=jr.IDCT_RANGE)
    for plane in s.planes:
        assert {32752, -30737} <= set(plane[:, :, 0].ravel().tolist())


def test_dc_sum_wraps_like_libjpeg():
    """40 differences of +2047: blocks 14-17 hold the int16 wrap of the running sum."""
    co = jw.zeros(8 * 40, 8, "L")
    co[0][0, :, 0] = 2047 * np.arange(1, 41)
    s = jw.write(8 * 40, 8, "L", co)
    coefs, st = jr.decode_coefficients(s.data, jr.parse(s.data))
    assert st == 0 and coefs[0][0, 14:18, 0].tolist() == [30705, 32752, -30737, -28690]
    assert np.array_equal(coefs[0], s.planes[0])


@pytest.mark.parametrize("mode", ju.MODES)
@pytest.mark.parametrize("w, h", [(17, 9), (31, 33)])
def test_blocks_without_eob_and_padded_mcus(mode, w, h):
    s = jw.endings_stream(mode, w, h, 3)
    _check(s, (mode, w, h))
    zz63 = s.planes[0][:, :, 63]
    assert (zz63 != 0).any() and (s.planes[0][:, :, 1:] == 0).all(-1).any()


@pytest.mark.parametrize("mode", ["444", "422", "420"])
def test_per_component_tables_in_any_slot(mode):
    _check(jw.per_component_stream(mode, 40, 24, 1), mode)


def test_worst_case_sync_streams():
    _check(jw.sync_stream(6, 5), "one table pair")
    _check(jw.sync_stream(6, 5, restart=4, split_tables=True), "split tables")


def test_dense_ones_stream():
    s = jw.dense_stream(40, restart=7, extra=(3, 2, 1))
    _check(s, "dense")
    assert s.raw.count(b"\xff\x00") > len(s.raw) // 4


def test_idct_range_flag_is_needed_and_tight():
    """Each flagged row is one step past an unflagged one, and there Pillow's byte (its SIMD IDCT saturates) differs
    from the C IDCT's wrapped byte: the flag is needed, and fires no earlier.  A pass-1 value can not be pushed out of
    int16 with the outputs in range: an 8-point row of the second pass carries the energy of its pass-1 values, so
    one pass-1 value of 32768 puts an output of its row past 32768 / 32 = 1024, twice the output bound."""
    for name, s, status in jw.idct_boundary_streams():
        _check(s, name, status)
        px, _ = jr.decode(s.data)
        want = ju.pillow_rgb(s.data)
        differs = int((px != want).sum())
        print(f"{name}: status {status}, Pillow {want[:, :, 0].min()}..{want[:, :, 0].max()}, {differs} bytes differ")
        assert (differs > 0) == (status != 0), name
    rows = {n: s for n, s, _ in jw.idct_boundary_streams()}
    assert ju.pillow_rgb(rows["dc 1023"].data)[0, 0, 0] == 255 and jr.decode(rows["dc 1023"].data)[0][0, 0, 0] == 0
    assert ju.pillow_rgb(rows["dc -1026"].data)[0, 0, 0] == 0 and jr.decode(rows["dc -1026"].data)[0][0, 0, 0] == 255


def test_header_classification_of_written_files():
    from multihmr_b200 import ops

    co = jw.zeros(40, 24, "444")
    jw.dc_fill(np.random.default_rng(0), co, "444", range(8))
    base = jw.write(40, 24, "444", co)
    _, fac = jw.flat_tables()
    decoys = (jw.dqt(0, [9] * 64) + jw.dht(0, 0, *jw.table({s: 5 for s in range(12)}))
              + jw.dht(1, 0, *jw.table({s: 9 for s in fac[1]})))
    rows = [("slots 2 / 3", jw.per_component_stream("420", 40, 24, 2)),
            ("tables redefined before the scan", jw.write(40, 24, "444", co, before=decoys)),
            ("DRI past the MCU count", jw.write(40, 24, "444", co, restart=1000)),
            ("DRI 1 on 1 x 1", jw.write(1, 1, "420", jw.zeros(1, 1, "420"), restart=1))]
    for name, s in rows:
        _check(s, name)
    redefined = rows[1][1].data
    assert redefined.count(b"\xff\xdb") == 2 and redefined.count(b"\xff\xc4") == 4
    assert jr.parse(redefined).qt[0].tolist() == [1] * 64
    swapped = jw.write(40, 24, "444", co, scan_order=[1, 0, 2]).data
    assert ops.jpeg_info(swapped) == (0, 0, 0, 0, 0, 0) and not jr.info(swapped)[4]
    assert ops.jpeg_info(base.data)[5] == 1
