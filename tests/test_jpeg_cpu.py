"""CPU: oracle/jpeg_ref.py, the numpy restatement of the device JPEG decode (csrc/jpeg.cu), equals the installed
Pillow's `Image.open(f).convert("RGB")` byte for byte; the host header parser behind `mhmr_jpeg_info` classifies files
as the restatement does; and corrupt entropy data is either flagged or decodes exactly as Pillow decodes it."""
import io

import numpy as np
import pytest

import jpeg_util as ju
from oracle import jpeg_ref as jr


@pytest.fixture(scope="module", autouse=True)
def _libjpeg_turbo():
    from PIL import features

    if not features.check_feature("libjpeg_turbo"):
        pytest.skip("Pillow's JPEG backend is not libjpeg-turbo: the restatement pins libjpeg-turbo's arithmetic")


def _check(data, what):
    got, status = jr.decode(data)
    assert status == 0, (what, status)
    want = ju.pillow_rgb(data)
    assert got.shape == want.shape and np.array_equal(got, want), what


@pytest.mark.parametrize("mode", ju.MODES)
def test_restatement_equals_pillow_at_every_small_size(mode):
    """1 x 1 to 17 x 17: partial MCUs on both axes, chroma 1 and 2 samples wide (box upsampling) and wider."""
    for w in range(1, 18):
        for h in range(1, 18):
            _check(ju.encode(ju.photo(w, h), mode, quality=90), (mode, w, h))


@pytest.mark.parametrize("mode", ju.MODES)
@pytest.mark.parametrize("quality", [1, 50, 90, 100])
def test_restatement_equals_pillow_across_qualities(mode, quality):
    for w, h in ((64, 48), (75, 33), (130, 97)):
        _check(ju.encode(ju.photo(w, h, quality), mode, quality=quality), (mode, quality, w, h))


@pytest.mark.parametrize("mode", ju.MODES)
def test_restatement_equals_pillow_with_optimised_tables_and_restarts(mode):
    img = ju.photo(83, 61, 5)
    _check(ju.encode(img, mode, quality=85, optimize=True), (mode, "optimize"))
    for blocks in (1, 3, 7):
        data = ju.encode(img, mode, quality=85, restart_marker_blocks=blocks)
        assert jr.parse(data).restart > 0
        _check(data, (mode, "restart blocks", blocks))
    _check(ju.encode(img, mode, quality=85, restart_marker_rows=1), (mode, "restart rows"))


@pytest.mark.parametrize("path", ju.GOLDEN)
def test_restatement_equals_pillow_on_the_golden_photos(path):
    data = open(path, "rb").read()
    _check(data, path)


def test_idct_range_flag_marks_where_pillow_saturates():
    """Quantisation tables of 255 over a full-contrast q100 stream push dequantised coefficients past int16: the
    restatement flags the photo (Pillow's SIMD IDCT saturates where libjpeg's C IDCT wraps)."""
    assert jr.decode(ju.saturating_quantisers())[1] == jr.IDCT_RANGE


def test_a_decompression_bomb_header_is_eligible_but_pillow_refuses_it():
    """The header alone passes (the device path's pixel bound is Pillow's own limit, applied by its callers)."""
    from PIL import Image

    data = ju.bomb_header()
    assert jr.info(data)[:2] == (65535, 65535) and jr.info(data)[4]
    with pytest.raises(Image.DecompressionBombError):
        Image.open(io.BytesIO(data))


def _table():
    """(name, bytes, eligible) of headers the device must take or refuse; refused ones are made by editing an encoded
    file's header where Pillow cannot encode them (parsed only, never decoded)."""
    from PIL import Image

    img = ju.photo(40, 24, 1)
    rows = [(m, ju.encode(img, m), True) for m in ju.MODES]
    rows.append(("restart", ju.encode(img, "420", restart_marker_blocks=2), True))
    rows += [(f"golden{i}", open(p, "rb").read(), True) for i, p in enumerate(ju.GOLDEN)]
    rows.append(("progressive", ju.encode(img, "420", progressive=True), False))
    d444 = ju.encode(img, "444")
    sof = ju.segment(d444, 0xC0)
    rows.append(("4:1:1", ju.edit(d444, sof + 11, [0x41]), False))
    rows.append(("4:4:0", ju.edit(d444, sof + 11, [0x12]), False))
    rows.append(("12-bit", ju.edit(d444, sof + 4, [12]), False))
    b = io.BytesIO()
    Image.fromarray(img).convert("CMYK").save(b, format="JPEG")
    rows.append(("cmyk", b.getvalue(), False))
    adobe = lambda t: b"Adobe\x00\x64\x00\x00\x00\x00" + bytes([t])   # noqa: E731
    nojfif = d444[:2] + d444[2 + 2 + (d444[4] << 8 | d444[5]):]          # the JFIF APP0 removed
    assert nojfif[3] != 0xE0
    rows.append(("adobe1", ju.insert_segment(nojfif, 0xEE, adobe(1)), True))
    rows.append(("adobe0", ju.insert_segment(nojfif, 0xEE, adobe(0)), False))
    rows.append(("adobe0+jfif", ju.insert_segment(d444, 0xEE, adobe(0)), False))
    ids_rgb = ju.edit(ju.edit(ju.edit(nojfif, ju.segment(nojfif, 0xC0) + 10, b"R"), ju.segment(nojfif, 0xC0) + 13, b"G"),
                      ju.segment(nojfif, 0xC0) + 16, b"B")
    rows.append(("ids RGB", ids_rgb, False))
    dqt = ju.segment(d444, 0xDB)
    rows.append(("16-bit dqt", ju.edit(d444, dqt + 4, [0x10 | d444[dqt + 4]]), False))
    dht = ju.segment(d444, 0xC4)
    rows.append(("truncated dht", ju.edit(d444, dht + 2, [0, 2 + 17 + 3]), False))
    counts = list(d444[dht + 5:dht + 21])                      # the first DC table: move codes to length 1
    assert counts[2] >= 2
    counts[0], counts[2] = counts[0] + 2, counts[2] - 2
    rows.append(("oversubscribed dht", ju.edit(d444, dht + 5, counts), False))
    rows.append(("length past the end", ju.edit(d444, dht + 2, [0xFF, 0xF0]), False))
    rows.append(("no EOI", d444[:-2], False))
    b = io.BytesIO()
    Image.fromarray(img).save(b, format="PNG")
    rows.append(("png", b.getvalue(), False))
    return rows


def test_header_parser_classifies_files():
    from multihmr_b200 import ops

    for name, data, eligible in _table():
        got = ops.jpeg_info(data)
        assert bool(got[5]) == eligible, name
        assert jr.info(data)[4] == eligible, name
        if eligible:
            from PIL import Image

            im = Image.open(io.BytesIO(data))
            assert (got[0], got[1]) == im.size, name
            hdr = jr.parse(data)
            assert got[:5] == (hdr.width, hdr.height, hdr.ncomp) + jr.info(data)[3], name
        else:
            assert got[:5] == (0, 0, 0, 0, 0), name


@pytest.mark.parametrize("mode", ju.MODES)
def test_corrupt_entropy_data_is_flagged_or_exact(mode):
    """The contract the device path relies on: a photo the restatement does not flag decodes to Pillow's bytes (and
    Pillow decodes it); flagged or ineligible photos go to the host.  Flips of an interval's 1-padding are never
    flagged."""
    from PIL import Image

    rng = np.random.default_rng(11 + len(mode))
    flagged = exact = 0
    kinds = set()
    for restart in (0, 2):
        data = ju.encode(ju.photo(48, 40, 3), mode, quality=75, **({"restart_marker_blocks": restart} if restart else {}))
        for what, bad in ju.corruptions(rng, data):
            kinds.add(what)
            try:
                got, status = jr.decode(bad)
            except jr.Ineligible:
                continue
            assert status == 0 or what != "padding flip", (mode, restart)
            if status:
                flagged += 1
                continue
            want = np.asarray(Image.open(io.BytesIO(bad)).convert("RGB"))
            assert np.array_equal(got, want), (mode, restart, what)
            exact += 1
    print(f"{mode}: {flagged} flagged, {exact} exact, kinds {sorted(kinds)}")
    assert flagged > 0 and exact + flagged >= 20
    assert {"padding flip", "garbage before rst", "empty interval", "truncate at rst"} <= kinds
