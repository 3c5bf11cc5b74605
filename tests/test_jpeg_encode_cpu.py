"""CPU: the numpy restatement of the JPEG encoder (oracle/jpeg_encode_ref.py, what csrc/jpeg_encode.cu computes) writes
the bytes Pillow's `Image.save(f, "JPEG", quality=q, subsampling=s)` writes: every quality's tables, every width and
height residue mod 16, 4:4:4 / 4:2:2 / 4:2:0 / gray, and images that reach the largest DC and AC categories, ZRL
symbols, dummy blocks at both edges and 0xFF stuffing (counted in the restatement)."""
import numpy as np
import pytest

import jpeg_encode_util as eu
from oracle import jpeg_encode_ref as er


def test_quant_tables_of_every_quality_equal_pillows_dqt():
    img = eu.image("noise", 8, 8)
    for q in range(0, 102):
        data = eu.pillow_jpeg(img, quality=q)
        luma, chroma = er.quant_tables(q)
        i = 2 + 18                     # after SOI and APP0: DQT luma, then DQT chroma
        assert data[i:i + 5] == b"\xff\xdb\x00\x43\x00" and data[i + 69:i + 74] == b"\xff\xdb\x00\x43\x01", q
        assert data[i + 5:i + 69] == bytes(luma[z] for z in er.ZIGZAG), q
        assert data[i + 74:i + 138] == bytes(chroma[z] for z in er.ZIGZAG), q
        assert er.encode(img, q) == data, q


@pytest.mark.parametrize("subsampling,gray", eu.SETTINGS)
def test_every_size_residue_mod_16(subsampling, gray):
    for h in list(range(1, 18)) + [31, 33]:
        for w in (1, 2, 7, 8, 9, 15, 16, 17, 23, 24, 25, 31, 32, 33, 40, 47):
            img = eu.image("noise" if (h + w) % 2 else "gradient", h, w, gray=gray)
            assert er.encode(img, 75, subsampling) == eu.pillow_jpeg(img, 75, subsampling), (h, w)


@pytest.mark.parametrize("subsampling,gray", eu.SETTINGS)
def test_kinds_and_qualities(subsampling, gray):
    for kind in eu.KINDS:
        for q in (1, 10, 50, 75, 95, 100):
            img = eu.image(kind, 37, 45, gray=gray)
            assert er.encode(img, q, subsampling) == eu.pillow_jpeg(img, q, subsampling), (kind, q)


def test_fixtures_reach_every_entropy_path():
    stats = {}
    for kind in eu.KINDS:
        for subsampling, gray in eu.SETTINGS:
            for q in (1, 75, 100):
                img = eu.image(kind, 37, 37, gray=gray)   # 5 x 5 luma blocks: dummies right and below at 4:2:0
                assert er.encode(img, q, subsampling, stats) == eu.pillow_jpeg(img, q, subsampling)
    assert stats["dc_cat"] == 11 and stats["ac_cat"] == 10
    assert stats["zrl"] > 0 and stats["stuffed"] > 0
    assert stats["dummy_right"] > 0 and stats["dummy_bottom"] > 0


def test_quality_clamp():
    img = eu.image("noise", 9, 11)
    assert er.encode(img, 0) == eu.pillow_jpeg(img, 0) == eu.pillow_jpeg(img, 1)
    assert er.encode(img, 101) == eu.pillow_jpeg(img, 101) == eu.pillow_jpeg(img, 100)


def test_larger_photo():
    img = eu.image("gradient", 123, 201)
    img[::7, ::5] = np.random.default_rng(0).integers(0, 256, img[::7, ::5].shape, dtype=np.uint8)
    for s in (0, 1, 2):
        assert er.encode(img, 90, s) == eu.pillow_jpeg(img, 90, s)
