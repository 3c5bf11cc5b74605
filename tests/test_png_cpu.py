"""CPU: the restatement of the device PNG decoder (oracle/png_ref.py) against Pillow's `Image.open(f).convert("RGB")`
on every eligible colour type from 1 x 1 to 17 x 17, 1-row and 1-column images, every filter forced per row (Paeth
ties included), Pillow levels 0-9, zlib strategies, OpenCV-written files and the golden photos as PNG; and the
eligibility of `mhmr_png_info`, which must agree with the restatement's chunk walk and refuse interlaced, 16-bit,
sub-byte and malformed files."""
import numpy as np
import pytest

import png_util as U
from oracle import png_ref as R

FILES = U.pillow_files()


@pytest.mark.parametrize("name, data", FILES, ids=[n for n, _ in FILES])
def test_restatement_equals_pillow(name, data):
    from multihmr_b200 import ops

    W, H, ct, eligible = ops.png_info(data)
    h = R.parse(data)
    assert eligible == 1 and h is not None and (W, H, ct) == (h["W"], h["H"], h["ctype"])
    status, rgb = R.decode(data)
    assert status == 0
    assert np.array_equal(rgb, U.pillow(data))


@pytest.mark.parametrize("name, data", U.ineligible_files(), ids=[n for n, _ in U.ineligible_files()])
def test_ineligible_files_are_refused(name, data):
    from multihmr_b200 import ops

    assert ops.png_info(data) == (0, 0, 0, 0)
    assert R.parse(data) is None


def test_info_of_other_bytes():
    from multihmr_b200 import ops

    for data in (b"", b"\x89PNG\r\n\x1a\n", b"GIF89a" + bytes(40), open(U.os.path.join(U.GOLDEN, sorted(
            f for f in U.os.listdir(U.GOLDEN) if f.endswith(".jpg"))[0]), "rb").read()):
        assert ops.png_info(data) == (0, 0, 0, 0)


def test_adler_and_idat_crc_as_pillow_sees_them():
    """Pillow ignores IDAT CRCs (the device does too) and refuses a wrong Adler-32 (the device flags it)."""
    import png_writer as pw

    rng = np.random.default_rng(0)
    f = bytearray(U.pillow_png(U.photo(rng, 7, 9, 3), 2))
    crc = bytearray(f)
    crc[-13] ^= 1   # the IDAT CRC (before IEND's 12 bytes)
    assert R.decode(bytes(crc))[0] == 0 and np.array_equal(R.decode(bytes(crc))[1], U.pillow(bytes(crc)))
    adler = bytearray(f)
    adler[-17] ^= 1
    assert R.decode(bytes(adler))[0] == R.BAD_ADLER and isinstance(U.pillow(bytes(adler)), OSError)
    assert pw.CHANNELS == R.CHANNELS
