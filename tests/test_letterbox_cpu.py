"""CPU: oracle/letterbox_ref.py, the numpy restatement of the letterbox (`ImageOps.contain` + `ImageOps.pad`, BICUBIC)
that csrc/letterbox.cu implements, equals the installed Pillow byte for byte."""
import numpy as np
import pytest

import letterbox_util as lu
from oracle import letterbox_ref as lr


@pytest.mark.parametrize("w, h, S", lu.SWEEP)
def test_restatement_equals_pillow_on_the_sweep(w, h, S):
    for i, content in enumerate(lu.CONTENTS):
        if w * h > 4_000_000 and content != lu.CONTENTS[S % 3]:
            continue                                    # one content per phone-sized photo keeps the test short
        img = lu.photo(w, h, content)
        for color in (0, 255) if i == 0 else (0,):
            got, box = lr.letterbox(img, S, color)
            assert np.array_equal(got, lu.pillow_letterbox(img, S, color)), (w, h, S, content, color)
            x0, y0, nw, nh = box
            assert (nw == S or nh == S) and 0 <= x0 <= S - nw and 0 <= y0 <= S - nh


def test_restatement_equals_pillow_on_random_sizes():
    rng = np.random.default_rng(2024)
    for _ in range(40):
        w, h = (int(v) for v in rng.integers(1, 700, size=2))
        S = int(rng.choice([224, 448, 518, 672, 896, 1288]))
        try:
            lr.contain_size(w, h, S)
        except ValueError:
            continue
        img = lu.photo(w, h, lu.CONTENTS[_ % 3], seed=_)
        assert np.array_equal(lr.letterbox(img, S)[0], lu.pillow_letterbox(img, S)), (w, h, S)


def test_contain_and_pad_rounding_is_half_to_even():
    assert lr.contain_size(1792, 3, 896) == (896, 2)            # 1.5 -> 2
    assert lr.contain_size(3, 1792, 896) == (2, 896)
    assert lr.contain_size(1792, 5, 896) == (896, 2)            # 2.5 -> 2
    assert lr.pad_box(1792, 5, 896) == (0, 447, 896, 2)         # (896 - 2) / 2 = 447
    assert lr.pad_box(513, 311, 518)[1] == round((518 - 314) * 0.5)
    assert lr.pad_box(224, 219, 224) == (0, 2, 224, 219)        # a difference of 5 -> 2.5 -> 2
    assert lr.pad_box(224, 221, 224) == (0, 2, 224, 221)        # a difference of 3 -> 1.5 -> 2
    assert lr.pad_box(1920, 1080, 896) == (0, 196, 896, 504)


def test_a_zero_sized_target_raises_like_pillow():
    from PIL import Image, ImageOps

    img = lu.photo(3000, 2, "noise")
    with pytest.raises(ValueError):
        lr.letterbox(img, 224)
    with pytest.raises(ValueError):
        ImageOps.pad(ImageOps.contain(Image.fromarray(img), (224, 224)), size=(224, 224))


def test_the_int32_accumulator_bound_holds_for_every_sweep_table():
    """255 * sum|k| + 2^21 < 2^31 on every coefficient row the sweep uses: the int32 sums cannot overflow."""
    for w, h, S in lu.SWEEP + [(100000, 500, 224), (5, 5, 1288)]:
        nw, nh = lr.contain_size(w, h, S)
        for n_in, n_out in ((w, nw), (h, nh)):
            k = lr.coefficients(n_in, n_out)[2].astype(np.int64)
            assert (255 * np.abs(k).sum(1) + (1 << 21)).max() < 2 ** 31
            assert np.all(np.abs(k.sum(1) - (1 << 22)) <= k.shape[1])    # normalised, up to the rounding
