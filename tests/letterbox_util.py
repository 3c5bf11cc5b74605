"""Seeded photos and Pillow's letterbox for the letterbox tests (oracle/letterbox_ref.py, csrc/letterbox.cu)."""
import numpy as np

CONTENTS = ("noise", "ramp", "checker")

# (w, h, S): the sweep both the restatement and the device kernels are held to.
SWEEP = [
    # downscales of camera and phone photos
    (1920, 1080, 224), (1920, 1080, 896), (1080, 1920, 518), (1080, 1920, 896), (4032, 3024, 896),
    (4032, 3024, 1288), (3024, 4032, 672),
    # upscales
    (640, 480, 896), (100, 60, 896), (60, 100, 1288),
    # already S x S (a copy), and S wide or high (padding only, no resampling)
    (224, 224, 224), (672, 672, 672), (448, 200, 448), (101, 672, 672),
    # extreme aspects (a 2 or 7 pixel short side), a `contain` tie (1792 x 3 -> 1.5 -> 2), odd pad differences
    (3000, 7, 896), (7, 3000, 896), (3000, 7, 224), (1792, 3, 896), (3, 1792, 896), (513, 311, 518),
    (97, 101, 224), (300, 7, 448), (1288, 1287, 1288),
    # either side of the 100:1 height-to-width ratio past which Pillow runs the vertical pass first
    (10, 1000, 448), (10, 1001, 448), (1001, 10, 448), (3, 1000, 224),
]


def photo(w: int, h: int, content: str, seed: int = 0) -> np.ndarray:
    """uint8 [h, w, 3]: uniform noise, smooth ramps, or 0/255 checkerboards of 1, 2 and 3 pixel cells (which push
    the filter's negative lobes into the clip at both ends)."""
    rng = np.random.default_rng(seed + 7919 * w + 104729 * h)
    if content == "noise":
        return rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    y, x = np.mgrid[0:h, 0:w]
    if content == "ramp":
        fx, fy = x / max(w - 1, 1), y / max(h - 1, 1)
        return np.stack([fx * 255, fy * 255, (0.5 + 0.5 * np.sin(6.0 * fx + 4.0 * fy)) * 255], -1).round() \
            .astype(np.uint8)
    assert content == "checker"
    return np.stack([((x // c + y // c) % 2) * 255 for c in (1, 2, 3)], -1).astype(np.uint8)


def pillow_letterbox(img: np.ndarray, S: int, color: int = 0) -> np.ndarray:
    """ImageOps.pad(ImageOps.contain(img, (S, S)), (S, S), color=(c, c, c)) as uint8 [S, S, 3]."""
    from PIL import Image, ImageOps

    im = ImageOps.contain(Image.fromarray(img), (S, S))
    return np.asarray(ImageOps.pad(im, size=(S, S), color=(color,) * 3)).copy()
