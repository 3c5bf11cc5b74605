"""GPU: the device PNG decode (csrc/png.cu, `mhmr_op_png_decode`) equals Pillow's `Image.open(f).convert("RGB")` byte
for byte on every eligible colour type, filter and encoder, from 1 x 1 to 4032 x 3024, batched, into row-padded
outputs whose guard bands stay untouched; and `api.open_images` returns what the host-decode path returns."""
import numpy as np
import pytest
import torch

import png_util as U
import png_writer as pw

pytestmark = pytest.mark.gpu


def _decode(blobs, cuda_device):
    from multihmr_b200 import preprocess

    return preprocess.decode_png(blobs, cuda_device)


def _assert_pillow(named, photos, ok):
    for (name, f), p, good in zip(named, photos, ok):
        assert good, name
        assert np.array_equal(p.cpu().numpy(), U.pillow(f)), name


def test_device_equals_pillow_on_every_family(cuda_device):
    named = U.pillow_files()
    photos, ok = _decode([f for _, f in named], cuda_device)
    _assert_pillow(named, photos, ok)


@pytest.mark.parametrize("ct", [0, 2, 3, 4, 6])
def test_production_sizes(ct, cuda_device):
    rng = np.random.default_rng(ct)
    C = pw.CHANNELS[ct]
    named = []
    for H, W in ((720, 1280), (1200, 1600), (3024, 4032)):
        px = U.photo(rng, H, W, C)
        named.append((f"pil-{W}x{H}", U.pillow_png(px, ct)))
        if ct == 2:
            named.append((f"cv2-{W}x{H}", U.cv2_png(px)))
    photos, ok = _decode([f for _, f in named], cuda_device)
    _assert_pillow(named, photos, ok)


def test_guard_bands_and_padded_pitches(cuda_device):
    """Outputs written into row-padded tensors between sentinel bands: only the photo's pixels change."""
    from multihmr_b200 import ops, preprocess

    named = U.pillow_files(seed=3, sizes=(1, 5, 17))[:40]
    blobs = [f for _, f in named]
    host, dev, spans = preprocess.upload_bytes([ops.png_idat(b) for b in blobs], cuda_device)
    frames, outs = [], []
    for b in blobs:
        W, H = ops.png_info(b)[:2]
        frame = torch.full((H + 2, 3 * W + 7 + 16), 0xA5, dtype=torch.uint8, device=cuda_device)
        frames.append(frame)
        outs.append(frame[1:H + 1, 8:8 + 3 * W].view(H, W, 3) if H > 0 else None)
    status = ops.png_decode(blobs, host, dev, spans, outs)
    assert status.cpu().tolist() == [0] * len(blobs)
    for (name, b), frame, o in zip(named, frames, outs):
        assert np.array_equal(o.cpu().numpy(), U.pillow(b)), name
        f = frame.cpu().numpy().copy()
        f[1:-1, 8:8 + o.shape[1] * 3] = 0xA5
        assert (f == 0xA5).all(), name


def test_ineligible_files_are_left_to_pillow(cuda_device):
    named = U.ineligible_files()
    photos, ok = _decode([f for _, f in named], cuda_device)
    assert ok == [False] * len(named) and photos == [None] * len(named)


def test_open_images_mixed_batch_equals_the_host_path(cuda_device, tmp_path, monkeypatch):
    """JPEG, eligible PNG of every colour type and an ineligible (16-bit) PNG in one batch: the same photos, batch
    and boxes as decoding every file with Pillow.  With a corrupt PNG added (a broken Adler-32, an interlace flag on
    plain data), both paths raise the same error."""
    import jpeg_util as ju

    from multihmr_b200 import api, preprocess

    rng = np.random.default_rng(5)
    files = [("a.jpg", ju.encode(ju.photo(320, 240), "420"))]
    for ct in (0, 2, 3, 4, 6):
        files.append((f"ct{ct}.png", U.pillow_png(U.photo(rng, 97 + ct, 131, pw.CHANNELS[ct]), ct)))
    files.append(("16bit.png", dict(U.ineligible_files())["16-bit"]))
    bad = bytearray(U.pillow_png(U.photo(rng, 50, 60, 3), 2))
    bad[-20] ^= 0xFF   # the Adler-32
    corrupt = [("adler.png", bytes(bad)), ("interlaced.png", dict(U.ineligible_files())["interlaced"])]
    paths = {}
    for name, b in files + corrupt:
        p = tmp_path / name
        p.write_bytes(b)
        paths[name] = str(p)
    good = [paths[n] for n, _ in files]

    def run(ps):
        try:
            return api.open_images(ps, 448, cuda_device, fused=True)
        except Exception as err:   # noqa: BLE001
            return err

    dev = [run(good)] + [run(good + [paths[n]]) for n, _ in corrupt]
    def host_only(blobs, device):
        return [None] * len(blobs), [False] * len(blobs)

    monkeypatch.setattr(preprocess, "decode_png", host_only)
    monkeypatch.setattr(preprocess, "decode_jpeg", host_only)
    host = [run(good)] + [run(good + [paths[n]]) for n, _ in corrupt]
    assert torch.equal(dev[0][0], host[0][0]) and torch.equal(dev[0][2], host[0][2])
    assert all(torch.equal(a, b) for a, b in zip(dev[0][1], host[0][1]))
    for d, h in zip(dev[1:], host[1:]):
        assert isinstance(h, Exception) and type(d) is type(h) and str(d) == str(h)
