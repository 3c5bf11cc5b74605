"""GPU: the device JPEG decode (csrc/jpeg.cu, `mhmr_op_jpeg_decode`) equals Pillow's `Image.open(f).convert("RGB")` byte
for byte from 1 x 1 to 4032 x 3024, batched, at any subsequence length of the parallel Huffman decoder; corrupt
streams are flagged; and `api.open_images` returns what the host-decode path returns."""
import io
import os

import numpy as np
import pytest
import torch

import jpeg_util as ju
from oracle import jpeg_ref as jr

pytestmark = pytest.mark.gpu


def _decode(blobs, cuda_device):
    from multihmr_b200 import preprocess

    return preprocess.decode_jpeg(blobs, cuda_device)


def _assert_pillow(blobs, photos, ok, what):
    for i, b in enumerate(blobs):
        assert ok[i], (what, i)
        assert np.array_equal(photos[i].cpu().numpy(), ju.pillow_rgb(b)), (what, i)


@pytest.mark.parametrize("mode", ju.MODES)
def test_device_equals_pillow_at_every_small_size(mode, cuda_device):
    blobs = [ju.encode(ju.photo(w, h), mode, quality=90) for w in range(1, 18) for h in range(1, 18)]
    photos, ok = _decode(blobs, cuda_device)
    _assert_pillow(blobs, photos, ok, mode)


@pytest.mark.parametrize("W, H", [(1920, 1080), (4032, 3024)])
@pytest.mark.parametrize("mode", ju.MODES)
def test_device_equals_pillow_at_production_sizes(W, H, mode, cuda_device):
    img = ju.photo(W, H, 17)
    blobs = [ju.encode(img, mode, quality=90), ju.encode(img, mode, quality=50, restart_marker_blocks=4),
             ju.encode(img, mode, quality=100, optimize=True), ju.encode(img, mode, quality=90, restart_marker_rows=1)]
    photos, ok = _decode(blobs, cuda_device)
    _assert_pillow(blobs, photos, ok, (W, H, mode))


def test_golden_photos(cuda_device):
    blobs = [open(p, "rb").read() for p in ju.GOLDEN]
    photos, ok = _decode(blobs, cuda_device)
    _assert_pillow(blobs, photos, ok, "golden")


def test_mixed_batch_equals_one_at_a_time_with_guard_bands_and_padded_pitches(cuda_device):
    from multihmr_b200 import ops, preprocess

    blobs = [ju.encode(ju.photo(w, h, i), ju.MODES[i % 4], quality=60 + 5 * i, **({"restart_marker_blocks": 3}
                                                                                   if i % 3 == 0 else {}))
             for i, (w, h) in enumerate([(640, 480), (33, 17), (1, 1), (301, 199), (2, 9), (1024, 768), (17, 3)])]
    host, dev, spans = preprocess.upload_bytes(blobs, cuda_device)
    frames, outs = [], []
    for b in blobs:
        h, w = ju.pillow_rgb(b).shape[:2]
        frame = torch.full((h + 4, w + 7, 3), 0xA5, dtype=torch.uint8, device=cuda_device)   # pitch 3 (w + 7)
        frames.append(frame)
        outs.append(frame[2:h + 2, 3:w + 3])
    status = ops.jpeg_decode(host, dev, spans, outs)
    assert status.cpu().tolist() == [0] * len(blobs)
    for b, frame, out in zip(blobs, frames, outs):
        want = ju.pillow_rgb(b)
        h, w = want.shape[:2]
        assert np.array_equal(out.cpu().numpy(), want)
        guard = frame.clone()
        guard[2:h + 2, 3:w + 3] = 0xA5
        assert bool((guard == 0xA5).all()), "a write left the photo's box"
        one, ok = _decode([b], cuda_device)
        assert ok[0] and torch.equal(one[0], out)


@pytest.mark.parametrize("subseq_bits", [1, 1024, 1 << 24])
def test_coefficients_identical_at_any_subsequence_length(subseq_bits, cuda_device):
    """Shorter than any codeword, the production length, and longer than a whole scan: the same coefficients as the
    restatement's sequential decode."""
    from multihmr_b200 import ops, preprocess

    blobs = [ju.encode(ju.photo(57, 41, 2), "420", quality=80), ju.encode(ju.photo(40, 33, 3), "L", quality=95),
             ju.encode(ju.photo(64, 24, 4), "422", quality=70, restart_marker_blocks=2),
             ju.encode(ju.photo(31, 29, 5), "444", quality=100, optimize=True)]
    if subseq_bits > 1:
        blobs.append(open(ju.GOLDEN[0], "rb").read())
    host, dev, spans = preprocess.upload_bytes(blobs, cuda_device)
    coefs, status, passes = ops.jpeg_coefficients(host, dev, spans, subseq_bits)
    assert status.cpu().tolist() == [0] * len(blobs)
    assert passes.item() >= 1
    for b, planes in zip(blobs, coefs):
        want, st = jr.decode_coefficients(b, jr.parse(b))
        assert st == 0
        for c, plane in enumerate(planes):
            assert np.array_equal(plane.cpu().numpy(), want[c]), (subseq_bits, c)


def _corrupt():
    """A fixed handful of corrupt streams, each flagged by the restatement: (name, bytes, the restatement's status)."""
    data = ju.encode(ju.photo(48, 40, 3), "420", quality=75, restart_marker_blocks=2)
    s, e = ju.ecs_span(data)
    rst = [i for i in range(s, e - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7]
    plain = ju.encode(ju.photo(48, 40, 3), "420", quality=75)
    ps, pe = ju.ecs_span(plain)
    cases = [("truncated", data[:s + (e - s) // 2] + b"\xff\xd9"),
             ("truncated without restarts", plain[:ps + (pe - ps) // 2] + b"\xff\xd9"),
             ("dropped rst", data[:rst[1]] + data[rst[1] + 2:]),
             ("swapped rst", ju.edit(ju.edit(data, rst[0] + 1, [data[rst[1] + 1]]), rst[1] + 1, [data[rst[0] + 1]])),
             ("all-ones run", data[:s + 8] + b"\xff\x00" * 6 + data[s + 20:]),
             ("saturating quantisers", ju.saturating_quantisers())]
    out = []
    for name, b in cases:
        st = jr.decode(b)[1]
        assert st != 0, name
        out.append((name, b, st))
    assert dict((n, st) for n, _, st in out)["truncated without restarts"] == jr.SHORT_DATA
    assert dict((n, st) for n, _, st in out)["saturating quantisers"] == jr.IDCT_RANGE
    return out


def test_device_status_carries_the_restatements_flag(cuda_device):
    """Each device flag fires where the restatement's does: the restatement stops at the first anomaly, the device
    reports every one it meets, so the device status holds the restatement's bit (the short-data check of a scan
    without restarts and the IDCT range check included)."""
    from multihmr_b200 import ops, preprocess

    cases = _corrupt()
    blobs = [b for _, b, _ in cases]
    host, dev, spans = preprocess.upload_bytes(blobs, cuda_device)
    outs = [torch.empty(40 if "saturating" not in n else 32, 48 if "saturating" not in n else 32, 3,
                        dtype=torch.uint8, device=cuda_device) for n, _, _ in cases]
    status = ops.jpeg_decode(host, dev, spans, outs).cpu().tolist()
    for (name, _, want), got in zip(cases, status):
        assert got & want == want, (name, got, want)
    assert status[[n for n, _, _ in cases].index("saturating quantisers")] == jr.IDCT_RANGE


def test_corrupt_streams_are_flagged_and_open_images_returns_pillows_result(cuda_device, tmp_path):
    from PIL import Image

    from multihmr_b200 import api

    cases = _corrupt()
    photos, ok = _decode([b for _, b, _ in cases], cuda_device)
    assert ok == [False] * len(cases) and photos == [None] * len(cases)
    for name, b, _ in cases:
        p = tmp_path / f"{name.replace(' ', '_')}.jpg"
        p.write_bytes(b)
        try:
            want = np.asarray(Image.open(p).convert("RGB"))
        except Exception as err:   # Pillow's own error must come out of open_images too
            with pytest.raises(type(err)):
                api.open_images([str(p)], 224, cuda_device, fused=True)
            continue
        _, full, _ = api.open_images([str(p)], 224, cuda_device, fused=True)
        assert np.array_equal(full[0].cpu().numpy(), want), name


def test_a_decompression_bomb_raises_pillows_error_before_any_device_work(cuda_device, tmp_path):
    """A header claiming 65535 x 65535 pixels: open_images raises Pillow's DecompressionBombError, as the host path
    did, and decode_jpeg refuses it without allocating its output."""
    from PIL import Image

    from multihmr_b200 import api, preprocess

    bomb = tmp_path / "bomb.jpg"
    bomb.write_bytes(ju.bomb_header())
    good = tmp_path / "good.jpg"
    good.write_bytes(ju.encode(ju.photo(64, 48), "420"))
    torch.cuda.synchronize()
    before = torch.cuda.max_memory_allocated(cuda_device)
    for paths in ([str(bomb)], [str(good), str(bomb)], [str(bomb), str(good)]):
        with pytest.raises(Image.DecompressionBombError):
            api.open_images(paths, 224, cuda_device, fused=True)
    photos, ok = preprocess.decode_jpeg([ju.bomb_header()], cuda_device)
    assert photos == [None] and ok == [False]
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated(cuda_device) - before < (64 << 20)


def test_open_images_on_a_mixed_folder_equals_the_host_decode_path(cuda_device, tmp_path):
    from PIL import Image

    from multihmr_b200 import api

    img = ju.photo(1280, 720, 9)
    files = {"a.jpg": ju.encode(img, "420", quality=90), "b.jpg": ju.encode(img, "420", progressive=True),
             "d.jpg": ju.encode(ju.photo(500, 640, 1), "L", quality=85),
             "e.jpg": open(ju.GOLDEN[1], "rb").read(), "f.jpg": ju.encode(img, "444", restart_marker_rows=1)}
    b = io.BytesIO()
    Image.fromarray(ju.photo(333, 250, 4)).save(b, format="PNG")
    files["c.png"] = b.getvalue()
    paths = []
    for name in sorted(files):
        (tmp_path / name).write_bytes(files[name])
        paths.append(str(tmp_path / name))
    for fused in (True, False):
        x, full, boxes = api.open_images(paths, 448, cuda_device, fused=fused)
        with torch.cuda.device(cuda_device):
            hx, hfull, hboxes = api._letterbox_photos([Image.open(p).convert("RGB") for p in paths], 448, cuda_device,
                                                      fused)
        assert torch.equal(x, hx) and torch.equal(boxes, hboxes)
        for a, h in zip(full, hfull):
            assert torch.equal(a, h)
    assert os.path.exists(paths[0])
