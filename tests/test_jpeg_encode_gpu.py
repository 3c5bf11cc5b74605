"""GPU: the device JPEG encode (csrc/jpeg_encode.cu, `mhmr_op_jpeg_encode`) writes the bytes of Pillow's
`Image.save(f, "JPEG", quality=q, subsampling=s)` for mixed batches of every setting and size residue, for 1080p and
12-megapixel photos and pitched views; it writes nothing outside its outputs, nothing of a file longer than its
capacity, and the same bytes alone, in a batch or again; it checks its arguments before any launch and returns before
queued device work has run.  The device resize (`mhmr_op_resize_u8`) equals `Image.resize`, and `api.create_jpeg`
writes the files of the reference's dataset conversion."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

import jpeg_encode_util as eu

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 1_000_000_000  # about half a second of device work at the H100's clocks


def _encode(images, quality=75, subsampling=None, **options):
    from multihmr_b200 import preprocess

    return preprocess.encode_jpeg(images, quality, subsampling, **options)


def _raw(images, quals, subs, caps, guard=64, sentinel=0xA5):
    """The C entry on its own: (buffer with sentinel guard bands, [(offset, capacity)], device sizes, statuses)."""
    from multihmr_b200._lib import call, stream

    offs, total = [], guard
    for c in caps:
        offs.append((total, c))
        total += c + guard
    buf = torch.full((total,), sentinel, dtype=torch.uint8, device=images[0].device)
    desc = torch.zeros(len(images), 9, dtype=torch.int64)
    for i, (im, q, s, (o, c)) in enumerate(zip(images, quals, subs, offs)):
        ch = 1 if im.dim() == 2 else 3
        desc[i] = torch.tensor([im.data_ptr(), im.shape[0], im.shape[1], im.stride(0), ch, q, s, buf.data_ptr() + o, c])
    sizes = torch.zeros(len(images), dtype=torch.int64, device=buf.device)
    status = torch.zeros(len(images), dtype=torch.int32, device=buf.device)
    call("mhmr_op_jpeg_encode", desc, len(images), sizes, status, stream())
    return buf, offs, sizes, status


@pytest.mark.parametrize("subsampling,gray", eu.SETTINGS)
def test_mixed_batch_of_every_residue_equals_pillow(cuda_device, subsampling, gray):
    imgs, quals = [], []
    for h in list(range(1, 18)) + [31, 33]:
        for w in (1, 2, 7, 8, 9, 15, 16, 17, 23, 24, 25, 33):
            kind = eu.KINDS[(h * 7 + w) % len(eu.KINDS)]
            imgs.append(eu.image(kind, h, w, gray=gray))
            quals.append([1, 10, 50, 75, 95, 100][(h + w) % 6])
    got = _encode([torch.from_numpy(i).to(cuda_device) for i in imgs], quals, subsampling)
    for i, (img, q) in enumerate(zip(imgs, quals)):
        assert got[i] == eu.pillow_jpeg(img, q, subsampling), (img.shape, q)


def test_kinds_at_every_quality_in_one_batch(cuda_device):
    imgs, quals, subs = [], [], []
    for kind in eu.KINDS:
        for s, gray in eu.SETTINGS:
            for q in (0, 1, 2, 25, 49, 50, 51, 75, 90, 99, 100, 101, -1):
                imgs.append(eu.image(kind, 37, 37, gray=gray))
                quals.append(q)
                subs.append(s)
    got = _encode([torch.from_numpy(i).to(cuda_device) for i in imgs], quals, subs)
    for g, img, q, s in zip(got, imgs, quals, subs):
        assert g == eu.pillow_jpeg(img, q, s), (img.shape, q, s)


@pytest.mark.parametrize("h,w,q,s", [(1080, 1920, 75, None), (3024, 4032, 95, 0), (896, 2688, 75, 2), (1080, 1920, 100, 1)])
def test_large_photos_equal_pillow(cuda_device, h, w, q, s):
    img = eu.image("gradient", h, w)
    img[::3, ::7] = eu.image("noise", h, w)[::3, ::7]
    assert _encode([torch.from_numpy(img).to(cuda_device)], q, s)[0] == eu.pillow_jpeg(img, q, s)


def test_pitched_views_and_guard_bands(cuda_device):
    from multihmr_b200 import ops

    big = torch.from_numpy(eu.image("noise", 120, 200)).to(cuda_device)
    bigg = torch.from_numpy(eu.image("gradient", 120, 200, gray=True)).to(cuda_device)
    views = [big[3:60, 5:66], big[10:11, 7:40], bigg[1:50, 2:39], big[:, 150:], bigg[7:8, 9:10]]
    subs = [2, 1, 0, 0, 2]
    caps = [ops.jpeg_capacity(v.shape[0], v.shape[1], 1 if v.dim() == 2 else 3, s) for v, s in zip(views, subs)]
    buf, offs, sizes, status = _raw(views, [75, 90, 50, 100, 10], subs, caps)
    sizes, status, host = sizes.cpu().tolist(), status.cpu().tolist(), buf.cpu().numpy()
    assert status == [0] * len(views)
    prev = 0
    for v, q, s, (o, c), n in zip(views, [75, 90, 50, 100, 10], subs, offs, sizes):
        assert (host[prev:o] == 0xA5).all()
        assert host[o:o + n].tobytes() == eu.pillow_jpeg(v.cpu().numpy(), q, s)
        assert (host[o + n:o + c] == 0xA5).all()   # nothing written past the file
        prev = o + c
    assert (host[prev:] == 0xA5).all()


def test_a_file_longer_than_its_capacity_is_not_written(cuda_device):
    imgs = [torch.from_numpy(eu.image("noise", 40, 40)).to(cuda_device)] * 2
    want = eu.pillow_jpeg(imgs[0].cpu().numpy(), 75, 2)
    buf, offs, sizes, status = _raw(imgs, [75, 75], [2, 2], [len(want) - 1, len(want)])
    host = buf.cpu().numpy()
    assert status.cpu().tolist() == [1, 0] and sizes.cpu().tolist() == [len(want)] * 2
    assert (host[offs[0][0]:offs[0][0] + offs[0][1]] == 0xA5).all()
    assert host[offs[1][0]:offs[1][0] + len(want)].tobytes() == want


def test_alone_equals_batched_and_repeats_are_identical(cuda_device):
    imgs = [torch.from_numpy(eu.image(k, 50 + 9 * i, 70 - 5 * i)).to(cuda_device) for i, k in enumerate(eu.KINDS)]
    batched = _encode(imgs, 90, 2)
    assert [_encode([im], 90, 2)[0] for im in imgs] == batched
    assert _encode(imgs, 90, 2) == batched


def test_empty_batch(cuda_device):
    from multihmr_b200._lib import call, stream

    assert _encode([]) == []
    call("mhmr_op_jpeg_encode", torch.zeros(0, 9, dtype=torch.int64), 0, None, None, stream())
    call("mhmr_op_resize_u8", torch.zeros(0, 8, dtype=torch.int64), 0, stream())


def test_bad_arguments_raise_before_any_launch(cuda_device):
    from multihmr_b200._lib import call, stream

    img = torch.zeros(16, 16, 3, dtype=torch.uint8, device=cuda_device)
    out = torch.zeros(1 << 16, dtype=torch.uint8, device=cuda_device)
    sizes = torch.full((2,), -7, dtype=torch.int64, device=cuda_device)
    status = torch.full((2,), -7, dtype=torch.int32, device=cuda_device)
    good = [img.data_ptr(), 16, 16, 48, 3, 75, 2, out.data_ptr(), 1 << 16]
    bad = {1: [0, 65536, -1], 2: [0, 65536], 3: [47], 4: [0, 2, 4], 5: [0, 101, -1], 6: [-1, 3], 0: [0], 7: [0],
           8: [-1]}
    for field, values in bad.items():
        for v in values:
            d = list(good)
            d[field] = v
            if field in (1, 2) and v > 0:
                d[3] = 3 * 65536
            desc = torch.tensor([good, d], dtype=torch.int64)   # the bad photo is second: nothing may run
            with pytest.raises(AssertionError):
                call("mhmr_op_jpeg_encode", desc, 2, sizes, status, stream())
    with pytest.raises(AssertionError):
        call("mhmr_op_jpeg_encode", torch.tensor([good]), 1, None, status, stream())
    rd = torch.tensor([[img.data_ptr(), 16, 16, 48, out.data_ptr(), 0, 8, 24]], dtype=torch.int64)
    with pytest.raises(AssertionError):
        call("mhmr_op_resize_u8", rd, 1, stream())
    torch.cuda.synchronize()
    assert sizes.cpu().tolist() == [-7, -7] and status.cpu().tolist() == [-7, -7] and not out.any()


def test_device_files_decode_as_pillows(cuda_device):
    from multihmr_b200 import preprocess

    imgs = [eu.image("gradient", 333, 251), eu.image("noise", 64, 48), eu.image("checker", 17, 9)]
    files = _encode([torch.from_numpy(i).to(cuda_device) for i in imgs], [75, 95, 100], [2, 1, 0])
    photos, ok = preprocess.decode_jpeg(files, cuda_device)
    for f, p, k in zip(files, photos, ok):
        assert k and np.array_equal(p.cpu().numpy(), np.asarray(Image.open(io.BytesIO(f)).convert("RGB")))


def test_entries_return_before_queued_work_has_run(cuda_device):
    from multihmr_b200 import ops

    src = torch.from_numpy(eu.image("gradient", 300, 401)).to(cuda_device)
    caps = [ops.jpeg_capacity(300, 401, 3, 2)]
    buf0, _, sizes0, _ = _raw([src], [75], [2], caps)
    want_resize = ops.resize_u8([src], [(123, 77)])[0]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        got = []
        for _ in range(3):
            img = src.clone()   # the kernel that writes the input, on `side`
            got.append((_raw([img], [75], [2], caps), ops.resize_u8([img], [(123, 77)])[0]))
        returned_early = not side.query()
    side.synchronize()
    assert returned_early, "the calls waited for their stream"
    for (buf, _, sizes, _), r in got:
        assert torch.equal(sizes, sizes0) and torch.equal(buf, buf0) and torch.equal(r, want_resize)


@pytest.mark.parametrize("h,w,sizes", [
    (480, 640, [(512, 384), (320, 240), (1000, 750), (640, 480), (640, 17)]),
    (1080, 1920, [(512, 288), (1920, 1079), (97, 1080)]),
    (5, 2000, [(512, 1), (512, 40)]),
    (3000, 7, [(3, 512), (7, 100)]),
    (1, 1, [(9, 4)])])
def test_resize_equals_pillow(cuda_device, h, w, sizes):
    from multihmr_b200 import preprocess

    img = eu.image("noise", h, w)
    img[h // 3:, : w // 2] = eu.image("gradient", h, w)[h // 3:, : w // 2]
    outs = preprocess.resize([torch.from_numpy(img).to(cuda_device)] * len(sizes), sizes)
    for o, size in zip(outs, sizes):
        assert np.array_equal(o.cpu().numpy(), np.asarray(Image.fromarray(img).resize(size))), size


def _reference_create_jpeg(root_dir, target_size):
    """datasets/bedlam.py:449-479, restated inline, writing `<name>.ref.jpg` files' bytes into a dict."""
    out = {}
    for dirpath, _, filenames in os.walk(root_dir):
        for fn in filenames:
            if fn[-4:] == ".png" and fn[0] != ".":
                img_pil = Image.open(os.path.join(dirpath, fn)).convert("RGB")
                width, height = img_pil.size
                if target_size is not None:
                    if width > height:
                        other_side = int(float(img_pil.size[1]) * float(target_size / float(img_pil.size[0])))
                        img_pil = img_pil.resize((target_size, other_side))
                    else:
                        other_side = int(float(img_pil.size[0]) * float(target_size / float(img_pil.size[1])))
                        img_pil = img_pil.resize((other_side, target_size))
                    name = os.path.join(dirpath, fn[:-4] + f"_{target_size}.jpg")
                else:
                    name = os.path.join(dirpath, fn[:-4] + ".jpg")
                buf = io.BytesIO()
                img_pil.save(buf, "JPEG")
                out[name] = buf.getvalue()
    return out


@pytest.mark.parametrize("target_size", [512, 200, None])
def test_create_jpeg_writes_the_reference_files(cuda_device, tmp_path, target_size):
    from multihmr_b200 import api

    rgb = eu.image("gradient", 300, 457)
    (tmp_path / "a" / "b").mkdir(parents=True)
    Image.fromarray(rgb).save(tmp_path / "rgb.png")
    Image.fromarray(rgb[:, :, 1]).save(tmp_path / "a" / "gray.png")
    Image.fromarray(rgb).quantize(64).save(tmp_path / "a" / "palette.png")
    rgba = np.concatenate([rgb, eu.image("noise", 300, 457)[..., :1]], -1)
    Image.fromarray(rgba[:211, :140]).save(tmp_path / "a" / "b" / "tall_rgba.png")
    Image.fromarray((rgb[:120, :120, 0].astype(np.uint16) * 257)).save(tmp_path / "a" / "b" / "sixteen.png")
    Image.fromarray(rgb).save(tmp_path / "a" / ".hidden.png")
    Image.fromarray(rgb[:50]).save(tmp_path / "a" / "other.jpg")
    want = _reference_create_jpeg(str(tmp_path), target_size)
    assert len(want) == 5
    api.create_jpeg(str(tmp_path), target_size=target_size, device=cuda_device, batch=3)
    for name, data in want.items():
        with open(name, "rb") as fh:
            assert fh.read() == data, name
