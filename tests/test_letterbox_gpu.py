"""GPU: the device letterbox (csrc/letterbox.cu, `mhmr_op_letterbox_u8`) equals Pillow's `ImageOps.pad(ImageOps.contain(
photo, (S, S)), (S, S))` byte for byte, batched over photos of different sizes, and `api.open_images` feeds
`Model.forward` the same bytes as the host path of `open_image`."""
import os

import numpy as np
import pytest
import torch

import letterbox_util as lu
from oracle import letterbox_ref as lr

pytestmark = pytest.mark.gpu


def _dev(img, cuda_device):
    return torch.from_numpy(img).to(cuda_device)


@pytest.mark.parametrize("w, h, S", lu.SWEEP)
def test_device_letterbox_equals_pillow_on_the_sweep(w, h, S, cuda_device):
    from multihmr_b200 import preprocess

    for content in lu.CONTENTS:
        img = lu.photo(w, h, content)
        for color in (0, 255):
            out, boxes = preprocess.letterbox([_dev(img, cuda_device)], S, color=color)
            assert out.shape == (1, S, S, 3) and out.dtype == torch.uint8 and out.is_cuda
            assert np.array_equal(out[0].cpu().numpy(), lu.pillow_letterbox(img, S, color)), (w, h, S, content, color)
            assert boxes.tolist() == [list(lr.pad_box(w, h, S))]


def test_mixed_size_batch_equals_one_at_a_time(cuda_device):
    """One call over photos of different sizes and pitches (host and device tensors, row-padded views whose padding
    would change the result if it were read) gives each photo's own letterbox."""
    from multihmr_b200 import preprocess

    S = 448
    sizes = [(1920, 1080), (1080, 1920), (448, 448), (448, 200), (10, 1001), (640, 480), (97, 101), (1001, 10)]
    imgs = [lu.photo(w, h, lu.CONTENTS[i % 3], seed=i) for i, (w, h) in enumerate(sizes)]
    photos = []
    for i, img in enumerate(imgs):
        h, w = img.shape[:2]
        if i % 3 == 0:
            photos.append(torch.from_numpy(img))                          # host: uploaded by letterbox
        else:                                                             # device view inside a sentinel frame
            frame = torch.full((h + 2, w + 5, 3), 255 if i % 2 else 0, dtype=torch.uint8)
            frame[0::2, :, 1] = 0
            frame[1:h + 1, 2:w + 2] = torch.from_numpy(img)
            photos.append(frame.to(cuda_device)[1:h + 1, 2:w + 2])
            assert photos[-1].stride(0) == 3 * (w + 5)
    out, boxes = preprocess.letterbox(photos, S)
    for i, img in enumerate(imgs):
        one, box = preprocess.letterbox([_dev(img, cuda_device)], S)
        assert torch.equal(out[i], one[0]) and torch.equal(boxes[i], box[0]), sizes[i]
        assert np.array_equal(out[i].cpu().numpy(), lu.pillow_letterbox(img, S)), sizes[i]
        assert tuple(boxes[i].tolist()) == lr.pad_box(img.shape[1], img.shape[0], S)


def _raw_call(photos, S, out, pad=0):
    from multihmr_b200 import _lib

    desc = torch.tensor([[p.data_ptr(), p.shape[0], p.shape[1], p.stride(0)] for p in photos], dtype=torch.int64)
    boxes = torch.full((len(photos), 4), -1, dtype=torch.int32)
    _lib.call("mhmr_op_letterbox_u8", desc, len(photos), S, pad, out, boxes, _lib.stream())
    return boxes


def test_guard_bands_around_the_output_stay_intact(cuda_device):
    S, B, G = 224, 3, 4096
    imgs = [lu.photo(w, h, "checker") for w, h in ((1920, 1080), (7, 3000), (224, 100))]
    buf = torch.full((G + B * S * S * 3 + G,), 0xA5, dtype=torch.uint8, device=cuda_device)
    out = buf[G:G + B * S * S * 3]
    _raw_call([_dev(im, cuda_device) for im in imgs], S, out, pad=7)
    torch.cuda.synchronize()
    assert bool((buf[:G] == 0xA5).all()) and bool((buf[-G:] == 0xA5).all())
    got = out.view(B, S, S, 3).cpu().numpy()
    for i, im in enumerate(imgs):
        assert np.array_equal(got[i], lu.pillow_letterbox(im, S, 7))


def test_a_zero_sized_target_raises_before_any_launch(cuda_device):
    S = 224
    good, bad = _dev(lu.photo(640, 480, "noise"), cuda_device), _dev(lu.photo(3000, 2, "noise"), cuda_device)
    out = torch.full((2, S, S, 3), 0x5A, dtype=torch.uint8, device=cuda_device)
    with pytest.raises(AssertionError, match="rounds to 0"):
        _raw_call([good, bad], S, out)
    with pytest.raises(AssertionError, match="pad value"):
        _raw_call([good], S, out, pad=256)
    torch.cuda.synchronize()
    assert bool((out == 0x5A).all())                   # nothing was written for the valid photo either
    from multihmr_b200 import preprocess

    with pytest.raises(AssertionError):
        preprocess.letterbox([bad], S)


def _write_photos(tmp_path):
    from PIL import Image

    paths = []
    for i, (w, h) in enumerate([(320, 240), (150, 400), (224, 224)]):
        p = os.path.join(tmp_path, f"photo{i}.png")
        Image.fromarray(lu.photo(w, h, ("noise", "ramp", "noise")[i], seed=i)).save(p)
        paths.append(p)
    return paths


def test_open_images_equals_open_image_per_file(cuda_device, tmp_path):
    from PIL import Image

    from multihmr_b200 import api

    paths = _write_photos(tmp_path)
    for S in (224, 518):
        x, full, boxes = api.open_images(paths, S, device=cuda_device)
        u8, full8, boxes8 = api.open_images(paths, S, device=cuda_device, fused=True)
        assert x.shape == (3, 3, S, S) and x.dtype == torch.float32 and u8.shape == (3, S, S, 3)
        assert torch.equal(boxes, boxes8)
        for i, p in enumerate(paths):
            x_host, pil = api.open_image(p, S, device=torch.device("cpu"))
            assert torch.equal(x[i].cpu(), x_host[0]), (p, S)
            if S % 4 == 0:
                x_dev, _ = api.open_image(p, S, device=cuda_device)
                u8_dev, _ = api.open_image(p, S, device=cuda_device, fused=True)
                assert torch.equal(x[i], x_dev[0]) and torch.equal(u8[i], u8_dev[0])
            arr = np.asarray(Image.open(p).convert("RGB"))
            assert np.array_equal(full[i].cpu().numpy(), arr) and np.array_equal(full8[i].cpu().numpy(), arr)
            assert tuple(boxes[i].tolist()) == lr.pad_box(pil.width, pil.height, S)


def test_forward_on_the_letterboxed_batch_equals_the_host_path(cuda_device, tmp_path):
    """Model.forward (synthetic weights, detection mode) on the uint8 batch of open_images returns the same persons,
    bit for bit, as on the batch of host-path open_image tensors (PIL letterbox, host normalisation)."""
    import parity_util as pu
    from multihmr_b200 import api, synth

    paths = _write_photos(tmp_path)
    case, sd, bm, _, _, _ = pu.build_inputs("s_224_S_detect")
    m = pu.build_engine(case, sd, bm, max_batch=len(paths))
    K = synth.make_cameras(len(paths), case["img_size"], seed=2).to(cuda_device)
    u8, _, _ = api.open_images(paths, case["img_size"], device=cuda_device, fused=True)
    x_host = torch.cat([api.open_image(p, case["img_size"], device=torch.device("cpu"))[0] for p in paths])
    a = api.forward_model(m, u8, K, det_thresh=0.3)
    a = [{k: v.clone() for k, v in h.items()} for h in a]
    b = api.forward_model(m, x_host.to(cuda_device), K, det_thresh=0.3)
    assert len(a) == len(b) > 0
    for ha, hb in zip(a, b):
        assert ha.keys() == hb.keys() and all(torch.equal(ha[k], hb[k]) for k in ha)
