"""GPU: the mesh renderer (csrc/render.cu via multihmr_b200.render) against the fp64 restatement oracle/render_ref.py.

One comparison, `check_view`: the oracle flags pixels whose centre lies within 1e-3 px of an edge (or near-plane clip
line) of a triangle covering or almost covering it, or whose nearest surface is within 1e-5 (relative) of the second
nearest.  There float32 may decide coverage or visibility differently.  On every other pixel the person map is equal,
depth within 1e-5 relative, the shaded colour within 1 level, and the composite within 1 level wherever the
foreground of the pixel and its 8 neighbours agree."""
import math
import os
import sys

import numpy as np
import pytest
import torch

from oracle import render_ref

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda"


def _neigh_all(mask):
    """True where the pixel and its 8 neighbours are all True (outside the image counts as True)."""
    m = torch.from_numpy(~mask).float()[None, None]
    return ~(torch.nn.functional.max_pool2d(m, 3, 1, 1)[0, 0].numpy() > 0)


def check_view(gpu: dict, gpu_alpha1: np.ndarray, ref: dict, img: np.ndarray, alpha: float, ref_overlay=None,
               max_flagged=0.05, tag=""):
    """gpu: {'overlay', 'depth', 'index'} numpy of one view at `alpha`; gpu_alpha1: its overlay at alpha 1; ref: the
    oracle's rasterize() of the same view.  Returns the number of flagged pixels."""
    flag = (ref["edge_dist"] < 1e-3) | (ref["depth_gap"] < 1e-5)
    ok = ~flag
    H, W = flag.shape
    assert flag.mean() <= max_flagged, f"{tag}: {flag.sum()} of {H * W} pixels flagged"
    bad = ok & (gpu["index"] != ref["index"])
    assert not bad.any(), f"{tag}: person map differs at {bad.sum()} unflagged pixels, e.g. {np.argwhere(bad)[:5]}"
    fg = ok & (ref["depth"] > 0)
    rel = np.abs(gpu["depth"][fg].astype(np.float64) - ref["depth"][fg]) / ref["depth"][fg]
    assert rel.size == 0 or rel.max() <= 1e-5, f"{tag}: depth rel err {rel.max():.3e}"
    assert np.array_equal(gpu["depth"][ok & (ref["depth"] == 0)], np.zeros(int((ok & (ref["depth"] == 0)).sum())))
    fg_gpu, fg_ref = gpu["depth"] > 0, ref["depth"] > 0
    agree = _neigh_all(fg_gpu == fg_ref)
    inner = np.zeros_like(ok)
    inner[1:-1, 1:-1] = True                    # the smoothing pads with zeros: fg < 1 on the image border
    interior = agree & _neigh_all(fg_ref) & ok & inner
    d = np.abs(gpu_alpha1.astype(np.int16) - ref["rgb"].astype(np.int16)).max(-1)
    assert d[interior].max(initial=0) <= 1, f"{tag}: shaded colour off by {d[interior].max()}"
    want = render_ref.composite(ref["rgb"], ref["depth"], img, alpha) if ref_overlay is None else ref_overlay
    d = np.abs(gpu["overlay"].astype(np.int16) - want.astype(np.int16)).max(-1)
    assert d[agree].max(initial=0) <= 1, f"{tag}: composite off by {d[agree].max()}"
    assert interior.sum() > 0.5 * fg.sum() - 4 * (H + W)
    print(f"{tag}: {int(flag.sum())} of {H * W} px flagged, {int(fg_ref.sum())} foreground")
    return int(flag.sum())


def _np(out, b=0):
    return {k: v[b].cpu().numpy() for k, v in out.items()}


def _K(cam):
    return np.array([[cam["focal"][0], 0, cam["princpt"][0]], [0, cam["focal"][1], cam["princpt"][1]], [0, 0, 1]])


def _pose(cam):
    if "R" not in cam:
        return None
    p = np.zeros((1, 3, 4))
    p[0, :, :3], p[0, :, 3] = cam["R"], cam["t"]
    return p


@pytest.mark.parametrize("name", ["render_square_224", "render_offcentre_333x250", "render_pose_flat_160x120"])
def test_goldens(name):
    from multihmr_b200.render import Renderer, render_meshes
    from oracle import make_golden_render as mg

    img, verts, faces, cam, colors, alpha, smooth = mg.scene_inputs(name)
    with np.load(os.path.join(GOLDEN_DIR, name + ".npz")) as g:
        gold_overlay = (g["overlay_minus_photo"] + img.astype(np.int16)).astype(np.uint8)
    r = Renderer(faces, DEV)
    K = torch.tensor(_K(cam), dtype=torch.float32)[None]
    kw = dict(pose=_pose(cam), colors=torch.tensor(colors), smooth=smooth, depth=True, index=True)
    imgs = torch.from_numpy(img)[None].to(DEV)
    out = _np(r.render(torch.from_numpy(verts), K, imgs, alpha=alpha, **kw))
    out1 = _np(r.render(torch.from_numpy(verts), K, imgs, alpha=1.0, **kw))
    ref = render_ref.rasterize(verts, faces, _K(cam), img.shape[0], img.shape[1], R=cam.get("R"), t=cam.get("t"),
                               colors=np.asarray(colors), smooth=smooth, device=DEV)
    check_view(out, out1["overlay"], ref, img, alpha, ref_overlay=gold_overlay, max_flagged=0.01, tag=name)
    # the numpy entry point is the same render
    again = render_meshes(img, list(verts), [faces] * len(verts), cam, color=list(colors), alpha=alpha, smooth=smooth)
    assert np.array_equal(again, out["overlay"])


def test_synthetic_smplx_faces_near_plane():
    """Random vertex triples (huge, degenerate, back-facing and off-screen triangles); the second person crosses the
    near plane, part of it behind the camera.  Thousands of edges cross every pixel, so many more pixels are flagged
    than on a real mesh."""
    from multihmr_b200 import synth
    from multihmr_b200.render import Renderer

    bm = synth.make_body_model(seed=7)
    faces = bm["faces"].numpy()
    vt = bm["v_template"].numpy()
    verts = np.stack([vt + [-0.3, 0.0, 2.5], vt * 0.3 + [0.3, 0.2, 0.1]]).astype(np.float32)
    H, W = 72, 96
    K = np.array([[70.0, 0, 47.3], [0, 72.0, 35.1], [0, 0, 1]])
    img = (np.random.default_rng(0).integers(0, 256, (H, W, 3))).astype(np.uint8)
    colors = np.asarray([[0.8, 0.3, 0.2], [0.2, 0.7, 0.4]], np.float32)
    r = Renderer(faces, DEV, num_verts=vt.shape[0])
    args = (torch.from_numpy(verts), torch.tensor(K, dtype=torch.float32)[None], torch.from_numpy(img)[None].to(DEV))
    for smooth in (True, False):
        out = _np(r.render(*args, colors=torch.from_numpy(colors), alpha=0.7, smooth=smooth, depth=True, index=True))
        out1 = _np(r.render(*args, colors=torch.from_numpy(colors), alpha=1.0, smooth=smooth, depth=True, index=True))
        ref = render_ref.rasterize(verts, faces, K, H, W, colors=colors, smooth=smooth, device=DEV)
        assert (ref["depth"] > 0).mean() > 0.2 and set(np.unique(ref["index"])) >= {0, 1}
        assert (ref["depth"][ref["depth"] > 0] < 0.5).any(), "some surface must be clipped close to the near plane"
        check_view(out, out1["overlay"], ref, img, 0.7, max_flagged=0.2, tag=f"smplx random faces smooth={smooth}")


def _engine_case():
    import parity_util as pu
    from multihmr_b200 import synth

    case, sd, bm, x, K, idx = pu.build_inputs("s_224_S_forced")      # 3 images, persons [2, 0, 3]
    m = pu.build_engine(case, sd, bm)
    t, P = m.forward_raw(x, K, idx=idx)
    imgs = synth.make_images_u8(case["batch"], case["img_size"], seed=5).to(DEV)
    return m, bm, t, P, K.to(DEV), imgs


def test_engine_forward_raw_to_renderer():
    from multihmr_b200.render import PALETTE, Renderer

    m, bm, t, P, K, imgs = _engine_case()
    faces = m.smpl_layer["neutral_10"].bm_x.faces
    r = Renderer(faces, DEV, num_verts=m.num_verts)
    out = r.render_outputs(t, imgs, K, alpha=0.8, depth=True, index=True)
    out1 = r.render_outputs(t, imgs, K, alpha=1.0, depth=True, index=True)
    torch.cuda.synchronize()
    det_b = t["det_idx"][0, :P].cpu().numpy()
    v3d = t["v3d"][:P].cpu().numpy()
    assert P == 5 and 1 not in det_b
    assert torch.equal(out["overlay"][1], imgs[1]), "an image without persons comes back unchanged"
    assert (out["index"][1] == -1).all() and (out["depth"][1] == 0).all()
    colors = np.asarray([PALETTE[i] for i in range(P)])
    for b in (0, 2):
        sel = np.nonzero(det_b == b)[0]
        ref = render_ref.rasterize(v3d[sel], faces, K[b].cpu().numpy(), 224, 224, colors=colors[sel], device=DEV)
        ref["index"] = np.where(ref["index"] >= 0, sel[np.maximum(ref["index"], 0)], -1)
        check_view(_np(out, b), out1["overlay"][b].cpu().numpy(), ref, imgs[b].cpu().numpy(), 0.8, max_flagged=0.1,
                   tag=f"engine image {b}")


def test_deterministic_and_views_batch_like_single_calls():
    from multihmr_b200 import synth
    from multihmr_b200.render import Renderer

    verts, faces = synth.make_blob_people([(-0.5, 0.0, 2.8), (0.4, 0.1, 3.4)], seed=3)
    H, W, nv = 180, 240, 5
    r = Renderer(faces, DEV)
    ang = np.linspace(0, 1.0, nv)
    c = verts[0].mean(0)
    pose = np.zeros((nv, 3, 4))
    for i, a in enumerate(ang):  # rotate about the first person's centre (demo.py:160-186)
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        pose[i, :, :3], pose[i, :, 3] = R, c - R @ c
    K = torch.tensor([[200.0, 0, 121.0], [0, 200.0, 88.0], [0, 0, 1]]).expand(nv, 3, 3)
    imgs = synth.make_images_u8(2, 256, seed=1)[:, :H, :W].contiguous().to(DEV)
    vi = [0, 1, 0, 1, 0]
    kw = dict(person_image=torch.zeros(2, dtype=torch.int32), alpha=0.8, depth=True, index=True)
    vi_img = [0, 0, 0, 0, 0]
    a = r.render(torch.from_numpy(verts), K, imgs, view_image=vi_img, pose=pose, **kw)
    b = r.render(torch.from_numpy(verts), K, imgs, view_image=vi_img, pose=pose, **kw)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    for i in range(nv):
        one = r.render(torch.from_numpy(verts), K[i:i + 1], imgs, view_image=[0], pose=pose[i:i + 1], **kw)
        for k in a:
            assert torch.equal(a[k][i], one[k][0]), (k, i)
    # views of an image without persons are the photo
    c2 = r.render(torch.from_numpy(verts), K, imgs, view_image=vi, pose=pose, **kw)
    for i in (1, 3):
        assert torch.equal(c2["overlay"][i], imgs[1])
    for i in (0, 2, 4):
        assert torch.equal(c2["overlay"][i], a["overlay"][i])


def test_count_is_read_on_the_device():
    m, bm, t, P, K, imgs = _engine_case()
    from multihmr_b200.render import Renderer

    r = Renderer(m.smpl_layer["neutral_10"].bm_x.faces, DEV, num_verts=m.num_verts)
    want = r.render_outputs(t, imgs, K, depth=True, index=True)
    torch.cuda.synchronize()
    t2 = dict(t)
    t2["count"] = torch.zeros_like(t["count"])
    torch.cuda._sleep(50_000_000)                   # the count is written long after render() has been enqueued
    t2["count"].copy_(t["count"])
    got = r.render_outputs(t2, imgs, K, depth=True, index=True)
    for k in want:
        assert torch.equal(want[k], got[k]), k


def test_anny_faces_render_through_the_same_path():
    from multihmr_b200 import synth
    from multihmr_b200.render import Renderer

    bm = synth.AnnyLikeBodyModel(1500, seed=4)
    faces = bm.faces.numpy()
    vt = bm.v_template.numpy()
    verts = np.stack([vt + [0.2, 0.0, 3.0], vt + [-0.5, 0.1, 3.6]]).astype(np.float32)
    K = np.array([[150.0, 0, 64.0], [0, 150.0, 48.0], [0, 0, 1]])
    img = np.full((96, 128, 3), 40, np.uint8)
    r = Renderer(faces, DEV, num_verts=vt.shape[0])
    args = (torch.from_numpy(verts), torch.tensor(K, dtype=torch.float32)[None], torch.from_numpy(img)[None].to(DEV))
    out = _np(r.render(*args, alpha=0.5, depth=True, index=True))
    out1 = _np(r.render(*args, alpha=1.0, depth=True, index=True))
    from multihmr_b200.render import PALETTE

    ref = render_ref.rasterize(verts, faces, K, 96, 128, colors=np.asarray(PALETTE[:2]), device=DEV)
    check_view(out, out1["overlay"], ref, img, 0.5, max_flagged=0.1, tag="anny faces")


def test_bad_faces_and_shapes_raise():
    from multihmr_b200.render import Renderer

    faces = np.array([[0, 1, 2], [1, 2, 3]])
    with pytest.raises(AssertionError, match="face vertex index"):
        Renderer(faces, DEV, num_verts=3)
    with pytest.raises(AssertionError, match="face vertex index"):
        Renderer(np.array([[0, -1, 2]]), DEV, num_verts=3)
    with pytest.raises(ValueError):
        Renderer(np.zeros((4, 2), np.int64), DEV)
    with pytest.raises(ValueError):
        Renderer(np.zeros((4, 3), np.float32), DEV)
    r = Renderer(faces, DEV)
    img = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device=DEV)
    K = torch.tensor([[[8.0, 0, 4], [0, 8, 4], [0, 0, 1]]])
    v = torch.rand(1, 4, 3)
    with pytest.raises(ValueError):
        r.render(torch.rand(1, 5, 3), K, img)
    with pytest.raises(ValueError):
        r.render(v, K[0], img)
    with pytest.raises(ValueError):
        r.render(v, K, img.float())
    with pytest.raises(ValueError):
        r.render(v, K, img, view_image=[1])
    with pytest.raises(ValueError):
        r.render(v, K, img, pose=torch.zeros(1, 3, 3))
    with pytest.raises(AssertionError, match="alpha"):
        r.render(v, K, img, alpha=1.5)
    out = r.render(v, K, img)
    assert out["overlay"].shape == (1, 8, 8, 3)
