"""GPU: the demo's views (Renderer.render_views: pose kernel + props in the z-buffer) against the fp64 restatement
oracle/render_views_ref.py, the public demo entry points, and on the engine's own outputs.  Pixel comparison rule as
in test_render_gpu.check_view."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import render_views_ref as rv

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"

# (H, W, focal, person positions): an odd and an even person count
SCENES = {"3p_160x120": (120, 160, 150.0, [(-0.5, 0.1, 3.2), (0.4, 0.0, 3.9), (0.9, 0.2, 3.5)]),
          "2p_224": (224, 224, 250.0, [(0.2, 0.0, 3.0), (-0.6, 0.1, 3.6)])}


def _scene(name):
    from multihmr_b200 import synth

    H, W, f, pos = SCENES[name]
    verts, faces = synth.make_blob_people(pos, seed=len(name))
    K = np.array([[f, 0, W / 2 + 0.3], [0, f, H / 2 - 0.2], [0, 0, 1]])
    photo = synth.make_images_u8(1, max(H, W), seed=3)[0, :H, :W].numpy().copy()
    t = {"v3d": torch.from_numpy(verts).to(DEV), "det_idx": torch.zeros(3, len(verts), dtype=torch.int32, device=DEV),
         "count": torch.full((1,), len(verts), dtype=torch.int32, device=DEV),
         "transl_pelvis": torch.tensor(np.asarray(pos), dtype=torch.float32, device=DEV)}
    return verts, faces, K, photo, t


def _glyph_renderer(faces, nv=None):
    from multihmr_b200.render import Renderer, camera_glyph

    return Renderer(faces, DEV, num_verts=nv, topologies=camera_glyph()[0])


@pytest.mark.parametrize("name", list(SCENES))
def test_views_against_oracle(name):
    from multihmr_b200.render import PALETTE
    from test_render_gpu import check_view

    verts, faces, K, photo, t = _scene(name)
    H, W = photo.shape[:2]
    r = _glyph_renderer(faces)
    kw = dict(orbit=(3, 40), side=True, depth=True, index=True)
    Kt = torch.tensor(K, dtype=torch.float32)[None]
    a = r.render_views(t, torch.from_numpy(photo)[None].to(DEV), Kt, alpha=0.8, **kw)
    a1 = r.render_views(t, torch.from_numpy(photo)[None].to(DEV), Kt, alpha=1.0, **kw)
    P = len(verts)
    colors = [PALETTE[i] for i in range(P)] + rv.glyph_meshes()[2]
    ref = rv.views(verts, faces, K, H, W, photo, 0.8, colors, np.asarray(SCENES[name][3])[:, 2], n_frames=3,
                   angle_range=40, side=True, device=DEV)
    refs = [ref["overlay"]] + ref["orbit"] + ref["side"]
    white = np.full_like(photo, 255)
    for w, rr in enumerate(refs):
        got = {"overlay": a["overlay"][0].cpu().numpy() if w == 0 else None,
               "depth": a["depth"][0, w].cpu().numpy(), "index": a["index"][0, w].cpu().numpy()}
        full = torch.cat([a["overlay"][:1], a["orbit"][0], a["side"][0]])
        full1 = torch.cat([a1["overlay"][:1], a1["orbit"][0], a1["side"][0]])
        got["overlay"] = full[w].cpu().numpy()
        alpha = 0.8 if w < 10 else 1.0
        check_view(got, full1[w].cpu().numpy(), rr, photo if w == 0 else white, alpha, ref_overlay=rr["overlay"],
                   max_flagged=0.02, tag=f"{name} view {w}")
    assert (a["index"][0, 10:] >= P).any(), "the glyph must be visible in the side views"


def test_poses_match_fp64_oracle():
    verts, faces, K, photo, t = _scene("2p_224")
    r = _glyph_renderer(faces)
    out = r.render_views(t, torch.from_numpy(photo)[None].to(DEV), torch.tensor(K, dtype=torch.float32)[None],
                         orbit=(20, 60), side=True)
    pose = out["pose"][0].double().cpu().numpy()
    want = np.concatenate([np.eye(3, 4)[None], rv.orbit_poses(verts[0], 20, 60),
                           rv.side_poses(np.asarray(SCENES["2p_224"][3])[:, 2].astype(np.float32))])
    assert np.abs(pose - want).max() <= 1e-6
    assert out["nonempty"].tolist() == [1] and out["rank"].tolist() == [0, 1]
    fo = out["frame_order"]
    assert len(fo) == 4 * (20 // 4) + 3 * (20 + 18) and fo[:5] == [0] * 5 and fo[5:7] == [1, 2]


def test_repeatable_and_views_batch_like_single_calls_with_props():
    from multihmr_b200.render import camera_glyph

    verts, faces, K, photo, t = _scene("3p_160x120")
    r = _glyph_renderer(faces)
    _, meshes = camera_glyph()
    props = [(tp, torch.tensor(v, dtype=torch.float32), c) for tp, v, c in meshes]
    poses = rv.side_poses([3.2, 3.9, 3.5])
    nv = 3
    Kb = torch.tensor(K, dtype=torch.float32).expand(nv, 3, 3)
    img = torch.from_numpy(photo)[None].to(DEV)
    kw = dict(props=props, alpha=0.7, depth=True, index=True, view_image=[0] * nv)
    a = r.render(torch.from_numpy(verts), Kb, img, pose=poses, **kw)
    b = r.render(torch.from_numpy(verts), Kb, img, pose=poses, **kw)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert (a["index"] >= 3).any()
    for i in range(nv):
        kw["view_image"] = [0]
        one = r.render(torch.from_numpy(verts), Kb[i:i + 1], img, pose=poses[i:i + 1], **kw)
        for k in a:
            assert torch.equal(a[k][i], one[k][0]), (k, i)
    v1 = r.render_views(t, img, torch.tensor(K, dtype=torch.float32)[None], orbit=(4, 30), side=True)
    v2 = r.render_views(t, img, torch.tensor(K, dtype=torch.float32)[None], orbit=(4, 30), side=True)
    for k in ("overlay", "orbit", "side", "pose"):
        assert torch.equal(v1[k], v2[k]), k


def _engine_case():
    import parity_util as pu
    from multihmr_b200 import synth

    case, sd, bm, x, K, idx = pu.build_inputs("s_224_S_forced")      # 3 images, persons [2, 0, 3]
    m = pu.build_engine(case, sd, bm)
    t, P = m.forward_raw(x, K, idx=idx)
    imgs = synth.make_images_u8(case["batch"], case["img_size"], seed=5).to(DEV)
    return m, t, P, K.to(DEV), imgs


def test_engine_render_views_equal_demo_functions():
    from multihmr_b200 import api
    from multihmr_b200.render import PALETTE, camera_glyph, render_side_views, renderer_for

    m, t, P, K, imgs = _engine_case()
    faces = m.smpl_layer["neutral_10"].bm_x.faces
    r = renderer_for(faces, m.num_verts, DEV, camera_glyph()[0])
    t2 = dict(t)
    t2["count"] = torch.zeros_like(t["count"])
    torch.cuda._sleep(50_000_000)                   # the count is written long after render_views is enqueued
    t2["count"].copy_(t["count"])
    r.render_views(t, imgs, K, orbit=(3, 30), side=True, alpha=0.8)   # first call: glyph and palette upload
    torch.cuda.set_sync_debug_mode("error")         # no host synchronisation inside render_views
    try:
        out = r.render_views(t2, imgs, K, orbit=(3, 30), side=True, alpha=0.8)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    det_b = t["det_idx"][0, :P].cpu().numpy()
    assert out["nonempty"].tolist() == [1, 0, 1]
    for b in range(3):
        sel = np.nonzero(det_b == b)[0]
        humans = [{"v3d": t["v3d"][i], "transl_pelvis": t["transl_pelvis"][i][None]} for i in sel]
        frames = api.create_rotating_video(humans, faces, K[b:b + 1], None, imgs[b].cpu().numpy(), alpha=0.8,
                                           n_frames=3, angle_range=30)
        sides = render_side_views(imgs[b].cpu().numpy(), list(PALETTE),
                                  humans, None, K[b:b + 1], faces)
        if len(sel) == 0:
            assert frames is None and all((s == 255).all() for s in sides)
            assert (out["side"][b] == 255).all() and torch.equal(out["overlay"][b], imgs[b])
            continue
        seq = torch.cat([out["overlay"][b:b + 1], out["orbit"][b]]).cpu().numpy()
        mine = [seq[i] for i in out["frame_order"]]
        assert len(frames) == len(mine)
        for i, (x, y) in enumerate(zip(frames, mine)):
            assert np.array_equal(x, y), (b, i)
        for k in range(3):
            assert np.array_equal(sides[k], out["side"][b, k].cpu().numpy()), (b, k)


def test_anny_closest_first():
    """ModelAnny lists persons closest first (stable in transl z): with `closest_first`, ranks and the orbit centre
    follow that order."""
    verts, faces, K, photo, t = _scene("3p_160x120")
    t["transl"] = torch.tensor([[0, 0, 3.9], [0, 0, 3.2], [0, 0, 3.2]], dtype=torch.float32, device=DEV)
    r = _glyph_renderer(faces)
    out = r.render_views(t, torch.from_numpy(photo)[None].to(DEV), torch.tensor(K, dtype=torch.float32)[None],
                         orbit=(2, 30), closest_first=True)
    assert out["rank"].tolist() == [2, 0, 1]
    want = rv.orbit_poses(verts[1], 2, 30)
    assert np.abs(out["pose"][0, 1:].double().cpu().numpy() - want).max() <= 1e-6


def test_malformed_input_is_refused():
    from multihmr_b200.render import Renderer

    faces = np.array([[0, 1, 2], [1, 2, 3]])
    with pytest.raises(AssertionError, match="topology face vertex index"):
        Renderer(faces, DEV, topologies=[np.array([[0, -1, 2]])])
    verts, faces, K, photo, t = _scene("3p_160x120")
    r = _glyph_renderer(faces)
    img = torch.from_numpy(photo)[None].to(DEV)
    Kt = torch.tensor(K, dtype=torch.float32)[None]
    with pytest.raises(ValueError, match="n_frames"):
        r.render_views(t, img, Kt, orbit=(1, 30))
    with pytest.raises(ValueError, match="K must be"):
        r.render_views(t, img, Kt[0])
    with pytest.raises(ValueError, match="K must be"):
        r.render_views(t, img, Kt.expand(2, 3, 3))
    # 2^20 + 1 faces leave 11 bits of the key for meshes: 2048 persons and one prop do not fit
    big = Renderer(np.tile([[0, 1, 2]], ((1 << 20) + 1, 1)), DEV, topologies=[np.array([[0, 1, 2]])])
    v = torch.rand(2048, 3, 3) + torch.tensor([0, 0, 2.0])
    small = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device=DEV)
    K8 = torch.tensor([[[8.0, 0, 4], [0, 8, 4], [0, 0, 1]]])
    big.render(v, K8, small)
    with pytest.raises(AssertionError, match="depth key"):
        big.render(v, K8, small, props=[(0, torch.rand(3, 3), (1.0, 0.0, 0.0))])
    with pytest.raises(ValueError, match="topology"):
        r.render(t["v3d"], Kt, img, props=[(5, torch.rand(3, 3), (1.0, 0.0, 0.0))])


@pytest.mark.parametrize("name", ["render_sideviews_3p_160x120", "render_sideviews_2p_224",
                                  "render_sideviews_empty_160x120"])
def test_sideview_goldens(name):
    """The reference's own render_side_views (oracle/make_golden_render_views.py) against render_views(side=True)."""
    from multihmr_b200.render import PALETTE, render_side_views
    from oracle import make_golden_render_views as mgv
    from test_render_gpu import check_view

    img, verts, faces, K, pos = mgv.scene_inputs(name)
    H, W = img.shape[:2]
    with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz")) as g:
        gold = (255 - g["white_minus_views"].astype(np.int16)).astype(np.uint8)
    P = len(verts)
    humans = [{"v3d": torch.from_numpy(verts[i]).float().to(DEV), "transl_pelvis": torch.from_numpy(pos[i])[None]}
              for i in range(P)]
    Kt = torch.tensor(K, dtype=torch.float32)[None]
    if not P:
        got = render_side_views(img, list(PALETTE), humans, None, Kt, faces)
        assert all(a.dtype == np.float64 and np.array_equal(a, b) for a, b in zip(got, gold))
        return
    r = _glyph_renderer(faces)
    t = {"v3d": torch.from_numpy(verts).float().to(DEV), "det_idx": torch.zeros(3, P, dtype=torch.int32, device=DEV),
         "count": torch.full((1,), P, dtype=torch.int32, device=DEV),
         "transl_pelvis": torch.from_numpy(pos).float().to(DEV)}
    white = torch.full((1, H, W, 3), 255, dtype=torch.uint8, device=DEV)
    out = r.render_views(t, white, Kt, side=True, alpha=1.0, depth=True, index=True)
    colors = [PALETTE[i] for i in range(P)] + rv.glyph_meshes()[2]
    ref = rv.views(verts, faces, K, H, W, img, 1.0, colors, pos[:, 2], side=True, device=DEV)
    for k in range(3):
        got = {"overlay": out["side"][0, k].cpu().numpy(), "depth": out["depth"][0, 1 + k].cpu().numpy(),
               "index": out["index"][0, 1 + k].cpu().numpy()}
        check_view(got, got["overlay"], ref["side"][k], np.full_like(img, 255), 1.0, ref_overlay=gold[k],
                   max_flagged=0.02, tag=f"{name} side {k}")
    again = render_side_views(img, list(PALETTE), humans, None, Kt, faces)
    for k in range(3):
        assert np.array_equal(again[k], out["side"][0, k].cpu().numpy())


def test_orbit_golden():
    """The reference's own create_rotating_video (oracle/make_golden_render_views.py) against render_views(orbit)."""
    from multihmr_b200 import api
    from multihmr_b200.render import PALETTE
    from oracle import make_golden_render_views as mgv
    from test_render_gpu import check_view

    name = "render_orbit_3p_160x120"
    img, verts, faces, K, pos = mgv.scene_inputs(name)
    H, W = img.shape[:2]
    with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz")) as g:
        overlay = (g["overlay_minus_photo"] + img.astype(np.int16)).astype(np.uint8)
        orbit = (255 - g["white_minus_orbit"].astype(np.int16)).astype(np.uint8)
        order = g["frame_order"].tolist()
    o = mgv.ORBIT
    P = len(verts)
    t = {"v3d": torch.from_numpy(verts).float().to(DEV), "det_idx": torch.zeros(3, P, dtype=torch.int32, device=DEV),
         "count": torch.full((1,), P, dtype=torch.int32, device=DEV),
         "transl_pelvis": torch.from_numpy(pos).float().to(DEV)}
    r = _glyph_renderer(faces)
    Kt = torch.tensor(K, dtype=torch.float32)[None]
    kw = dict(orbit=(o["n_frames"], o["angle_range"]), depth=True, index=True)
    out = r.render_views(t, torch.from_numpy(img)[None].to(DEV), Kt, alpha=o["alpha"], **kw)
    out1 = r.render_views(t, torch.from_numpy(img)[None].to(DEV), Kt, alpha=1.0, **kw)
    assert out["frame_order"] == order
    ref = rv.views(verts, faces, K, H, W, img, o["alpha"], [PALETTE[i] for i in range(P)], pos[:, 2],
                   n_frames=o["n_frames"], angle_range=o["angle_range"], device=DEV)
    gpu = [out["overlay"][0]] + list(out["orbit"][0])
    gpu1 = [out1["overlay"][0]] + list(out1["orbit"][0])
    for w, (rr, gold) in enumerate(zip([ref["overlay"]] + ref["orbit"], [overlay] + list(orbit))):
        got = {"overlay": gpu[w].cpu().numpy(), "depth": out["depth"][0, w].cpu().numpy(),
               "index": out["index"][0, w].cpu().numpy()}
        check_view(got, gpu1[w].cpu().numpy(), rr, img if w == 0 else np.full_like(img, 255), o["alpha"],
                   ref_overlay=gold, max_flagged=0.02, tag=f"{name} frame {w}")
    humans = [{"v3d": torch.from_numpy(verts[i]).float().to(DEV)} for i in range(P)]
    assert api.create_rotating_video([], faces, Kt, None, img) is None
    frames = api.create_rotating_video(humans, faces, Kt, None, img, alpha=o["alpha"], n_frames=o["n_frames"],
                                       angle_range=o["angle_range"])
    seq = [g.cpu().numpy() for g in gpu]
    assert len(frames) == len(order) and all(np.array_equal(f, seq[i]) for f, i in zip(frames, order))


def test_anny_engine_closest_first():
    """ModelAnny with the synthetic body model: forward_raw + the body model + place() on the device, then
    render_views(closest_first=True) equals the demo functions over each image's person list of ModelAnny.forward
    (closest first, stable in transl z)."""
    import anny_util as au
    from multihmr_b200 import api
    from multihmr_b200.render import PALETTE, camera_glyph, render_side_views, renderer_for

    case, sd, bm, x, K, idx = au.build_inputs("anny_224_S_forced")      # 3 images, persons [2, 0, 3]
    m = au.build_engine(case, sd, bm)
    persons = m(x, K=K, idx=idx)
    t, P = m.forward_raw(x, K, idx=idx)
    shape = t["shape"][:P]
    out_bm = m.body_model(pose_parameters=t["rotmat_homo"][:P],
                          phenotype_kwargs={k: shape[:, col] for k, col in m._shape_cols})
    pl = m.place(out_bm, t, P, want_v2d=False)
    tt = {"v3d": pl["v3d"], "transl_pelvis": pl["transl_pelvis"], "transl": t["transl"][:P],
          "det_idx": t["det_idx"][:, :P], "count": t["count"]}
    faces = m.body_model.faces
    r = renderer_for(faces, pl["v3d"].shape[1], DEV, camera_glyph()[0])
    Kd = K.to(DEV)
    imgs = torch.full((3, 224, 224, 3), 90, dtype=torch.uint8, device=DEV)
    out = r.render_views(tt, imgs, Kd, orbit=(2, 30), side=True, alpha=0.8, closest_first=True)
    det_b = t["det_idx"][0, :P].cpu().numpy()
    transl = t["transl"][:P].cpu()
    image_of = [int(det_b[[torch.equal(transl[i], p["transl"].cpu()) for i in range(P)].index(True)])
                for p in persons]
    for b in range(3):
        humans = [p for p, ib in zip(persons, image_of) if ib == b]
        frames = api.create_rotating_video(humans, faces, Kd[b:b + 1], None, imgs[b].cpu().numpy(), alpha=0.8,
                                           n_frames=2, angle_range=30)
        sides = render_side_views(imgs[b].cpu().numpy(), list(PALETTE), humans, None, Kd[b:b + 1], faces)
        if not humans:
            assert frames is None and out["nonempty"][b] == 0
            continue
        assert len(humans) >= 2
        seq = torch.cat([out["overlay"][b:b + 1], out["orbit"][b]]).cpu().numpy()
        assert all(np.array_equal(f, seq[i]) for f, i in zip(frames, out["frame_order"]))
        for k in range(3):
            assert np.array_equal(sides[k], out["side"][b, k].cpu().numpy()), (b, k)
