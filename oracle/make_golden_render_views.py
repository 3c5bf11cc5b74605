"""Pins oracle/render_views_ref.py against the reference's OWN `utils/render.py:render_side_views` and
`demo.py:create_rotating_video`, and writes tests/golden/render_{sideviews,orbit}_*.npz.

Runs ONLY where the reference checkout exists.  Both files are loaded UNMODIFIED.  The pyrender / trimesh shims of
oracle/make_golden_render.py are widened to several topologies and materials in one scene, and trimesh merges
coincident points on construction.  A `pyvista` shim serves `Cone`, `Box` and `Arrow` from the restatement of
render_views_ref.  demo.py is loaded as a file: `utils` (the loaded render module, `demo_color` = this package's
PALETTE), `model`, `multi_hmr_anny.multi_hmr` and `ipdb` are stand-ins, since the functions run here only render.
The script asserts shim run == restatement before writing.

Usage:  python -m oracle.make_golden_render_views            (from the repo root)
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
REFERENCE = "/root/reference"
GOLDEN = os.path.join(REPO, "tests", "golden")

from oracle import make_golden_render as mg  # noqa: E402
from oracle import render_views_ref as rv  # noqa: E402

# name -> (H, W, focal, person positions); an odd, an even and an empty person list
SIDE_SCENES = {"render_sideviews_3p_160x120": (120, 160, 150.0, [(-0.5, 0.1, 3.2), (0.4, 0.0, 3.9), (0.9, 0.2, 3.5)]),
               "render_sideviews_2p_224": (224, 224, 250.0, [(0.2, 0.0, 3.0), (-0.6, 0.1, 3.6)]),
               "render_sideviews_empty_160x120": (120, 160, 150.0, [])}
ORBIT_SCENES = {"render_orbit_3p_160x120": (120, 160, 150.0, [(-0.4, 0.1, 3.0), (0.5, 0.0, 3.6), (0.1, 0.2, 4.2)]),
                "render_orbit_empty_160x120": (120, 160, 150.0, [])}
ORBIT = dict(n_frames=4, angle_range=40, alpha=0.8)


def scene_inputs(name):
    """Seeded inputs: photo uint8 [H,W,3] (a gradient), verts fp64 [P,V,3], faces, K [3,3], pelvis positions."""
    from multihmr_b200 import synth

    H, W, f, pos = {**SIDE_SCENES, **ORBIT_SCENES}[name]
    verts, faces = synth.make_blob_people(pos if pos else [(0.0, 0.0, 3.0)], seed=len(name))
    verts = verts[:len(pos)].astype(np.float64)
    yy, xx = np.mgrid[0:H, 0:W]
    img = np.stack([(xx * 255 // (W - 1)), (yy * 255 // (H - 1)), np.full_like(xx, 96)], -1).astype(np.uint8)
    K = np.array([[f, 0, W / 2 + 0.3], [0, f, H / 2 - 0.2], [0, 0, 1]])
    return img, verts, faces, K, np.asarray(pos, np.float64).reshape(-1, 3)


def orbit_frames(views, n_frames):
    """demo.py:212-221's order over the restatement's views."""
    central = views["overlay"]["overlay"]
    sw = [[v["overlay"] for v in views["orbit"][s * n_frames:(s + 1) * n_frames]] for s in range(3)]
    c = [central] * (n_frames // 4)
    return c + sw[0] + sw[0][::-1][1:-1] + c + sw[1] + sw[1][::-1][1:-1] + c + sw[2] + sw[2][::-1][1:-1] + c


def frame_order(n_frames):
    """demo.py:212-221 as indices into [overlay] + the 3 n_frames orbit views."""
    sw = [[1 + s * n_frames + i for i in range(n_frames)] for s in range(3)]
    c = [0] * (n_frames // 4)
    return c + sw[0] + sw[0][::-1][1:-1] + c + sw[1] + sw[1][::-1][1:-1] + c + sw[2] + sw[2][::-1][1:-1] + c


# ---------------------------------------------------------------------------------------------- widened shims
class _Trimesh(mg._Trimesh):
    def __init__(self, vertices, faces, process=True, **kw):
        v, f = (rv.merge_vertices(vertices, faces) if process else (vertices, faces))
        super().__init__(v, f)


class _Renderer(mg._Renderer):
    def render(self, scene, flags=None):
        meshes = [(o, p) for o, p in scene.nodes if isinstance(o, mg._Mesh)]
        (cam, cam_pose), = [(o, p) for o, p in scene.nodes if isinstance(o, mg._Camera)]
        (light, light_pose), = [(o, p) for o, p in scene.nodes if isinstance(o, mg._Light)]
        assert np.array_equal(light_pose, cam_pose), "the restatement's light sits at the camera"
        for _, p in meshes:
            assert np.array_equal(p, np.eye(4))
        world_to_cv = mg._CV2GL @ np.linalg.inv(cam_pose)
        mats = {(m.material.metallic, m.material.roughness) for m, _ in meshes}
        assert len(mats) == 1
        (metallic, roughness), = mats
        smooth = {m.smooth for m, _ in meshes}
        assert len(smooth) == 1
        smooth = smooth.pop()
        out = rv.rasterize_meshes(
            [m.vertices for m, _ in meshes], [m.faces for m, _ in meshes], cam.K, self.H, self.W,
            R=world_to_cv[:3, :3], t=world_to_cv[:3, 3], normals=[m.normals for m, _ in meshes] if smooth else None,
            colors=[m.material.color[:3] for m, _ in meshes], intensity=light.intensity, metallic=metallic,
            roughness=roughness, smooth=smooth)
        rgba = np.concatenate([out["rgb"], np.where(out["depth"] > 0, 255, 0).astype(np.uint8)[..., None]], -1)
        return rgba, out["depth"].astype(np.float32)


def install_shims():
    mg.install_shims()
    sys.modules["pyrender"].OffscreenRenderer = _Renderer
    sys.modules["trimesh"].Trimesh = _Trimesh
    pyvista = types.ModuleType("pyvista")
    pyvista.Cone, pyvista.Box, pyvista.Arrow = rv.pyvista_cone, rv.pyvista_box, rv.pyvista_arrow
    sys.modules["pyvista"] = pyvista


def load_reference():
    """(utils/render.py module, demo.py module), both unmodified."""
    from multihmr_b200.render import PALETTE

    install_shims()
    spec = importlib.util.spec_from_file_location("_ref_render_views", os.path.join(REFERENCE, "utils", "render.py"))
    render = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(render)
    utils = types.ModuleType("utils")
    for k in ("render_meshes", "print_distance_on_image", "render_side_views", "create_scene"):
        setattr(utils, k, getattr(render, k))
    utils.normalize_rgb = utils.get_focalLength_from_fieldOfView = None
    utils.demo_color = list(PALETTE)
    utils.MEAN_PARAMS, utils.CACHE_DIR_MULTIHMR, utils.SMPLX_DIR = "", "", ""
    stubs = {"utils": utils, "model": types.ModuleType("model"), "multi_hmr_anny": types.ModuleType("multi_hmr_anny"),
             "multi_hmr_anny.multi_hmr": types.ModuleType("multi_hmr_anny.multi_hmr"), "ipdb": types.ModuleType("ipdb")}
    stubs["model"].Model = None
    stubs["multi_hmr_anny.multi_hmr"].Multi_HMR = None
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    try:
        spec = importlib.util.spec_from_file_location("_ref_demo", os.path.join(REFERENCE, "demo.py"))
        demo = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(demo)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return render, demo


def humans_of(verts, pos):
    return [{"v3d": torch.from_numpy(verts[i]), "transl_pelvis": torch.from_numpy(pos[i])[None]}
            for i in range(len(verts))]


def main():
    from PIL import Image

    from multihmr_b200.render import PALETTE

    render, demo = load_reference()
    total = 0
    for name in SIDE_SCENES:
        img, verts, faces, K, pos = scene_inputs(name)
        H, W = img.shape[:2]
        colors = [PALETTE[i] for i in range(len(verts))]
        got = render.render_side_views(img, colors, humans_of(verts, pos), None,
                                       torch.from_numpy(K)[None], faces)
        got = np.stack(got)
        if len(verts):
            assert got.dtype == np.uint8
            mine = rv.views(verts, faces, K, H, W, img, 1.0, colors + rv.glyph_meshes()[2], pos[:, 2], side=True)
            assert np.array_equal(got, np.stack([v["overlay"] for v in mine["side"]])), f"{name}: reference != restatement"
            glyph = np.stack([(v["index"] >= len(verts)).sum() for v in mine["side"]])
            assert glyph[0] > 20, f"{name}: the glyph must show in the displaced view ({glyph})"
        else:
            assert got.dtype == np.float64 and (got == 255).all()
        path = os.path.join(GOLDEN, name + ".npz")
        np.savez_compressed(path, white_minus_views=(255 - got).astype(np.uint8), dtype=str(got.dtype))
        total += os.path.getsize(path)
        print(f"{name}: {os.path.getsize(path)} bytes")
    for name in ORBIT_SCENES:
        img, verts, faces, K, pos = scene_inputs(name)
        H, W = img.shape[:2]
        got = demo.create_rotating_video(humans_of(verts, pos), faces, torch.from_numpy(K)[None], None,
                                         Image.fromarray(img), alpha=ORBIT["alpha"], fn=None,
                                         n_frames=ORBIT["n_frames"], angle_range=ORBIT["angle_range"])
        path = os.path.join(GOLDEN, name + ".npz")
        if not len(verts):
            assert got is None
            np.savez_compressed(path, none=np.ones(1, np.uint8))
        else:
            got = np.stack(got)
            colors = [PALETTE[i] for i in range(len(verts))]
            mine = rv.views(verts, faces, K, H, W, img, ORBIT["alpha"], colors, pos[:, 2],
                            n_frames=ORBIT["n_frames"], angle_range=ORBIT["angle_range"])
            want = np.stack(orbit_frames(mine, ORBIT["n_frames"]))
            assert np.array_equal(got, want), f"{name}: reference != restatement"
            # the distinct frames (overlay, then the 3 n_frames orbit views) and the reference's order over them
            order = frame_order(ORBIT["n_frames"])
            distinct = np.stack([mine["overlay"]["overlay"]] + [v["overlay"] for v in mine["orbit"]])
            assert np.array_equal(got, distinct[order])
            np.savez_compressed(path, overlay_minus_photo=distinct[0].astype(np.int16) - img,
                                white_minus_orbit=(255 - distinct[1:]).astype(np.uint8), frame_order=np.asarray(order))
        total += os.path.getsize(path)
        print(f"{name}: {os.path.getsize(path)} bytes")
    print(f"total {total} bytes")
    assert total < 300_000


if __name__ == "__main__":
    main()
