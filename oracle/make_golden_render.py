"""Pins oracle/render_ref.py against the reference's OWN `utils/render.py:render_meshes` and writes
tests/golden/render_*.npz.

Runs ONLY where the reference checkout exists.  It loads /root/reference/utils/render.py UNMODIFIED (as a file, so
that the package's __init__ is not imported), with `pyrender` and `trimesh` replaced by functional shims built on the
restatement: `Scene`, `Mesh.from_trimesh`, `MetallicRoughnessMaterial`, `IntrinsicsCamera`, `DirectionalLight`,
`OffscreenRenderer.render` (RGBA uint8, depth) and `delete`; `Trimesh` with `vertex_normals` / `face_normals`.  The
shims do only what pyrender would do (rasterize + shade); the camera-pose conventions, colour handling, foreground
smoothing and blend are the reference's.  The script asserts shim-run == restatement before writing.  The
files hold the reference's overlay minus the photo (zero off the meshes, so it compresses), the restatement's shaded
colours, depth and person map; the inputs are regenerated from `SCENES` by `scene_inputs`.

Usage:  python -m oracle.make_golden_render            (from the repo root)
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

from oracle import render_ref  # noqa: E402

# (name, H, W, focal, princpt, person positions, R/t?, smooth, alpha, seed)
SCENES = {
    "render_square_224": dict(H=224, W=224, focal=(260.0, 260.0), princpt=(112.0, 112.0),
                              positions=[(-0.7, 0.1, 3.2), (0.15, 0.0, 4.0), (0.9, 0.2, 3.6)], smooth=True,
                              alpha=0.8, seed=11),
    "render_offcentre_333x250": dict(H=250, W=333, focal=(300.0, 290.0), princpt=(140.5, 131.25),
                                     positions=[(-0.4, 0.0, 3.0), (0.5, 0.1, 3.3)], smooth=True, alpha=1.0,
                                     seed=12),
    "render_pose_flat_160x120": dict(H=120, W=160, focal=(150.0, 150.0), princpt=(80.0, 60.0),
                                     positions=[(0.0, 0.0, 0.0), (0.6, 0.0, 0.5)], smooth=False, alpha=0.6,
                                     seed=13, yaw=0.5, eye_t=(0.1, -0.1, 3.5)),
}


def scene_inputs(name):
    """Seeded inputs of one golden scene: photo uint8 [H,W,3], verts [P,V,3], faces, cam_param, colours, alpha."""
    from multihmr_b200 import synth

    sc = SCENES[name]
    H, W = sc["H"], sc["W"]
    verts, faces = synth.make_blob_people(sc["positions"], seed=sc["seed"])
    yy, xx = np.mgrid[0:H, 0:W]
    img = np.stack([(xx * 255 // max(W - 1, 1)), (yy * 255 // max(H - 1, 1)), np.full_like(xx, 96)], -1)
    img = img.astype(np.uint8)
    g = np.random.default_rng(sc["seed"])
    colors = [tuple(float(c) for c in g.integers(1, 225, 3) / 255.0) for _ in range(len(verts))]
    cam = {"focal": np.asarray(sc["focal"]), "princpt": np.asarray(sc["princpt"])}
    if "yaw" in sc:
        a = sc["yaw"]
        cam["R"] = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        cam["t"] = np.asarray(sc["eye_t"])
    return img, verts, faces, cam, colors, sc["alpha"], sc["smooth"]


# ---------------------------------------------------------------------------------------------- shims
_CV2GL = np.diag([1.0, -1.0, -1.0, 1.0])


class _Trimesh:
    def __init__(self, vertices, faces, process=True, **kw):
        self.vertices = np.asarray(vertices, np.float64)
        self.faces = np.asarray(faces, np.int64)

    @property
    def face_normals(self):
        return render_ref.face_normals(torch.from_numpy(self.vertices), torch.from_numpy(self.faces)).numpy()

    @property
    def vertex_normals(self):
        return render_ref.vertex_normals(torch.from_numpy(self.vertices), torch.from_numpy(self.faces)).numpy()


class _Material:
    def __init__(self, metallicFactor=0.0, roughnessFactor=1.0, alphaMode="OPAQUE", baseColorFactor=(1, 1, 1, 1),
                 **kw):
        assert alphaMode == "OPAQUE"
        self.metallic, self.roughness = float(metallicFactor), float(roughnessFactor)
        self.color = tuple(float(c) for c in baseColorFactor)


class _Mesh:
    @staticmethod
    def from_trimesh(mesh, material=None, smooth=True):
        m = _Mesh()
        m.vertices, m.faces, m.material, m.smooth = mesh.vertices, mesh.faces, material, smooth
        m.normals = mesh.vertex_normals if smooth else None
        return m


class _Camera:
    def __init__(self, fx, fy, cx, cy, znear=0.05, zfar=100.0):
        self.K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
        assert znear == render_ref.ZNEAR and zfar == render_ref.ZFAR


class _Light:
    def __init__(self, color=None, intensity=1.0):
        assert color is None or np.allclose(color, 1.0)
        self.intensity = float(intensity)


class _Scene:
    def __init__(self, ambient_light=(0.0, 0.0, 0.0), bg_color=None):
        assert np.allclose(ambient_light, render_ref.AMBIENT)
        self.nodes = []

    def add(self, obj, name=None, pose=None):
        self.nodes.append((obj, np.eye(4) if pose is None else np.asarray(pose, np.float64)))


class _Renderer:
    def __init__(self, viewport_width, viewport_height, point_size=1.0):
        self.W, self.H = int(viewport_width), int(viewport_height)

    def render(self, scene, flags=None):
        meshes = [(o, p) for o, p in scene.nodes if isinstance(o, _Mesh)]
        (cam, cam_pose), = [(o, p) for o, p in scene.nodes if isinstance(o, _Camera)]
        (light, light_pose), = [(o, p) for o, p in scene.nodes if isinstance(o, _Light)]
        assert np.array_equal(light_pose, cam_pose), "the restatement's light sits at the camera"
        for _, p in meshes:
            assert np.array_equal(p, np.eye(4))
        world_to_cv = _CV2GL @ np.linalg.inv(cam_pose)
        faces = meshes[0][0].faces
        assert all(np.array_equal(m.faces, faces) for m, _ in meshes)
        mats = {(m.material.metallic, m.material.roughness) for m, _ in meshes}
        assert len(mats) == 1
        (metallic, roughness), = mats
        smooth = meshes[0][0].smooth
        out = render_ref.rasterize(
            np.stack([m.vertices for m, _ in meshes]), faces, cam.K, self.H, self.W, R=world_to_cv[:3, :3],
            t=world_to_cv[:3, 3], normals=np.stack([m.normals for m, _ in meshes]) if smooth else None,
            colors=np.asarray([m.material.color[:3] for m, _ in meshes]), intensity=light.intensity,
            metallic=metallic, roughness=roughness, smooth=smooth)
        rgba = np.concatenate([out["rgb"], np.where(out["depth"] > 0, 255, 0).astype(np.uint8)[..., None]], -1)
        return rgba, out["depth"].astype(np.float32)

    def delete(self):
        pass


def install_shims():
    pyrender = types.ModuleType("pyrender")
    pyrender.Scene, pyrender.Mesh, pyrender.MetallicRoughnessMaterial = _Scene, _Mesh, _Material
    pyrender.IntrinsicsCamera, pyrender.DirectionalLight, pyrender.OffscreenRenderer = _Camera, _Light, _Renderer
    pyrender.RenderFlags = types.SimpleNamespace(RGBA=1)
    sys.modules["pyrender"] = pyrender
    trimesh = types.ModuleType("trimesh")
    trimesh.Trimesh = _Trimesh
    sys.modules["trimesh"] = trimesh


def load_reference_render():
    install_shims()
    spec = importlib.util.spec_from_file_location("_ref_render", os.path.join(REFERENCE, "utils", "render.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ref = load_reference_render()
    total = 0
    for name in SCENES:
        img, verts, faces, cam, colors, alpha, smooth = scene_inputs(name)
        got = ref.render_meshes(img.copy(), list(verts), [faces] * len(verts), cam, color=list(colors), alpha=alpha,
                                smooth=smooth)
        mine = render_ref.render_meshes(img, verts, faces, np.array([[cam["focal"][0], 0, cam["princpt"][0]],
                                                                       [0, cam["focal"][1], cam["princpt"][1]],
                                                                       [0, 0, 1]]),
                                        R=cam.get("R"), t=cam.get("t"), colors=np.asarray(colors), alpha=alpha,
                                        smooth=smooth)
        assert np.array_equal(got, mine["overlay"]), f"{name}: reference run != restatement"
        fg = int((mine["depth"] > 0).sum())
        assert fg > 0.05 * img.shape[0] * img.shape[1], f"{name}: too little foreground ({fg} px)"
        path = os.path.join(GOLDEN, name + ".npz")
        np.savez_compressed(path, overlay_minus_photo=got.astype(np.int16) - img, rgb=mine["rgb"], depth=mine["depth"].astype(np.float32),
                            index=mine["index"])
        total += os.path.getsize(path)
        print(f"{name}: {fg} foreground px, {os.path.getsize(path)} bytes")
    print(f"total {total} bytes")
    assert total < 300_000


if __name__ == "__main__":
    main()
