"""CPU: the fp64 restatement of the mesh overlay (oracle/render_ref.py) against the committed goldens (the reference's
own `render_meshes` run through pyrender / trimesh shims, oracle/make_golden_render.py) and against second sources
(analytic depth and silhouette area, fill rule, winding, angle-weighted normals); the library exports the renderer."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import render_ref

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _K(f, cx, cy, fy=None):
    return np.array([[f, 0, cx], [0, f if fy is None else fy, cy], [0, 0, 1]], np.float64)


@pytest.mark.parametrize("name", ["render_square_224", "render_offcentre_333x250", "render_pose_flat_160x120"])
def test_restatement_reproduces_golden(name):
    from oracle import make_golden_render as mg

    img, verts, faces, cam, colors, alpha, smooth = mg.scene_inputs(name)
    K = _K(cam["focal"][0], cam["princpt"][0], cam["princpt"][1], fy=cam["focal"][1])
    out = render_ref.render_meshes(img, verts, faces, K, R=cam.get("R"), t=cam.get("t"), colors=np.asarray(colors),
                                   alpha=alpha, smooth=smooth)
    with np.load(os.path.join(GOLDEN_DIR, name + ".npz")) as g:
        gold = {k: g[k] for k in g.files}
    assert np.array_equal(out["index"], gold["index"])
    assert np.array_equal(out["depth"].astype(np.float32), gold["depth"])
    d = np.abs(out["rgb"].astype(np.int16) - gold["rgb"])
    assert d.max() <= 1 and (d == 0).mean() > 0.999
    # The overlay truncates fg * blend + (1 - fg) * img to uint8, with fg the reference's fp32 3x3 conv.  Its last bit
    # depends on the CPU kernel the conv runs (AVX-512 and AVX2 kernels round 2/9 + ... + 2/9 - 1 differently), so
    # where fg > 0 and the exact value lies within 1e-3 of an integer the truncation may go either way: +-1 there.
    # Every other value must be exact.
    overlay = gold["overlay_minus_photo"] + img.astype(np.int16)
    fgm = (gold["depth"] > 0).astype(np.float64)
    H, W = fgm.shape
    pad = np.pad(fgm, 1)
    box = sum(pad[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3))
    fg = (np.maximum(2.0 * box / 9.0 - 1.0, 0.0) * fgm)[..., None]
    val = fg * (alpha * gold["rgb"].astype(np.float64) + (1.0 - alpha) * img) + (1.0 - fg) * img
    either = (fg > 0) & (np.abs(val - np.round(val)) < 1e-3)
    d = np.abs(out["overlay"].astype(np.int16) - overlay)
    assert d.max() <= 1 and np.all(d[~either] == 0)
    assert (gold["depth"] > 0).mean() > 0.05


def _plane(z0, tilt, half=2.0):
    """A square plane through (0, 0, z0) with normal (0, -sin, -cos)*, facing the camera, as two triangles."""
    c, s = math.cos(tilt), math.sin(tilt)
    corners = np.array([[-half, -half, 0], [half, -half, 0], [half, half, 0], [-half, half, 0]], np.float64)
    R = np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    v = corners @ R.T + [0, 0, z0]
    return v, np.array([[0, 3, 2], [0, 2, 1]])


@pytest.mark.parametrize("tilt", [0.0, 0.6])
def test_plane_depth_is_the_ray_plane_intersection(tilt):
    v, f = _plane(2.5, tilt)
    K = _K(40.0, 16.3, 12.1)
    out = render_ref.rasterize(v[None], f, K, 24, 32, colors=[[0.5, 0.5, 0.5]])
    assert (out["index"] == 0).all(), "the plane fills the view"
    n = np.cross(v[1] - v[0], v[2] - v[0])
    yy, xx = np.mgrid[0:24, 0:32]
    d = np.stack([(xx + 0.5 - 16.3) / 40.0, (yy + 0.5 - 12.1) / 40.0, np.ones_like(xx, dtype=np.float64)], -1)
    z = (n @ v[0]) / (d @ n)
    np.testing.assert_allclose(out["depth"], z, rtol=1e-12)


def test_sphere_silhouette_area_matches_projected_ellipse():
    from multihmr_b200 import synth

    uv, uf = synth._ellipsoid(64, 128)
    r, c = 0.5, np.array([0.3, -0.2, 4.0])
    f, H, W = 300.0, 120, 140
    out = render_ref.rasterize((uv * r + c)[None], uf, _K(f, 70.0, 60.0), H, W, colors=[[0.5, 0.5, 0.5]])
    area = (out["depth"] > 0).sum()
    L = np.linalg.norm(c)
    yy, xx = np.mgrid[0:H, 0:W]
    d = np.stack([(xx + 0.5 - 70.0) / f, (yy + 0.5 - 60.0) / f, np.ones((H, W))], -1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    inside = (d @ c) ** 2 - (L * L - r * r) >= 0                         # the pixel's ray meets the sphere
    assert abs(area - inside.sum()) <= 0.01 * inside.sum()
    # the cone tangent to the sphere (half-angle a, sin a = r / L) cuts the image plane, whose normal is at theta to
    # the cone's axis, in an ellipse of semi-axes f sin a cos a / (cos^2 theta - sin^2 a) and
    # f sin a / sqrt(cos^2 theta - sin^2 a)
    sa = r / L
    ca, ct = math.sqrt(1 - sa * sa), c[2] / L
    analytic = math.pi * f * f * sa * sa * ca / (ct * ct - sa * sa) ** 1.5
    # the inscribed polygon loses area ~ (pi / n)^2 / 3 of the disc; the analytic value bounds the count from above
    assert 0.985 * analytic <= area <= 1.005 * analytic


def test_quad_split_covers_each_pixel_once():
    # two triangles sharing the diagonal of a quad whose corners fall exactly on pixel corners
    v = np.array([[-1.0, -1.0, 2.0], [1.0, -1.0, 2.0], [1.0, 1.0, 2.0], [-1.0, 1.0, 2.0]])
    for f in (np.array([[0, 3, 2], [0, 2, 1]]), np.array([[0, 3, 1], [3, 2, 1]])):
        K = _K(8.0, 8.0, 8.0)                       # the quad spans pixel coordinates [4, 12] x [4, 12]
        per_face = []
        for k in range(2):
            out = render_ref.rasterize(v[None], f[k:k + 1], K, 16, 16, colors=[[0.5, 0.5, 0.5]])
            per_face.append(out["index"] == 0)
        both = render_ref.rasterize(v[None], f, K, 16, 16, colors=[[0.5, 0.5, 0.5]])
        assert not (per_face[0] & per_face[1]).any(), "a pixel covered twice"
        assert np.array_equal(per_face[0] | per_face[1], both["index"] == 0)
        yy, xx = np.mgrid[0:16, 0:16]
        cx, cy = xx + 0.5, yy + 0.5
        strict = (cx > 4) & (cx < 12) & (cy > 4) & (cy < 12)
        assert (both["index"][strict] == 0).all()
        # top-left: the left and top boundaries are in, the right and bottom ones out (centres at x.5 never sit on
        # an integer boundary here, so the quad holds exactly the 8 x 8 centres inside it)
        assert (both["index"] == 0).sum() == 64


def test_winding_fixtures_cull_as_derived():
    # counter-clockwise on screen (y down: (0,0) -> (0,1) -> (1,0) seen from the camera) is GL's front face
    tri = np.array([[0.0, 0.0, 2.0], [0.0, 1.0, 2.0], [1.0, 0.0, 2.0]])
    K = _K(10.0, 1.0, 1.0)
    front = render_ref.rasterize(tri[None], np.array([[0, 1, 2]]), K, 8, 8, colors=[[0.5, 0.5, 0.5]])
    back = render_ref.rasterize(tri[None], np.array([[0, 2, 1]]), K, 8, 8, colors=[[0.5, 0.5, 0.5]])
    assert (front["index"] == 0).sum() >= 8 and (back["index"] == 0).sum() == 0
    # the front face's normal (v1 - v0) x (v2 - v0) points at the camera (-z)
    n = np.cross(tri[1] - tri[0], tri[2] - tri[0])
    assert n[2] < 0


def test_cube_corner_angle_weighted_normal():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [0, 1, 1], [1, 0, 1]], np.float64)
    # at vertex 0: two triangles on each of the faces z=0, x=0, y=0 (45 deg each at vertex 0)
    f = np.array([[0, 2, 4], [0, 4, 1], [0, 3, 5], [0, 5, 2], [0, 1, 6], [0, 6, 3]])
    vn = render_ref.vertex_normals(torch.from_numpy(v), torch.from_numpy(f)).numpy()
    # each face of the cube contributes 90 degrees in total: the sum is 90 deg x (-1,-1,-1) -> (-1,-1,-1)/sqrt(3)
    np.testing.assert_allclose(vn[0], -np.ones(3) / math.sqrt(3), atol=1e-12)
    # one triangle per face on two faces, both halves of the third: weights 45, 45, 90 deg
    f2 = np.array([[0, 2, 4], [0, 3, 5], [0, 1, 6], [0, 6, 3]])
    w = np.array([math.pi / 4, math.pi / 4, math.pi / 2])  # z=0, x=0, y=0
    expect = -(w[0] * np.array([0, 0, 1.0]) + w[1] * np.array([1.0, 0, 0]) + w[2] * np.array([0, 1.0, 0]))
    got = render_ref.vertex_normals(torch.from_numpy(v), torch.from_numpy(f2)).numpy()[0]
    np.testing.assert_allclose(got, expect / np.linalg.norm(expect), atol=1e-12)


def test_library_exports_renderer():
    from multihmr_b200 import _lib

    lib = _lib.load()
    for n in ("mhmr_render_create", "mhmr_render_forward", "mhmr_render_destroy", "mhmr_render_info"):
        assert hasattr(lib, n)
        assert n in _lib.declared_symbols()


def test_render_meshes_refuses_what_it_does_not_render():
    from multihmr_b200 import render

    img = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(NotImplementedError):
        render.render_meshes(img, [], [], {"focal": (1, 1), "princpt": (4, 4)}, show_camera=True)
    with pytest.raises(ValueError):
        render.render_meshes(img + 0.5, [], [], {"focal": (1, 1), "princpt": (4, 4)})
    out = render.render_meshes(img.astype(np.float64) + 255.0, [], [], {"focal": (1, 1), "princpt": (4, 4)})
    assert out.dtype == np.uint8 and (out == 255).all()
