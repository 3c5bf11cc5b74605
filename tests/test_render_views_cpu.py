"""CPU: the demo-view restatement (oracle/render_views_ref.py) against the reference's own lookAt and against the
vertex-rotating orbit it replaces; the camera glyph's meshes; the library exports the new entry points."""
import os

import numpy as np
import pytest

from oracle import render_ref
from oracle import render_views_ref as rv

REFERENCE = "/root/reference"


@pytest.mark.skipif(not os.path.isdir(REFERENCE), reason="needs the reference checkout")
def test_look_at_equals_the_reference():
    from oracle import make_golden_render as mg

    ref = mg.load_reference_render()
    for eye, target in [([2.0, -1, -2], [0, 0, 3]), ([2.2 * 3.7, 0, 3.7], [0, 0, 3.7]),
                        ([0.0, -2 * 3.7, 3.7 - 0.001], [0, 0, 3.7]), ([0.3, 0.2, -1.0], [0.1, -0.4, 5.0])]:
        assert np.array_equal(rv.look_at(eye, target), ref.lookAt(eye=eye, target=target))


def test_side_poses_use_numpy_median():
    odd, even = rv.side_poses([3.0, 5.0, 4.0]), rv.side_poses([3.0, 5.0, 4.0, 6.0])
    assert np.allclose(odd[1], rv.look_at([2.2 * 4.0, 0, 4.0], [0, 0, 4.0])[:3])
    assert np.allclose(even[2], rv.look_at([0.0, -9.0, 4.5 - 0.001], [0, 0, 4.5])[:3])
    for q in odd:  # proper rotations
        assert np.allclose(q[:, :3] @ q[:, :3].T, np.eye(3)) and np.isclose(np.linalg.det(q[:, :3]), 1.0)


def test_orbit_by_camera_pose_equals_orbit_by_rotated_vertices():
    from multihmr_b200 import synth

    verts, faces = synth.make_blob_people([(-0.4, 0.1, 3.0), (0.5, 0.0, 3.6)], seed=21)
    K = np.array([[140.0, 0, 80.0], [0, 140.0, 60.0], [0, 0, 1]])
    colors = [(0.8, 0.3, 0.2), (0.2, 0.6, 0.8)]
    c = verts[0].astype(np.float64).mean(0)
    poses = rv.orbit_poses(verts[0], 3, 60)
    for s, (rng, axis) in enumerate(((60, "y"), (-60, "y"), (60, "x"))):
        q = poses[3 * s + 2]
        R = rv.orbit_rotation(rng, axis)
        assert np.allclose(q[:, :3], R)
        moved = (verts.astype(np.float64) - c) @ R.T + c                     # demo.py:181
        a = render_ref.rasterize(moved, faces, K, 120, 160, colors=colors)
        b = rv.rasterize_meshes(list(verts), [faces] * 2, K, 120, 160, R=q[:, :3], t=q[:, 3], colors=colors)
        ok = (a["edge_dist"] >= 1e-3) & (a["depth_gap"] >= 1e-5) & (b["edge_dist"] >= 1e-3) & (b["depth_gap"] >= 1e-5)
        assert ok.mean() > 0.97 and (a["depth"] > 0).mean() > 0.05
        assert np.array_equal(a["index"][ok], b["index"][ok])
        assert np.allclose(a["depth"][ok], b["depth"][ok], rtol=1e-9)
        assert np.abs(a["rgb"][ok].astype(int) - b["rgb"][ok]).max() <= 1


def test_rasterize_meshes_with_one_topology_is_rasterize():
    from multihmr_b200 import synth

    verts, faces = synth.make_blob_people([(-0.3, 0.0, 2.8), (0.4, 0.1, 3.3)], seed=5)
    K = np.array([[120.0, 0, 48.0], [0, 120.0, 40.0], [0, 0, 1]])
    a = render_ref.rasterize(verts, faces, K, 80, 96, colors=[(0.5, 0.5, 0.5), (0.9, 0.1, 0.1)])
    b = rv.rasterize_meshes(list(verts), [faces] * 2, K, 80, 96, colors=[(0.5, 0.5, 0.5), (0.9, 0.1, 0.1)])
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_glyph_meshes_are_closed_and_consistently_wound():
    from multihmr_b200.render import camera_glyph

    topo, meshes = camera_glyph()
    assert [t for t, _, _ in meshes] == [0, 1, 2, 2, 2]
    for t, v, col in meshes:
        f = topo[t]
        assert f.min() == 0 and f.max() == len(v) - 1
        edges = {}
        for tri in f:
            for k in range(3):
                e = (int(tri[k]), int(tri[(k + 1) % 3]))
                edges[e] = edges.get(e, 0) + 1
        for (a, b), n in edges.items():
            assert n == 1 and edges.get((b, a)) == 1, (t, a, b)
        # outward: the signed volume is positive
        p = v[f]
        assert np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() > 0
    cone, box = meshes[0][1], meshes[1][1]
    assert np.isclose(cone[:, 2].min(), -0.2) and np.isclose(cone[:, 2].max(), 0.0)
    assert np.allclose(box.min(0), [-0.1, -0.1, -0.5]) and np.allclose(box.max(0), [0.1, 0.1, -0.2])
    tips = [m[1][np.argmax(np.abs(m[1] - [0.4, 0.0, -0.2]).sum(1))] for m in meshes[2:]]
    assert np.allclose(tips, [[0.6, 0, -0.2], [0.4, 0.2, -0.2], [0.4, 0, 0.0]])


def test_library_exports_view_entry_points():
    from multihmr_b200 import _lib

    lib = _lib.load()
    for n in ("mhmr_render_create_topologies", "mhmr_render_forward_extra", "mhmr_render_view_poses"):
        assert hasattr(lib, n)
        assert n in _lib.declared_symbols()


def test_create_rotating_video_refuses_a_file_name():
    from multihmr_b200 import api

    with pytest.raises(NotImplementedError):
        api.create_rotating_video([], None, None, None, None, fn="rotating.mp4")
    assert api.create_rotating_video([], None, None, None, None) is None


SIDE = ["render_sideviews_3p_160x120", "render_sideviews_2p_224"]
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _close(a, b):
    """Equal but for +-1 where the reference's fp32 3x3 conv may truncate either way (see test_render_cpu)."""
    d = np.abs(a.astype(np.int16) - b.astype(np.int16))
    return d.max() <= 1 and (d == 0).mean() > 0.999


@pytest.mark.parametrize("name", SIDE + ["render_sideviews_empty_160x120"])
def test_restatement_reproduces_sideview_golden(name):
    from multihmr_b200.render import PALETTE
    from oracle import make_golden_render_views as mgv

    img, verts, faces, K, pos = mgv.scene_inputs(name)
    with np.load(os.path.join(GOLDEN_DIR, name + ".npz")) as g:
        gold = 255 - g["white_minus_views"].astype(np.int16)
        dtype = str(g["dtype"])
    if not len(verts):
        assert dtype == "float64" and (gold == 255).all()
        return
    colors = [PALETTE[i] for i in range(len(verts))] + rv.glyph_meshes()[2]
    mine = rv.views(verts, faces, K, *img.shape[:2], img, 1.0, colors, pos[:, 2], side=True)
    for k in range(3):
        assert _close(mine["side"][k]["overlay"], gold[k]), k


def test_restatement_reproduces_orbit_golden():
    from multihmr_b200.render import PALETTE
    from oracle import make_golden_render_views as mgv

    name = "render_orbit_3p_160x120"
    img, verts, faces, K, pos = mgv.scene_inputs(name)
    with np.load(os.path.join(GOLDEN_DIR, name + ".npz")) as g:
        overlay = g["overlay_minus_photo"] + img.astype(np.int16)
        orbit = 255 - g["white_minus_orbit"].astype(np.int16)
        order = g["frame_order"].tolist()
    o = mgv.ORBIT
    assert order == mgv.frame_order(o["n_frames"]) and len(orbit) == 3 * o["n_frames"]
    mine = rv.views(verts, faces, K, *img.shape[:2], img, o["alpha"], [PALETTE[i] for i in range(len(verts))],
                    pos[:, 2], n_frames=o["n_frames"], angle_range=o["angle_range"])
    assert _close(mine["overlay"]["overlay"], overlay)
    for k in range(len(orbit)):
        assert _close(mine["orbit"][k]["overlay"], orbit[k]), k
    with np.load(os.path.join(GOLDEN_DIR, "render_orbit_empty_160x120.npz")) as g:
        assert "none" in g.files


@pytest.mark.skipif(not os.path.isdir(REFERENCE), reason="needs the reference checkout")
def test_reference_show_camera_glyph_equals_camera_glyph():
    """The reference's own show_camera code (utils/render.py:236-274) over the pyvista restatement builds the glyph
    that multihmr_b200.render.camera_glyph returns: the same merged points and the same rendered surface."""
    import sys

    from multihmr_b200.render import camera_glyph
    from oracle import make_golden_render_views as mgv

    render, _ = mgv.load_reference()
    seen = []

    class Capture(mgv._Renderer):
        def render(self, scene, flags=None):
            seen.extend(o for o, _ in scene.nodes if hasattr(o, "faces"))
            return super().render(scene, flags)

    sys.modules["pyrender"].OffscreenRenderer = Capture
    try:
        from multihmr_b200 import synth

        verts, faces = synth.make_blob_people([(0.0, 0.0, 3.0)], seed=2)
        H = rv.look_at([2.0, -1, -2], [0, 0, 3])
        render.render_meshes(np.full((96, 128, 3), 255.0), list(verts), [faces], {
            "focal": np.array([110.0, 110.0]), "princpt": np.array([64.0, 48.0]), "R": H[:3, :3], "t": H[:3, 3]},
            color=[(0.5, 0.2, 0.2)], show_camera=True)
    finally:
        sys.modules["pyrender"].OffscreenRenderer = mgv._Renderer
    ref = [(m.vertices, m.faces, m.material.color[:3]) for m in seen[1:]]
    topo, mine = camera_glyph()
    assert len(ref) == len(mine) == 5
    K = np.array([[110.0, 0, 64.0], [0, 110.0, 48.0], [0, 0, 1]])
    for (rv_, rf, rc), (t, v, c) in zip(ref, mine):
        assert tuple(rc) == tuple(c)
        a, b = np.unique(np.round(rv_, 6), axis=0), np.unique(np.round(v, 6), axis=0)
        assert a.shape == b.shape and np.allclose(a, b, atol=1e-6)
        x = rv.rasterize_meshes([rv_], [rf], K, 96, 128, R=H[:3, :3], t=H[:3, 3], colors=[c])
        y = rv.rasterize_meshes([v], [topo[t]], K, 96, 128, R=H[:3, :3], t=H[:3, 3], colors=[c])
        ok = (x["edge_dist"] > 1e-3) & (y["edge_dist"] > 1e-3)
        assert np.array_equal(x["index"][ok], y["index"][ok])
        assert np.allclose(x["depth"][ok], y["depth"][ok], rtol=1e-6)
        assert np.abs(x["rgb"][ok].astype(int) - y["rgb"][ok]).max() <= 1
