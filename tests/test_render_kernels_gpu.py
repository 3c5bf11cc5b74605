"""GPU: the renderer's kernels (csrc/render.cu) where rasterizers go wrong, against exact and fp64 references
(render_kernels_util, oracle/render_ref.py, oracle/render_views_ref.py).

A. exact tie scenes: ownership of every pixel, edges and vertices included, equals the oracle's top-left rule;
B. watertightness inside one mesh whose interior edges pass through pixel centres with rounded edge values;
C. depth ties go to the smaller (mesh, face) key;  D. the tools/bench_render.py workloads against fp64 (check_view);
E. more queued big triangles than the queue holds;  F. the depth key's bit limits;  G. the device count contract;
H. the pose kernel against a numpy restatement.

Every comparison states its tolerance next to it, and every comparison has a sensitivity check: a reference with one
plausible mistake lands outside that tolerance, and the output shows by how much."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import render_ref
from oracle import render_views_ref as rv

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import render_kernels_util as ru  # noqa: E402
from test_render_gpu import check_view  # noqa: E402

DEV = "cuda"
U32 = 2.0 ** -24


def _np(out, b=0):
    return {k: v[b].cpu().numpy() for k, v in out.items()}


def _photo(H, W, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (1, H, W, 3), dtype=np.uint8)).to(DEV)


def _palette(n):
    from multihmr_b200.render import PALETTE

    return np.asarray([PALETTE[i % len(PALETTE)] for i in range(n)], np.float64)


# ------------------------------------------------------------------------------------------ A. exact tie scenes
EXACT = ru.exact_scenes()


@pytest.mark.parametrize("name", list(EXACT))
def test_exact_scene_ownership_at_every_pixel(name):
    """All arithmetic is exact (test_render_kernels_cpu proves it), so the kernels must reproduce the top-left rule
    bit for bit: tolerance 0 on the index map, 0 on the depth."""
    from multihmr_b200.render import Renderer

    s = EXACT[name]
    H, W, T = s["H"], s["W"], len(s["verts"])
    r = Renderer([[0, 1, 2]], DEV)
    assert r.face_bits == 0
    out = _np(r.render(torch.from_numpy(s["verts"]), torch.tensor(s["K"], dtype=torch.float32)[None],
                       _photo(H, W, 1), colors=torch.from_numpy(_palette(T)), depth=True, index=True))
    ref = render_ref.rasterize(s["verts"], [[0, 1, 2]], s["K"], H, W, colors=_palette(T), device=DEV)
    bad = out["index"] != ref["index"]
    assert not bad.any(), f"{name}: owner differs at {int(bad.sum())} pixels, e.g. {np.argwhere(bad)[:5].tolist()}"
    fg = out["index"] >= 0
    assert np.array_equal(out["depth"][fg], s["z"][out["index"][fg]]), "depth is the plane's z exactly"
    assert (out["depth"][~fg] == 0).all()
    for box in s.get("outlines", []):
        assert fg[ru.inside_outline(H, W, box)].all(), "a hole inside the grid"
    for centre, rad in s.get("fans", []):
        assert fg[ru.inside_fan(H, W, centre, rad)].all(), "a hole inside a fan"
    on_edge = int((ref["edge_dist"] == 0).sum())
    msg = [f"{name}: {T} triangles, {on_edge} of {H * W} pixel centres exactly on an edge, all owned as the oracle"]
    for rule in ("bottom_right", "both"):
        other, _ = ru.owner_map(s["verts"], s["K"], H, W, rule)
        diff = int((other != out["index"]).sum())
        msg.append(f"tie rule {rule}: {diff} pixels differ")
        assert diff >= 10, f"the {rule} reference must differ from the kernels"
    print("; ".join(msg))


# ------------------------------------------------------------------------------------- B. watertight inside a mesh
WATERTIGHT = ru.watertight_scenes()


@pytest.mark.parametrize("name", list(WATERTIGHT))
def test_no_crack_along_interior_edges(name):
    """Every pixel the oracle covers that lies more than 1e-3 px from a silhouette edge (interior shared edges are not
    flagged) is covered.  Pixel centres on a vertex are reported apart (see test_render_kernels_cpu)."""
    from multihmr_b200.render import Renderer

    s = WATERTIGHT[name]
    v, f, K, H, W = s["verts"], s["faces"], s["K"], s["H"], s["W"]
    r = Renderer(f, DEV, num_verts=v.shape[1])
    out = _np(r.render(torch.from_numpy(v), torch.tensor(K, dtype=torch.float32)[None], _photo(H, W, 2),
                       depth=True, index=True))
    ref = render_ref.rasterize(v, f, K, H, W, colors=_palette(1), device=DEV)
    must = (ref["depth"] > 0) & (ru.silhouette_distance(v[0], f, K, H, W) > 1e-3)
    on_vertex = ru.vertex_distance(v[0], K, H, W) <= 1e-3
    hole = must & (out["depth"] == 0)
    own = ru.per_triangle_coverage_f32(v[0], f, K, H, W, canonical=False)
    print(f"{name}: {int(must.sum())} interior pixels ({int((ref['edge_dist'] < 1e-3).sum())} on an edge): "
          f"{int((hole & ~on_vertex).sum())} cracks, {int((hole & on_vertex).sum())} on vertices; per-triangle "
          f"planes would leave {int((must & ~own & ~on_vertex).sum())}")
    assert not (hole & ~on_vertex).any(), f"cracks at {np.argwhere(hole & ~on_vertex)[:5].tolist()}"
    assert (must & ~own & ~on_vertex).any(), "sensitivity: per-triangle planes must crack this scene"


# ---------------------------------------------------------------------------------------- C. depth ties by the key
def _blob3():
    from multihmr_b200 import synth

    verts, faces = synth.make_blob_people([(-0.5, 0.1, 3.2), (0.3, 0.0, 3.5), (0.55, 0.05, 3.3)], seed=4)
    K = torch.tensor([[150.0, 0, 80.3], [0, 150.0, 60.2], [0, 0, 1]])[None]
    return verts, faces, K, _photo(120, 160, 3)


@pytest.mark.parametrize("order", [[0, 1, 0, 2, 1], [1, 0, 2, 0, 1], [2, 2, 1, 0, 0]])
def test_coincident_persons_go_to_the_lower_index(order):
    """Bit-identical copies tie in depth at every pixel: the lower list index wins there.  Exact: index, depth and
    overlay equal those of a render of the distinct persons in the winners' colours."""
    from multihmr_b200.render import Renderer

    verts, faces, K, img = _blob3()
    r = Renderer(faces, DEV)
    cols = np.random.default_rng(sum(order)).uniform(0.1, 0.9, (len(order), 3))
    got = _np(r.render(torch.from_numpy(verts[order]), K, img, colors=torch.tensor(cols, dtype=torch.float32),
                       alpha=0.8, depth=True, index=True))
    first = [order.index(u) for u in range(3)]
    want = _np(r.render(torch.from_numpy(verts), K, img, colors=torch.tensor(cols[first], dtype=torch.float32),
                        alpha=0.8, depth=True, index=True))
    exp_index = np.where(want["index"] >= 0, np.asarray(first)[np.maximum(want["index"], 0)], -1)
    assert np.array_equal(got["index"], exp_index) and np.array_equal(got["depth"], want["depth"])
    assert np.array_equal(got["overlay"], want["overlay"])
    last = [len(order) - 1 - order[::-1].index(u) for u in range(3)]
    wrong = _np(r.render(torch.from_numpy(verts), K, img, colors=torch.tensor(cols[last], dtype=torch.float32),
                         alpha=0.8))
    d = int((wrong["overlay"] != got["overlay"]).any(-1).sum())
    print(f"order {order}: winners {first}; ties to the higher index would change {d} pixels")
    assert d > 100


def test_coincident_prop_loses_to_the_person():
    """A prop identical to person 0 is mesh P + 0 of the key: the person wins every tie (exact)."""
    from multihmr_b200.render import Renderer

    verts, faces, K, img = _blob3()
    r = Renderer(faces, DEV, topologies=[faces])
    kw = dict(colors=torch.tensor(_palette(3), dtype=torch.float32), alpha=0.8, depth=True, index=True)
    base = _np(r.render(torch.from_numpy(verts), K, img, **kw))
    got = _np(r.render(torch.from_numpy(verts), K, img, props=[(0, torch.from_numpy(verts[0]), (1.0, 0.0, 0.0))],
                       **kw))
    for k in base:
        assert np.array_equal(got[k], base[k]), k
    alone = _np(r.render(torch.from_numpy(verts[1:]), K, img, props=[(0, torch.from_numpy(verts[0]),
                                                                     (1.0, 0.0, 0.0))],
                         colors=torch.tensor(_palette(3)[1:], dtype=torch.float32), alpha=0.8, index=True))
    assert (alone["index"] == 2).sum() > 100, "the prop is drawn as mesh P + 0 where the person is absent"
    d = int((alone["overlay"] != got["overlay"]).any(-1).sum())
    print(f"prop vs person 0: the prop winning would change {d} pixels")
    assert d > 100


# -------------------------------------------------------------------------------------- D. production sizes, fp64
PROD = ru.production_scenes()


# Flagged pixels (within 1e-3 px of an edge, or within 1e-5 of the second-nearest surface) per foreground pixel: the
# blob goldens of test_render_gpu have 0.15-0.45 %; the production scenes, with 16 times the faces per person, and the
# side view with the camera glyph's coincident parts, reach about 1.1 %.
MAX_FLAGGED_FG = 0.015


def _compare_view(tag, got, got1, ref, img, alpha, max_flagged_fg, meshes, R=None, t=None, ref_overlay=None):
    """check_view (person map off the flagged pixels, depth 1e-5 relative, colour and composite 1 level), with two
    refinements for production sizes:
    - depth: on faces seen almost edge-on the fp32 rounding bound of the depth (ru.depth_bound, derived there)
      exceeds 1e-5; there the depth must lie within that bound instead;
    - composite: a flagged pixel may legitimately take the other surface (another person, or with flat shading the
      neighbouring face), whose colour differs by more than a level, so the composite is not compared on flagged
      pixels, as the person map already is not.
    At most `max_flagged_fg` flagged pixels per foreground pixel.  meshes: (verts list, faces list, K) of the
    oracle's view.  Prints the flagged fraction (per image and per foreground pixel) and the worst errors."""
    bound = ru.depth_bound(meshes[0], meshes[1], meshes[2], ref, R=R, t=t)
    flag = (ref["edge_dist"] < 1e-3) | (ref["depth_gap"] < 1e-5)
    fg = ~flag & (ref["depth"] > 0)
    wide = fg & (bound > 1e-5)
    rel = np.abs(got["depth"].astype(np.float64) - ref["depth"]) / np.where(ref["depth"] > 0, ref["depth"], 1.0)
    assert (rel[wide] <= bound[wide]).all(), f"{tag}: depth outside its rounding bound, worst err/bound " \
                                             f"{(rel[wide] / bound[wide]).max():.3g}"
    ref = dict(ref, depth=np.where(wide, got["depth"], ref["depth"]))
    if ref_overlay is None:
        ref_overlay = render_ref.composite(ref["rgb"], ref["depth"], img, alpha)
    ref_overlay = np.where(flag[..., None], got["overlay"], ref_overlay)
    nfg = max(int((ref["depth"] > 0).sum()), 1)
    assert flag.sum() / nfg <= max_flagged_fg, f"{tag}: {int(flag.sum())} pixels flagged, {nfg} foreground"
    check_view(got, got1, ref, img, alpha, ref_overlay=ref_overlay, max_flagged=1.0, tag=tag)
    frac, derr, cerr = ru.view_errors(got, got1, ref)
    print(f"{tag}: flagged {100 * frac:.4f} % of the image, {100 * flag.sum() / nfg:.3f} % of the foreground "
          f"(bound {100 * max_flagged_fg:.3f} %); worst "
          f"depth rel err {derr:.2e} (tol 1e-5; {int(wide.sum())} px on near edge-on faces within their bound, worst "
          f"err/bound {(rel[wide] / bound[wide]).max(initial=0):.3f}); worst colour {cerr} level(s) (tol 1)")
    return bound


PROD_CASES = [("896x896_4p", 0, True), ("896x896_4p", 0, False), ("1920x1080_20p", 0, True),
              ("offcentre_1920x1080_6p", 0, True)] + [("rotate20_1920x1080_3p", b, True) for b in (0, 7, 13, 19)]


@pytest.mark.parametrize("name,view,smooth", PROD_CASES)
def test_production_view_against_fp64(name, view, smooth):
    from multihmr_b200.render import Renderer

    s = PROD[name]
    H, W, P = s["H"], s["W"], len(s["verts"])
    r = Renderer(s["faces"], DEV)
    img = _photo(H, W, len(name))
    K = torch.tensor(s["K"][view:view + 1], dtype=torch.float32)
    pose = None if s["pose"] is None else s["pose"][view:view + 1]
    kw = dict(pose=pose, colors=torch.tensor(_palette(P), dtype=torch.float32), smooth=smooth, depth=True,
              index=True)
    got = _np(r.render(torch.from_numpy(s["verts"]), K, img, alpha=0.8, **kw))
    got1 = _np(r.render(torch.from_numpy(s["verts"]), K, img, alpha=1.0, **kw))
    R, t = (None, None) if pose is None else (pose[0, :, :3], pose[0, :, 3])
    ref = render_ref.rasterize(s["verts"], s["faces"], s["K"][view], H, W, R=R, t=t, colors=_palette(P),
                               smooth=smooth, device=DEV, chunk_pairs=1 << 21)
    tag = f"{name} view {view} {'smooth' if smooth else 'flat'}"
    bound = _compare_view(tag, got, got1["overlay"], ref, img[0].cpu().numpy(), 0.8, MAX_FLAGGED_FG,
                          (list(s["verts"]), [s["faces"]] * P, s["K"][view]), R=R, t=t)
    if (name, view) == ("rotate20_1920x1080_3p", 19):
        # persons turned 60 degrees about the first one come close to the camera, with faces large enough on screen
        # for screen-space interpolation to show (on the unrotated 1080p scene it stays just inside: 0.97x)
        ss = ru.screen_space_depth(s["verts"], s["faces"], s["K"][view], ref, R=R, t=t)
        ok = ((ref["edge_dist"] >= 1e-3) & (ref["depth_gap"] >= 1e-5) & (ref["depth"] > 0))
        ratio = np.abs(ss[ok] - got["depth"][ok]) / ref["depth"][ok] / np.maximum(bound[ok], 1e-5)
        print(f"{tag}: screen-space barycentrics would be {ratio.max():.1f}x the depth tolerance "
              f"({int((ratio > 1).sum())} px outside)")
        assert ratio.max() > 1.0


def test_render_views_production_frames():
    """tools/bench_render.py's demo orbit (1920 x 1080, 3 persons, n_frames 20, angle_range 60) with the side views:
    an orbit frame and the side view, with the camera glyph, against fp64 at the oracle's fp64 poses."""
    from multihmr_b200.render import Renderer, camera_glyph

    verts, faces, K, H, W = ru.demo_views_scene()
    P = len(verts)
    r = Renderer(faces, DEV, topologies=camera_glyph()[0])
    t = {"v3d": torch.from_numpy(verts).to(DEV), "det_idx": torch.zeros(3, P, dtype=torch.int32, device=DEV),
         "count": torch.full((1,), P, dtype=torch.int32, device=DEV),
         "transl_pelvis": torch.from_numpy(verts.mean(1)).to(DEV)}
    photo = _photo(H, W, 9)
    kw = dict(orbit=(20, 60), side=True, depth=True, index=True)
    Kt = torch.tensor(K, dtype=torch.float32)[None]
    a = r.render_views(t, photo, Kt, alpha=0.8, **kw)
    a1 = r.render_views(t, photo, Kt, alpha=1.0, **kw)
    assert a["rank"].tolist() == [0, 1, 2]
    white = np.full((H, W, 3), 255, np.uint8)
    gv, gf, gc = rv.glyph_meshes()
    orbit = rv.orbit_poses(verts[0], 20, 60)
    side = rv.side_poses(verts.mean(1)[:, 2])
    for tag, w, q, glyph in (("orbit frame 27", 1 + 27, orbit[27], False), ("side view", 1 + 60 + 1, side[1], True)):
        lv, lf, lc = list(verts), [faces] * P, list(_palette(P))
        if glyph:
            lv, lf, lc = lv + gv, lf + gf, lc + gc
        ref = rv.rasterize_meshes(lv, lf, K, H, W, R=q[:, :3], t=q[:, 3], colors=lc, device=DEV,
                                  chunk_pairs=1 << 21)
        alpha, bg = (1.0, white.astype(np.float64)) if glyph else (0.8, white)
        seq = torch.cat([a["overlay"][:1], a["orbit"][0], a["side"][0]])
        seq1 = torch.cat([a1["overlay"][:1], a1["orbit"][0], a1["side"][0]])
        got = {"overlay": seq[w].cpu().numpy(), "depth": a["depth"][0, w].cpu().numpy(),
               "index": a["index"][0, w].cpu().numpy()}
        _compare_view(f"render_views 1080p {tag}", got, seq1[w].cpu().numpy(), ref, white, alpha,
                      MAX_FLAGGED_FG, (lv, lf, K), R=q[:, :3], t=q[:, 3],
                      ref_overlay=render_ref.composite(ref["rgb"], ref["depth"], bg, alpha))
        if glyph:
            assert (got["index"] >= P).any(), "the glyph is visible in the side view"


# ----------------------------------------------------------------------------------------- E. queue overflow
def test_queue_overflow_equals_per_view_calls():
    """9 views x 64 persons x 2048 sliver faces queue 1 179 648 big triangles, over the queue's 2^20; each view
    alone queues 131 072 (test_render_kernels_cpu proves both counts).  The excess is rasterized by its own thread:
    the whole call must equal the per-view calls (drawn from the queue alone) bit for bit, and two views agree with
    fp64 under check_view.  64 overlapping layers of slivers put about 10 % of the foreground within 1e-3 px of an
    edge; the flagged bound is 15 %."""
    from multihmr_b200.render import Renderer

    v, f, K, pose = ru.sliver_scene()
    B, P, H, W = ru.SLIVER["views"], ru.SLIVER["persons"], ru.SLIVER["H"], ru.SLIVER["W"]
    r = Renderer(f, DEV)
    img = _photo(H, W, 5)
    kw = dict(colors=torch.tensor(_palette(P), dtype=torch.float32), alpha=0.8, depth=True, index=True)
    Kt = torch.tensor(K, dtype=torch.float32)
    vt = torch.from_numpy(v)
    whole = r.render(vt, Kt, img, view_image=[0] * B, pose=pose, **kw)
    for b in range(B):
        one = r.render(vt, Kt[b:b + 1], img, view_image=[0], pose=pose[b:b + 1], **kw)
        for k in whole:
            assert torch.equal(whole[k][b], one[k][0]), (k, b)
    whole1 = r.render(vt, Kt, img, view_image=[0] * B, pose=pose, **dict(kw, alpha=1.0))
    for b in (0, B - 1):
        ref = render_ref.rasterize(v, f, K[b], H, W, R=pose[b, :, :3], t=pose[b, :, 3], colors=_palette(P),
                                   device=DEV, chunk_pairs=1 << 21)
        _compare_view(f"slivers view {b}", _np(whole, b), whole1["overlay"][b].cpu().numpy(), ref,
                      img[0].cpu().numpy(), 0.8, 0.15, (list(v), [f] * P, K[b]), R=pose[b, :, :3], t=pose[b, :, 3])


# ------------------------------------------------------------------------------------------ F. depth-key limits
def _key_renderer(F, topologies=None):
    """F faces: 0..F-2 degenerate (three collinear vertices), F-1 the real triangle (vertices 3, 4, 5)."""
    from multihmr_b200.render import Renderer

    faces = np.zeros((F, 3), np.int32)
    faces[:] = [0, 1, 2]
    faces[-1] = [3, 4, 5]
    return Renderer(faces, DEV, num_verts=6, topologies=topologies)


def _cell_tri(cell, ncol, z=2.0, f=64.0, c=(64.0, 48.0)):
    """A front-facing triangle in cell `cell` of a grid of 20-px cells, vertices off the pixel centres."""
    u0, v0 = 3.3 + 20 * (cell % ncol), 2.7 + 20 * (cell // ncol)
    scr = ru.orient_front(np.array([[[u0, v0], [u0 + 15.1, v0 + 2.3], [u0 + 4.2, v0 + 14.6]]]))[0]
    zz = np.array([z, z + 0.1, z + 0.2])
    return np.stack([(scr[:, 0] - c[0]) * zz / f, (scr[:, 1] - c[1]) * zz / f, zz], 1).astype(np.float32)


def _key_case(F, P, drawn, prop, H=96, W=128):
    r = _key_renderer(F, topologies=[np.array([[0, 1, 2]])] if prop else None)
    verts = np.zeros((P, 6, 3), np.float32)
    verts[:, :3] = [[0, 0, 2.0], [0.1, 0, 2.0], [0.2, 0, 2.0]]       # collinear: faces 0..F-2 cover nothing
    tris = {}
    for k, p in enumerate(drawn):
        verts[p, 3:] = tris[p] = _cell_tri(k, W // 20)
    pimg = torch.ones(P, dtype=torch.int32)                            # image 1: no view shows it
    pimg[list(drawn)] = 0
    props = None
    if prop:
        tris[P] = _cell_tri(len(drawn), W // 20)
        props = [(0, torch.from_numpy(tris[P]), (0.9, 0.2, 0.1))]
    K = np.array([[64.0, 0, 64.0], [0, 64.0, 48.0], [0, 0, 1]])
    cols = _palette(P)
    img = _photo(H, W, 7)
    kw = dict(person_image=pimg, colors=torch.tensor(cols, dtype=torch.float32), smooth=False, depth=True,
              index=True, props=props)
    got = _np(r.render(torch.from_numpy(verts), torch.tensor(K, dtype=torch.float32)[None], img, alpha=0.8, **kw))
    got1 = _np(r.render(torch.from_numpy(verts), torch.tensor(K, dtype=torch.float32)[None], img, alpha=1.0, **kw))
    ids = sorted(tris)
    lc = [cols[i] if i < P else (0.9, 0.2, 0.1) for i in ids]
    ref = rv.rasterize_meshes([tris[i] for i in ids], [[[0, 1, 2]]] * len(ids), K, H, W, colors=lc, smooth=False,
                              device=DEV)
    ref["index"] = np.where(ref["index"] >= 0, np.asarray(ids)[np.maximum(ref["index"], 0)], -1)
    _compare_view(f"F={F} P={P} ids {ids}", got, got1["overlay"], ref, img[0].cpu().numpy(), 0.8, 0.05,
                  ({i: tris[i] for i in ids}, {i: [[0, 1, 2]] for i in ids}, K))
    for i in ids:
        assert (got["index"] == i).sum() > 50, f"mesh {i} must be drawn"
    return r


def test_depth_key_bit31_decodes_person_prop_and_face():
    """2^20 + 1 faces: 21 face bits, 11 mesh bits; 2047 persons + 1 prop = 2^11, so the prop's key sets bit 31.  Only
    face F-1 is a real triangle: a wrong decode would set up a degenerate face.  Persons outside {0, 1, 1023, 1024,
    2045, 2046} sit in an image no view shows."""
    r = _key_case((1 << 20) + 1, 2047, [0, 1, 1023, 1024, 2045, 2046], prop=True)
    assert r.face_bits == 21


@pytest.mark.parametrize("F,bits", [(1 << 17, 17), ((1 << 17) + 1, 18)])
def test_face_bits_boundary(F, bits):
    """F = 2^k needs k face bits, 2^k + 1 needs k + 1.  The largest person id 2^(32-bits) - 1 with face F - 1 fills
    the key's low word (all ones at F = 2^17); one person more is refused."""
    pmax = 1 << (32 - bits)
    r = _key_case(F, pmax, [0, pmax - 1], prop=False)
    assert r.face_bits == bits
    with pytest.raises(AssertionError, match="depth key"):
        r.render(torch.zeros(pmax + 1, 6, 3), torch.tensor([[[64.0, 0, 64], [0, 64, 48], [0, 0, 1]]]),
                 _photo(8, 8, 0))


# -------------------------------------------------------------------------------------------- G. count contract
@pytest.mark.parametrize("count", [3 + 5, (1 << 31) - 1, 0, -1])
def test_device_count_is_clamped_to_zero_and_max_persons(count):
    from multihmr_b200.render import Renderer

    verts, faces, K, img = _blob3()
    r = Renderer(faces, DEV)
    kw = dict(alpha=0.8, depth=True, index=True)
    got = r.render(torch.from_numpy(verts), K, img, count=torch.tensor([count], dtype=torch.int32, device=DEV), **kw)
    if count > 0:
        want = r.render(torch.from_numpy(verts), K, img, count=3, **kw)
        for k in want:
            assert torch.equal(got[k], want[k]), k
    else:
        assert torch.equal(got["overlay"], img) and (got["depth"] == 0).all() and (got["index"] == -1).all()
    full = r.render(torch.from_numpy(verts), K, img, **kw)
    assert (full["index"] >= 0).sum() > 1000, "sensitivity: the persons are visible when counted"


def test_person_of_an_unshown_image_is_not_drawn():
    from multihmr_b200.render import Renderer

    verts, faces, K, img = _blob3()
    r = Renderer(faces, DEV)
    imgs = torch.cat([img, _photo(120, 160, 8)])
    cols = torch.tensor(_palette(3), dtype=torch.float32)
    got = _np(r.render(torch.from_numpy(verts), K, imgs, person_image=torch.tensor([0, 1, 0], dtype=torch.int32),
                       view_image=[0], colors=cols, depth=True, index=True))
    want = _np(r.render(torch.from_numpy(verts[[0, 2]]), K, imgs, view_image=[0], colors=cols[[0, 2]], depth=True,
                        index=True))
    assert np.array_equal(got["index"], np.where(want["index"] == 1, 2, want["index"]))
    assert np.array_equal(got["depth"], want["depth"]) and np.array_equal(got["overlay"], want["overlay"])
    all3 = _np(r.render(torch.from_numpy(verts), K, imgs, view_image=[0], colors=cols, index=True))
    assert (all3["index"] == 1).sum() > 100, "sensitivity: person 1 is visible when its image is shown"


# ----------------------------------------------------------------------------------------------- H. pose kernel
def _pose_case(name):
    """(images, max_persons, count, person_image, verts, pelvis, transl) of one case."""
    g = np.random.default_rng(len(name))
    V = 300                                                     # > 256: the vertex sum strides
    if name in ("4img_interleaved_4096", "count_above_max", "count_negative"):
        images, Pm = 4, 4096
        ids = [0] * 601 + [1] * 64 + [2] * 41 + [4, -2]         # image 3 empty; 4 and -2 outside [0, images)
        count = len(ids)
    else:                                                       # even and odd counts with ties in the middle
        images, Pm = 2, 16
        ids = [0] * 4 + [1] * 5
        count = len(ids)
    ids = np.asarray(ids)[g.permutation(len(ids))]
    pimg = np.concatenate([ids, g.choice([0, 1, 2, 7, -3], Pm - len(ids))]).astype(np.int32)   # stale past count
    verts = g.uniform(-1, 1, (Pm, V, 3)) * [0.4, 0.9, 0.2] + g.uniform(-2, 2, (Pm, 1, 3)) + [0, 0, 5]
    tz = 2.0 + 0.5 * g.integers(0, 6, Pm)                       # exact ties in transl z
    pz = 2.0 + 0.25 * g.integers(0, 8, Pm)                      # and in pelvis z
    if name == "even_odd_ties":
        first = np.nonzero(pimg[:count] == 0)[0]
        pz[first] = [3.0, 2.5, 3.25, 2.5]                        # even, tied below the middle: median 2.75
    tr = np.stack([g.normal(size=Pm), g.normal(size=Pm), tz], 1)
    tp = np.stack([g.normal(size=Pm), g.normal(size=Pm), pz], 1)
    tr[count:] = np.nan
    tp[count:] = np.nan
    if name == "count_above_max":
        count = Pm + 7
        pimg[len(ids):] = g.integers(0, images, Pm - len(ids))
        tr[len(ids):, 2] = tz[len(ids):]
        tp[len(ids):, 2] = pz[len(ids):]
        tr[len(ids):, :2] = tp[len(ids):, :2] = 0.0
    elif name == "count_negative":
        count = -1
    return images, Pm, count, pimg, verts.astype(np.float32), tp.astype(np.float32), tr.astype(np.float32)


def _pose_ref(images, count, pimg, verts, tp, tr, nf, ar, side, unstable=False, upper_median=False,
              second_centre=False):
    P = len(pimg)
    n = min(max(count, 0), P)
    vpi = 1 + 3 * nf + (3 if side else 0)
    rank = -np.ones(P, np.int64)
    nonempty = np.zeros(images, np.int64)
    pose = np.tile(np.eye(3, 4), (images, vpi, 1, 1))
    for b in range(images):
        ids = np.asarray([p for p in range(n) if pimg[p] == b], np.int64)
        if len(ids) == 0:
            continue
        nonempty[b] = 1
        order = ids
        if tr is not None:
            key = tr[ids, 2].astype(np.float64)
            order = ids[np.lexsort((-ids, key))] if unstable else ids[np.argsort(key, kind="stable")]
        rank[order] = np.arange(len(order))
        if nf:
            c = order[1] if second_centre and len(order) > 1 else order[0]
            pose[b, 1:1 + 3 * nf] = rv.orbit_poses(verts[c], nf, ar)
        if side:
            z = np.sort(tp[ids, 2].astype(np.float64))
            pose[b, 1 + 3 * nf:] = rv.side_poses([z[len(z) // 2]] if upper_median else z)
    return rank, nonempty, pose


def _run_pose_kernel(images, Pm, count, pimg, verts, tp, tr, nf, ar, side):
    from multihmr_b200 import _lib

    vpi = 1 + 3 * nf + (3 if side else 0)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    pose = torch.full((images, vpi, 3, 4), 7.0, device=DEV)
    nonempty = torch.full((images,), 9, dtype=torch.uint8, device=DEV)
    rank = torch.full((Pm,), 12345, dtype=torch.int32, device=DEV)
    keep = [d(np.array([count], np.int32)), d(pimg), d(verts), d(tp), None if tr is None else d(tr)]
    pa = _lib.struct("mhmr_render_pose_args", images=images, max_persons=Pm, num_verts=verts.shape[1],
                     count=keep[0], person_image=keep[1], verts=keep[2], transl_pelvis=keep[3], transl=keep[4],
                     n_frames=nf, angle_range=ar, side=int(side), pose=pose, nonempty=nonempty, rank=rank)
    _lib.call("mhmr_render_view_poses", pa, _lib.stream(torch.device(DEV)))
    torch.cuda.synchronize()
    return rank.cpu().numpy(), nonempty.cpu().numpy(), pose.double().cpu().numpy()


@pytest.mark.parametrize("closest_first", [False, True])
@pytest.mark.parametrize("name", ["4img_interleaved_4096", "even_odd_ties", "count_above_max", "count_negative"])
def test_pose_kernel_against_numpy(name, closest_first):
    """Ranks and nonempty exactly; poses within one rounding of the fp64 result to fp32.  Bound: the kernel and numpy
    both work in fp64 and differ only in the order of the V-term vertex mean and in a few ulps of cos / sin / sqrt,
    which is below 2^-40 (1 + S) absolute, S = the largest |vertex coordinate| or 3 |median pelvis z| (|c| and the
    eyes 2.2 zt of lookAt are below it); rounding to fp32 then adds at most 2^-24 |pose|."""
    images, Pm, count, pimg, verts, tp, tr, = _pose_case(name)
    tr = tr if closest_first else None
    nf, ar = 3, 40.0
    rank, nonempty, pose = _run_pose_kernel(images, Pm, count, pimg, verts, tp, tr, nf, ar, True)
    rrank, rnon, rpose = _pose_ref(images, count, pimg, verts, tp, tr, nf, ar, True)
    assert np.array_equal(rank, rrank), f"ranks differ at {np.nonzero(rank != rrank)[0][:8].tolist()}"
    assert np.array_equal(nonempty, rnon)
    n = min(max(count, 0), Pm)
    zt = np.abs(tp[:n, 2]).max(initial=0.0) if n else 0.0
    S = max(float(np.abs(verts[:n]).max(initial=0.0)), 3.0 * float(zt))
    tol = U32 * np.abs(rpose) + 2.0 ** -40 * (1.0 + S)
    ratio = (np.abs(pose - rpose) / tol).max()
    msg = [f"{name} closest_first={closest_first}: worst pose err/tol {ratio:.3f}"]
    assert ratio <= 1.0
    if name == "even_odd_ties":
        for what, kw in (("ranks not stable", dict(unstable=True)), ("upper median", dict(upper_median=True)),
                         ("second person as centre", dict(second_centre=True))):
            if what == "ranks not stable" and tr is None:
                continue
            wr, _, wp = _pose_ref(images, count, pimg, verts, tp, tr, nf, ar, True, **kw)
            if what == "ranks not stable":
                msg.append(f"{what}: {int((wr != rank).sum())} ranks differ")
                assert (wr != rank).any()
            else:
                r2 = (np.abs(pose - wp) / tol).max()
                msg.append(f"{what}: err/tol {r2:.3g}")
                assert r2 > 1.0
    print("; ".join(msg))
