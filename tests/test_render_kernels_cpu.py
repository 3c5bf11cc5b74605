"""CPU companions of test_render_kernels_gpu.py: the exact scenes are exact by construction (fp32 in the kernels'
fmaf order, fp64 and exact rationals agree on every edge plane and edge value), the ownership references the GPU test
uses are right and their planted mistakes are visible, the watertightness scenes would catch per-triangle edge
planes, and the queue-overflow call really overflows the queue while each of its views does not."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import render_ref

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import render_kernels_util as ru  # noqa: E402

EXACT = ru.exact_scenes()
WATERTIGHT = ru.watertight_scenes()


@pytest.mark.parametrize("name", list(EXACT))
def test_exact_scene_is_exact_in_fp32_fp64_and_rationals(name):
    s = EXACT[name]
    k32, k64, kq = ru.edge_values_three_ways(s)
    # the canonical planes (p_hi - p_lo) x p_lo of tri_setup, the oracle's p_j x p_i and the exact value: equal
    assert np.array_equal(k32["planes"], k64["planes"])
    assert all((kq["planes"] == k64["planes"]).ravel())
    # every edge value at every pixel of every box, edges and vertices included: equal, with both signs and zeros
    assert np.array_equal(k32["e"], k64["e"])
    assert all((kq["e"] == k64["e"]).ravel())
    zero = (k64["e"] == 0).any(1)
    inside = (k64["e"] >= 0).all(1) & (k64["e"].sum(1) > 0)
    assert zero.sum() > 0.05 * len(zero), "the scene must put many pixel centres on edges"
    # tri_cover's depth at every covered pixel is the plane's z exactly
    t, _, _ = ru.box_pixels(s["verts"], s["K"], s["H"], s["W"])
    assert np.array_equal(k32["z"][inside], s["z"][t][inside].astype(np.float64))
    print(f"{name}: {len(zero)} box pixels, {int(zero.sum())} on an edge or vertex, all exact")


@pytest.mark.parametrize("name", list(EXACT))
def test_owner_reference_matches_oracle_and_planted_rules_differ(name):
    s = EXACT[name]
    ref = render_ref.rasterize(s["verts"], [[0, 1, 2]], s["K"], s["H"], s["W"],
                               colors=np.full((len(s["verts"]), 3), 0.5))
    own, cover = ru.owner_map(s["verts"], s["K"], s["H"], s["W"])
    assert np.array_equal(own, ref["index"])
    for outline in s.get("outlines", []):
        inside = ru.inside_outline(s["H"], s["W"], outline)
        assert (cover[inside] == 1).all(), "a single plane: every pixel inside the outline exactly once"
    for rule in ("bottom_right", "both"):
        other, cov2 = ru.owner_map(s["verts"], s["K"], s["H"], s["W"], rule)
        diff = int((other != ref["index"]).sum())
        print(f"{name}: tie rule {rule} differs from the top-left oracle at {diff} pixels")
        assert diff >= 10


def test_exact_scenes_reach_both_sides_of_the_queue_threshold():
    seen = set()
    for name, s in EXACT.items():
        a = ru.box_areas(s["verts"], s["K"], s["H"], s["W"])
        seen |= set(a.tolist())
    assert {255, 256} <= seen and {258, 272, 1849} <= seen
    assert max(a for a in seen if a <= ru.BIG_AREA) == 256 and min(a for a in seen if a > ru.BIG_AREA) == 258


@pytest.mark.parametrize("name", list(WATERTIGHT))
def test_per_triangle_edge_planes_open_cracks(name):
    """The scenes put pixel centres exactly on interior edges while the edge values there are rounded.  Evaluating each
    edge once, lower vertex id first (as tri_setup does), leaves no crack along an edge even in plain float32;
    evaluating each triangle's own planes (p_j - p_i) x p_i opens some, so the GPU watertightness test would catch
    that regression.  Pixel centres on a vertex are counted apart: there the rounded planes of the fan no longer meet
    in one ray, and even canonical edges may leave the centre to no triangle."""
    s = WATERTIGHT[name]
    v, f, K, H, W = s["verts"][0], s["faces"], s["K"], s["H"], s["W"]
    ref = render_ref.rasterize(s["verts"], f, K, H, W, colors=[[0.5, 0.5, 0.5]])
    must = (ref["depth"] > 0) & (ru.silhouette_distance(v, f, K, H, W) > 1e-3)
    on_vertex = ru.vertex_distance(v, K, H, W) <= 1e-3
    canon = ru.per_triangle_coverage_f32(v, f, K, H, W, canonical=True)
    own = ru.per_triangle_coverage_f32(v, f, K, H, W, canonical=False)
    cracks = int((must & ~own & ~on_vertex).sum())
    print(f"{name}: {int(must.sum())} interior pixels, {int((ref['edge_dist'] < 1e-3).sum())} on an edge; "
          f"per-triangle planes leave {cracks} uncovered ({int((must & ~own & on_vertex).sum())} more on vertices), "
          f"canonical {int((must & ~canon & ~on_vertex).sum())} ({int((must & ~canon & on_vertex).sum())} on vertices)")
    assert (must & ~canon & ~on_vertex).sum() == 0
    assert cracks >= 5


def test_sliver_call_overflows_the_queue_and_its_views_do_not():
    v, f, K, pose = ru.sliver_scene()
    H, W = ru.SLIVER["H"], ru.SLIVER["W"]
    counts, amin, amax = ru.queued_counts(v, f, K, pose, H, W)
    print(f"queued per view {counts}, total {sum(counts)}; boxes {amin}..{amax} px")
    # every (view, person, face) is front-facing and its box lies well over the threshold (fp32 cannot move it across)
    assert all(c == ru.SLIVER["faces"] * ru.SLIVER["persons"] for c in counts) and amin >= ru.BIG_AREA + 40
    assert max(counts) < ru.QUEUE_CAP < sum(counts)
