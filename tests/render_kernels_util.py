"""Scene builders and exact references for the renderer's kernel tests (test_render_kernels_cpu.py / _gpu.py).

Exact scenes: triangles whose vertices project onto pixel centres of a plane z = const, with fx = fy a power of two and
cx, cy at half-integers, so that every coordinate, edge plane and edge value the kernels compute in fp32 is a small
dyadic rational, exact in fp32, fp64 and `fractions.Fraction` alike (test_render_kernels_cpu proves it scene by
scene).  Each triangle is its own person of `Renderer([[0, 1, 2]])` (3 vertices, no face bits), so the `index` output
is the owning triangle and ownership can be compared at every pixel, edges and vertices included.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np
import torch

from oracle import render_ref

# ----------------------------------------------------------------------------------------------------- exact scenes


def orient_front(tri: np.ndarray) -> np.ndarray:
    """Winds screen triangles [T,3,2] (u right, v down) counter-clockwise on screen, GL's front face."""
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    cr = (b[:, 0] - a[:, 0]) * (c[:, 1] - a[:, 1]) - (b[:, 1] - a[:, 1]) * (c[:, 0] - a[:, 0])
    assert (cr != 0).all(), "degenerate screen triangle"
    out = tri.copy()
    back = cr > 0
    out[back] = out[back][:, [0, 2, 1]]
    return out


def grid_tris(u0, v0, cols, rows):
    """A grid of cells with the given column widths and row heights (pixels) from the pixel centre (u0, v0), each cell
    split along its main diagonal or its anti-diagonal in a checkerboard: horizontal, vertical and both diagonal
    edges.  Returns [T,3,2] screen triangles and the outline (umin, vmin, umax, vmax)."""
    us = u0 + np.concatenate([[0], np.cumsum(cols)])
    vs = v0 + np.concatenate([[0], np.cumsum(rows)])
    tris = []
    for j in range(len(rows)):
        for i in range(len(cols)):
            a, b = (us[i], vs[j]), (us[i + 1], vs[j])
            c, d = (us[i + 1], vs[j + 1]), (us[i], vs[j + 1])
            tris += [[a, b, c], [a, c, d]] if (i + j) % 2 == 0 else [[a, b, d], [b, c, d]]
    return orient_front(np.asarray(tris, np.float64)), (us[0], vs[0], us[-1], vs[-1])


def square_ring(r, step):
    """Integer offsets on the boundary of the square of half-size r, `step` apart, in angular order."""
    pts = [(r, k) for k in range(-r, r, step)] + [(k, r) for k in range(r, -r, -step)]
    pts += [(-r, k) for k in range(r, -r, -step)] + [(k, -r) for k in range(-r, r, step)]
    return pts


def fan_tris(cu, cv, ring):
    n = len(ring)
    tris = [[(cu, cv), (cu + ring[k][0], cv + ring[k][1]), (cu + ring[(k + 1) % n][0], cv + ring[(k + 1) % n][1])]
            for k in range(n)]
    return orient_front(np.asarray(tris, np.float64))


def lift(tris_px, z, fx, fy, cx, cy):
    """Camera-space float32 vertices [T,3,3] of screen triangles on the planes z (scalar or [T])."""
    z = np.broadcast_to(np.asarray(z, np.float64), (len(tris_px),))[:, None]
    x = (tris_px[..., 0] - cx) * z / fx
    y = (tris_px[..., 1] - cy) * z / fy
    v = np.stack([x, y, np.broadcast_to(z, x.shape)], -1)
    assert np.array_equal(v.astype(np.float32).astype(np.float64), v), "not exact in fp32"
    return v.astype(np.float32)


def _exact_scene(W, H, parts, f=32.0):
    """parts: [(screen triangles, z)].  Camera fx = fy = f, (cx, cy) at the pixel centre nearest the middle."""
    cx, cy = W // 2 + 0.5, H // 2 + 0.5
    tris = np.concatenate([p for p, _ in parts])
    z = np.concatenate([np.full(len(p), zz) for p, zz in parts])
    K = np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float64)
    return {"verts": lift(tris, z, f, f, cx, cy), "z": z.astype(np.float32), "K": K, "H": H, "W": W, "px": tris}


def exact_scenes() -> dict:
    """name -> {'verts' [T,3,3] fp32, 'z' [T], 'K', 'H', 'W', 'px' screen triangles, 'outlines' or 'fans'}."""
    out = {}
    # 3-px cells spanning the image: the outline runs along the first and last pixel rows and columns
    g, box = grid_tris(0.5, 0.5, [3] * 21, [3] * 15)
    out["grid_3px_64x46"] = dict(_exact_scene(64, 46, [(g, 2.0)]), outlines=[box])
    # 1-px cells: every pixel centre is a vertex
    g, box = grid_tris(0.5, 0.5, [1] * 23, [1] * 19)
    out["grid_1px_24x20"] = dict(_exact_scene(24, 20, [(g, 2.0)]), outlines=[box])
    # fans of 8 and 16 triangles on two planes (the z = 4 fan partly hidden), and one around the last pixel centre
    fa = fan_tris(15.5, 19.5, square_ring(8, 8))
    fb = fan_tris(30.5, 20.5, square_ring(8, 4))
    fc = fan_tris(47.5, 39.5, square_ring(6, 3))
    fd = fan_tris(0.5, 0.5, square_ring(4, 2))
    s = _exact_scene(48, 40, [(fa, 2.0), (fb, 4.0), (fc, 2.0), (fd, 4.0)])
    out["fans_48x40"] = dict(s, fans=[((15.5, 19.5), 8), ((30.5, 20.5), 8), ((47.5, 39.5), 6), ((0.5, 0.5), 4)])
    # bounding boxes (x1 - x0 + 3) x (y1 - y0 + 3) around the queue threshold of 256 px: 13 x 13 cells give 256 (drawn
    # by the per-face threads), 14 x 13 give 272 (queued); 12 x 14 give 255, 3 x 40 give 258 (257 is prime: no box
    # of a non-degenerate on-screen triangle has it); 40 x 40 give 1849
    g, box = grid_tris(2.5, 2.5, [13, 14] * 3, [13] * 3 + [14])
    out["grid_box256_272"] = dict(_exact_scene(88, 60, [(g, 2.0)]), outlines=[box])
    g, box = grid_tris(2.5, 2.5, [12, 3] * 3, [14, 40])
    out["grid_box255_258"] = dict(_exact_scene(50, 60, [(g, 2.0)]), outlines=[box])
    g, box = grid_tris(2.5, 2.5, [40] * 3, [40] * 2)
    out["grid_box1849"] = dict(_exact_scene(126, 86, [(g, 4.0)], f=64.0), outlines=[box])
    return out


def box_areas(verts, K, H, W) -> np.ndarray:
    """The kernels' bounding-box pixel counts of front-facing triangles [T,3,3], from the oracle's `_bbox`."""
    x0, x1, y0, y1 = render_ref._bbox(torch.as_tensor(np.asarray(verts), dtype=torch.float64),
                                      torch.as_tensor(K), W, H)
    return ((x1 - x0 + 1).clamp_min(0) * (y1 - y0 + 1).clamp_min(0)).numpy()


def inside_outline(H, W, box):
    """Pixel centres strictly inside the rectangle (umin, vmin, umax, vmax)."""
    yy, xx = np.mgrid[0:H, 0:W] + 0.5
    return (xx > box[0]) & (xx < box[2]) & (yy > box[1]) & (yy < box[3])


def inside_fan(H, W, centre, r):
    yy, xx = np.mgrid[0:H, 0:W] + 0.5
    return (np.abs(xx - centre[0]) < r) & (np.abs(yy - centre[1]) < r)


def owner_map(verts, K, H, W, rule="top_left"):
    """Exact fp64 ownership of one-triangle persons on planes: index of the nearest covering triangle (ties to the
    lower index), -1 where none, and the number of triangles covering each pixel.  rule: 'top_left' (the kernels'),
    'bottom_right' (the tie rule flipped) or 'both' (an edge's pixels belong to both sides)."""
    v = np.asarray(verts, np.float64)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    yy, xx = np.mgrid[0:H, 0:W]
    dx, dy = (xx + 0.5 - cx) / fx, (yy + 0.5 - cy) / fy
    best_z = np.full((H, W), np.inf)
    idx = np.full((H, W), -1, np.int32)
    cover = np.zeros((H, W), np.int32)
    for t in range(len(v)):
        p = v[t]
        ok = np.ones((H, W), bool)
        for k in range(3):
            m = np.cross(p[(k + 2) % 3], p[(k + 1) % 3])
            e = m[0] * dx + m[1] * dy + m[2]
            if rule == "top_left":
                own = m[0] > 0 or (m[0] == 0 and m[1] > 0)
            elif rule == "bottom_right":
                own = m[0] < 0 or (m[0] == 0 and m[1] < 0)
            else:
                own = True
            ok &= (e > 0) | ((e == 0) & own)
        z = p[0, 2]
        cover += ok
        win = ok & (z < best_z)
        best_z[win] = z
        idx[win] = t
    return idx, cover


# --- the kernels' fp32 arithmetic, emulated exactly enough to prove exactness ---------------------------------------

def _f32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def _fmaf(a, b, c):
    """fmaf on fp32 values held in fp64: the product is exact in fp64; when the fp64 sum is exact too, rounding it
    to fp32 is fmaf.  (If it is not, the result differs from the exact value and the exactness check fails.)"""
    return _f32(a * b + c)


def _cross_fmaf(a, b):
    return np.stack([_fmaf(a[..., 1], b[..., 2], -_f32(a[..., 2] * b[..., 1])),
                     _fmaf(a[..., 2], b[..., 0], -_f32(a[..., 0] * b[..., 2])),
                     _fmaf(a[..., 0], b[..., 1], -_f32(a[..., 1] * b[..., 0]))], -1)


def kernel_planes_f32(verts):
    """tri_setup's canonical edge planes for faces [0, 1, 2]: (p_hi - p_lo) x p_lo, lower vertex id first, negated
    when the edge runs the other way.  [T,3 edges,3]."""
    p = np.asarray(verts, np.float64)
    ms = []
    for k in range(3):
        i, j = (k + 1) % 3, (k + 2) % 3
        lo, hi = (p[:, i], p[:, j]) if i < j else (p[:, j], p[:, i])
        cm = _cross_fmaf(_f32(hi - lo), lo)
        ms.append(cm if i < j else -cm)
    return np.stack(ms, 1)


def box_pixels(verts, K, H, W):
    """(triangle, x, y) of every pixel in every front-facing triangle's box."""
    x0, x1, y0, y1 = render_ref._bbox(torch.as_tensor(np.asarray(verts), dtype=torch.float64), torch.as_tensor(K),
                                      W, H)
    tt, xs, ys = [], [], []
    for t in range(len(verts)):
        yy, xx = np.mgrid[int(y0[t]):int(y1[t]) + 1, int(x0[t]):int(x1[t]) + 1]
        tt.append(np.full(xx.size, t))
        xs.append(xx.ravel())
        ys.append(yy.ravel())
    return np.concatenate(tt), np.concatenate(xs), np.concatenate(ys)


def edge_values_three_ways(scene):
    """Edge planes and edge values at every box pixel of an exact scene, evaluated (1) as the kernels do in fp32
    (fmaf order, ray by __fdiv_rn), (2) as the fp64 oracle does and (3) in exact rationals.  Returns dicts
    {'planes': [T,3,3], 'e': [N,3], 'z': [N]} (the depth of (1) at the covered pixels is also returned)."""
    v, K, H, W = scene["verts"], scene["K"], scene["H"], scene["W"]
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    t, xs, ys = box_pixels(v, K, H, W)
    # (1) fp32 as in tri_setup / tri_cover / ray_x
    m32 = kernel_planes_f32(v)
    dx32 = _f32(_f32(_f32(xs + 0.5) - _f32(cx)) / _f32(fx))
    dy32 = _f32(_f32(_f32(ys + 0.5) - _f32(cy)) / _f32(fy))
    e32 = np.stack([_fmaf(m32[t, k, 0], dx32, _fmaf(m32[t, k, 1], dy32, m32[t, k, 2])) for k in range(3)], 1)
    pz = np.asarray(v, np.float64)[t, :, 2]
    s32 = _f32(_f32(e32[:, 0] + e32[:, 1]) + e32[:, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        z32 = _f32(_fmaf(e32[:, 0], pz[:, 0], _fmaf(e32[:, 1], pz[:, 1], _f32(e32[:, 2] * pz[:, 2]))) / s32)
    # (2) fp64 as in render_ref.rasterize
    p64 = torch.as_tensor(np.asarray(v, np.float64))
    m64 = render_ref._edge_planes(p64).numpy()
    dx64, dy64 = (xs + 0.5 - cx) / fx, (ys + 0.5 - cy) / fy
    e64 = m64[t, :, 0] * dx64[:, None] + m64[t, :, 1] * dy64[:, None] + m64[t, :, 2]
    # (3) exact
    F = np.vectorize(Fraction, otypes=[object])
    pf = F(np.asarray(v, np.float64))
    mq = np.stack([np.cross(pf[:, (k + 2) % 3], pf[:, (k + 1) % 3]) for k in range(3)], 1)
    dxq = (F(xs.astype(np.float64)) + Fraction(1, 2) - Fraction(cx)) / Fraction(fx)
    dyq = (F(ys.astype(np.float64)) + Fraction(1, 2) - Fraction(cy)) / Fraction(fy)
    eq = np.stack([mq[t, k, 0] * dxq + mq[t, k, 1] * dyq + mq[t, k, 2] for k in range(3)], 1)
    return ({"planes": m32, "e": e32, "z": z32, "s": s32}, {"planes": m64, "e": e64}, {"planes": mq, "e": eq})


# ----------------------------------------------------------------------------------- watertightness (inexact) scenes

def _on_centre_rays(uv, z, K):
    """Vertices on the rays of the pixel centres uv [N,2] at depths z rounded to 12 significant bits: with fx, fy
    powers of two and cx, cy half-integers they are exact in fp32 and lie exactly on those rays, while the products of
    the edge planes need more than 24 bits, so the kernels' fp32 edge values are rounded."""
    zq = np.ldexp(np.round(np.ldexp(z, 10)), -10)
    assert (zq >= 1).all() and (zq < 4).all()
    v = np.stack([(uv[:, 0] - K[0, 2]) * zq / K[0, 0], (uv[:, 1] - K[1, 2]) * zq / K[1, 1], zq], 1)
    assert np.array_equal(v.astype(np.float32).astype(np.float64), v)
    return v.astype(np.float32)


def watertight_scenes() -> dict:
    """name -> {'verts' [1,V,3] fp32, 'faces', 'K', 'H', 'W'}: meshes whose fp32 vertices lie exactly on pixel-centre
    rays at varying depths, so that interior edges pass exactly through pixel centres while every edge value the
    kernels compute there is rounded."""
    out = {}
    H, W = 64, 80
    K = np.array([[32.0, 0, 40.5], [0, 32.0, 30.5], [0, 0, 1]])
    ring = square_ring(12, 3)
    for name, apex_z, rim_z in (("pyramid_convex", 1.7, 2.3), ("pyramid_concave", 2.9, 2.1)):
        ap = np.array([40.5, 30.5])
        uv = np.asarray([ap] + [ap + np.asarray(o, np.float64) for o in ring])
        z = np.array([apex_z] + [rim_z + 0.13 * math.sin(1.7 * k) for k in range(len(ring))])
        n = len(ring)
        f = np.array([[0, 1 + k, 1 + (k + 1) % n] for k in range(n)])
        scr = uv[f]
        back = ((scr[:, 1, 0] - scr[:, 0, 0]) * (scr[:, 2, 1] - scr[:, 0, 1])
                - (scr[:, 1, 1] - scr[:, 0, 1]) * (scr[:, 2, 0] - scr[:, 0, 0])) > 0
        f[back] = f[back][:, [0, 2, 1]]
        out[name] = {"verts": _on_centre_rays(uv, z, K)[None], "faces": f, "K": K, "H": H, "W": W}
    # a blob person turned about two axes, every vertex moved along its depth onto the nearest pixel-centre ray
    from multihmr_b200 import synth

    verts, faces = synth.make_blob_people([(0.0, 0.0, 0.0)], seed=11, n_lat=10, n_lon=16)
    a, b = 0.7, 0.35
    Ry = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])
    Rz = np.array([[math.cos(b), -math.sin(b), 0], [math.sin(b), math.cos(b), 0], [0, 0, 1]])
    v = verts[0].astype(np.float64) @ (Rz @ Ry).T + [0.05, 0.02, 2.4]
    Kb = np.array([[128.0, 0, 80.5], [0, 128.0, 100.5], [0, 0, 1]])
    uv = np.floor(np.stack([Kb[0, 0] * v[:, 0] / v[:, 2] + Kb[0, 2], Kb[1, 1] * v[:, 1] / v[:, 2] + Kb[1, 2]], 1)) + 0.5
    out["blob_rotated_on_centres"] = {"verts": _on_centre_rays(uv, v[:, 2], Kb)[None], "faces": faces, "K": Kb,
                                      "H": 200, "W": 160}
    return out


def vertex_distance(verts, K, H, W):
    """Per pixel, the screen distance (px) of its centre to the nearest projected vertex."""
    v = np.asarray(verts, np.float64)
    u = K[0, 0] * v[:, 0] / v[:, 2] + K[0, 2]
    w = K[1, 1] * v[:, 1] / v[:, 2] + K[1, 2]
    d = np.full((H, W), np.inf)
    ix, iy = np.floor(u).astype(int), np.floor(w).astype(int)
    ok = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
    np.minimum.at(d, (iy[ok], ix[ok]), np.hypot(u[ok] - ix[ok] - 0.5, w[ok] - iy[ok] - 0.5))
    return d


def silhouette_distance(verts, faces, K, H, W):
    """Per pixel, the screen distance (px) of its centre to the nearest silhouette edge: an edge with exactly one
    front-facing neighbour (fp64 on the given vertices)."""
    v = np.asarray(verts, np.float64)
    p = v[faces]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    front = (n * p[:, 0]).sum(-1) < 0
    cnt = {}
    for f in faces[front]:
        for k in range(3):
            e = tuple(sorted((int(f[k]), int(f[(k + 1) % 3]))))
            cnt[e] = cnt.get(e, 0) + 1
    sil = np.array([e for e, c in cnt.items() if c == 1], np.int64).reshape(-1, 2)
    u = K[0, 0] * v[:, 0] / v[:, 2] + K[0, 2]
    w = K[1, 1] * v[:, 1] / v[:, 2] + K[1, 2]
    yy, xx = np.mgrid[0:H, 0:W] + 0.5
    d = np.full((H, W), np.inf)
    for a, b in sil:
        ax, ay, bx, by = u[a], w[a], u[b], w[b]
        ex, ey = bx - ax, by - ay
        L2 = ex * ex + ey * ey
        s = np.clip(((xx - ax) * ex + (yy - ay) * ey) / max(L2, 1e-300), 0.0, 1.0)
        d = np.minimum(d, np.hypot(xx - ax - s * ex, yy - ay - s * ey))
    return d


def per_triangle_coverage_f32(verts, faces, K, H, W, canonical: bool):
    """Coverage of the pixel centres in torch float32 with per-triangle edge planes (p_j - p_i) x p_i in each
    triangle's own vertex order, or (canonical=True) with one plane per edge, lower vertex id first, as tri_setup
    does.  Top-left rule, back faces culled.  Returns a bool [H,W]."""
    v = torch.as_tensor(np.asarray(verts, np.float32))
    f = torch.as_tensor(np.asarray(faces, np.int64))
    p = v[f]
    n = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=-1)
    keep = (n * p[:, 0]).sum(-1) < 0
    p, f = p[keep], f[keep]
    ms = []
    for k in range(3):
        i, j = (k + 1) % 3, (k + 2) % 3
        if canonical:
            fwd = (f[:, i] < f[:, j])[:, None]
            lo = torch.where(fwd, p[:, i], p[:, j])
            hi = torch.where(fwd, p[:, j], p[:, i])
            cm = torch.cross(hi - lo, lo, dim=-1)
            ms.append(torch.where(fwd, cm, -cm))
        else:
            ms.append(torch.cross(p[:, j] - p[:, i], p[:, i], dim=-1))
    m = torch.stack(ms, 1)                                              # [T,3,3]
    fx, fy, cx, cy = (torch.tensor(float(K[0, 0])), torch.tensor(float(K[1, 1])), torch.tensor(float(K[0, 2])),
                      torch.tensor(float(K[1, 2])))
    dx = (torch.arange(W, dtype=torch.float32) + 0.5 - cx) / fx
    dy = (torch.arange(H, dtype=torch.float32) + 0.5 - cy) / fy
    cov = torch.zeros(H, W, dtype=torch.bool)
    for t in range(m.shape[0]):
        ok = torch.ones(H, W, dtype=torch.bool)
        for k in range(3):
            e = m[t, k, 0] * dx[None, :] + (m[t, k, 1] * dy[:, None] + m[t, k, 2])
            own = bool(m[t, k, 0] > 0) or (bool(m[t, k, 0] == 0) and bool(m[t, k, 1] > 0))
            ok &= (e > 0) | ((e == 0) & own)
        cov |= ok
    return cov.numpy()


# --------------------------------------------------------------------------------- production-size scenes (D)

def bench_people(n, W, H, f, seed, K=None):
    """tools/bench_render.py's people: n blob people of 18 432 faces (32 x 48 segments) between 3 and 8 m, spread
    over the image of intrinsics K (default f, centred principal point)."""
    from multihmr_b200 import synth

    fx, fy, cx, cy = (f, f, W / 2, H / 2) if K is None else (K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    g = np.random.default_rng(seed)
    z = g.uniform(3.0, 8.0, n)
    x = (g.uniform(0.05, 0.95, n) * W - cx) * z / fx
    y = (g.uniform(0.4, 0.6, n) * H - cy) * z / fy
    return synth.make_blob_people(np.stack([x, y, z], 1), seed=seed, n_lat=32, n_lon=48)


def production_scenes() -> dict:
    """The workloads of tools/bench_render.py, rebuilt from its parameters (seed = len(name)), plus a camera with
    fx != fy and the principal point outside the image.  name -> {'verts', 'faces', 'K' [views,3,3], 'pose'
    [views,3,4] or None, 'H', 'W'}."""
    out = {}
    for name, (W, H, n, views) in {"896x896_4p": (896, 896, 4, 1), "1920x1080_20p": (1920, 1080, 20, 1),
                                   "rotate20_1920x1080_3p": (1920, 1080, 3, 20)}.items():
        f = max(W, H) / (2 * np.tan(np.radians(30)))
        verts, faces = bench_people(n, W, H, f, seed=len(name))
        K = np.tile(np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]]), (views, 1, 1))
        pose = None
        if views > 1:
            c = verts[0].mean(0)
            pose = np.zeros((views, 3, 4))
            for i, a in enumerate(np.deg2rad(np.linspace(0, 60, views))):
                R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
                pose[i, :, :3], pose[i, :, 3] = R, c - R @ c
        out[name] = dict(verts=verts, faces=faces, K=K, pose=pose, W=W, H=H)
    W, H = 1920, 1080
    Kp = np.array([[1210.0, 0, -37.3], [0, 1040.5, 1105.2], [0, 0, 1]])  # principal point left of and below the image
    verts, faces = bench_people(6, W, H, None, seed=6, K=Kp)
    out["offcentre_1920x1080_6p"] = dict(verts=verts, faces=faces, K=Kp[None], pose=None, W=W, H=H)
    return out


def demo_views_scene():
    """tools/bench_render.py's `demo_orbit_1920x1080_3p` (seed 23): verts, faces, K [3,3], H, W."""
    W, H = 1920, 1080
    f = max(W, H) / (2 * np.tan(np.radians(30)))
    verts, faces = bench_people(3, W, H, f, seed=len("demo_orbit_1920x1080_3p"))
    return verts, faces, np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]]), H, W


def view_errors(gpu: dict, gpu_alpha1: np.ndarray, ref: dict):
    """(flagged fraction, worst relative depth error off the flagged pixels, worst shaded-colour difference on the
    interior pixels), the quantities check_view bounds."""
    flag = (ref["edge_dist"] < 1e-3) | (ref["depth_gap"] < 1e-5)
    fg = ~flag & (ref["depth"] > 0)
    rel = np.abs(gpu["depth"][fg].astype(np.float64) - ref["depth"][fg]) / ref["depth"][fg]
    same = (gpu["depth"] > 0) == (ref["depth"] > 0)
    m = torch.from_numpy(~(same & (ref["depth"] > 0) & ~flag)).float()[None, None]
    interior = ~(torch.nn.functional.max_pool2d(m, 3, 1, 1)[0, 0].numpy() > 0)
    interior[[0, -1], :] = False
    interior[:, [0, -1]] = False
    d = np.abs(gpu_alpha1.astype(np.int16) - ref["rgb"].astype(np.int16)).max(-1)
    return float(flag.mean()), float(rel.max(initial=0.0)), int(d[interior].max(initial=0))


def depth_bound(l_verts, l_faces, K, ref, R=None, t=None, c=8.0):
    """Per foreground pixel, a bound on the relative error of the kernels' fp32 depth at the oracle's winning face:
    z = sum(e_k z_k) / s with e_k = m_k . d, s = sum(e_k).  Each e_k carries an absolute rounding error of a few u
    |m_k|_1 |d|_inf (the canonical plane and its dot product), which moves z by sum(de_k (z_k - z)) / s; so
    |dz| / z <= c u sum_k(|m_k|_1 |d|_inf |z_k - z|) / (|s| z) + c u.  It exceeds 1e-5 only on faces seen almost
    edge-on, where s is small.  0 on the background."""
    H, W = ref["depth"].shape
    out = np.zeros(H * W)
    idx, face = ref["index"].ravel(), ref["face"].ravel()
    dt = torch.float64
    Rm = torch.eye(3, dtype=dt) if R is None else torch.as_tensor(np.asarray(R), dtype=dt)
    tv = torch.zeros(3, dtype=dt) if t is None else torch.as_tensor(np.asarray(t), dtype=dt).reshape(3)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    for i in np.unique(idx[idx >= 0]):
        pix = np.nonzero(idx == i)[0]
        v = torch.as_tensor(np.asarray(l_verts[i]), dtype=dt) @ Rm.T + tv
        p = v[torch.as_tensor(np.asarray(l_faces[i])[face[pix]])]                     # [N,3,3]
        m = render_ref._edge_planes(p)
        d = torch.stack([torch.as_tensor((pix % W + 0.5 - cx) / fx), torch.as_tensor((pix // W + 0.5 - cy) / fy),
                         torch.ones(len(pix), dtype=dt)], 1)
        e = (m * d[:, None]).sum(-1)
        s_ = e.sum(1)
        z = (e * p[..., 2]).sum(1) / s_
        dinf = d.abs().amax(1, keepdim=True)
        k = (m.abs().sum(-1) * dinf * (p[..., 2] - z[:, None]).abs()).sum(1) / (s_.abs() * z)
        out[pix] = (c * 2.0 ** -24 * (k + 1.0)).numpy()
    return out.reshape(H, W)


def screen_space_depth(verts, faces, K, ref, R=None, t=None):
    """Depth at the oracle's winning face of every foreground pixel with screen-space (not perspective-correct)
    barycentrics: the plausible mistake the depth tolerance must catch.  [H,W], 0 on the background."""
    v = np.asarray(verts, np.float64)
    if R is not None:
        v = v @ np.asarray(R).T + np.asarray(t).reshape(3)
    H, W = ref["depth"].shape
    pix = np.nonzero(ref["index"].ravel() >= 0)[0]
    p = v[ref["index"].ravel()[pix][:, None], np.asarray(faces)[ref["face"].ravel()[pix]]]         # [N,3,3]
    u = K[0, 0] * p[..., 0] / p[..., 2] + K[0, 2]
    w = K[1, 1] * p[..., 1] / p[..., 2] + K[1, 2]
    x, y = pix % W + 0.5, pix // W + 0.5
    area = lambda ax, ay, bx, by, cx_, cy_: (bx - ax) * (cy_ - ay) - (by - ay) * (cx_ - ax)
    l0 = area(x, y, u[:, 1], w[:, 1], u[:, 2], w[:, 2])
    l1 = area(u[:, 0], w[:, 0], x, y, u[:, 2], w[:, 2])
    l2 = area(u[:, 0], w[:, 0], u[:, 1], w[:, 1], x, y)
    s = l0 + l1 + l2
    out = np.zeros(H * W)
    out[pix] = (l0 * p[:, 0, 2] + l1 * p[:, 1, 2] + l2 * p[:, 2, 2]) / s
    return out.reshape(H, W)


# ------------------------------------------------------------------------------------------ queue overflow (E)

QUEUE_CAP = 1 << 20
BIG_AREA = 256
SLIVER = dict(faces=2048, persons=64, views=9, H=480, W=640)


def sliver_scene():
    """64 persons of 2048 sliver faces (each face its own three vertices): long thin triangles 40-46 px wide and
    5-8 px tall on screen (boxes of 301-528 px, over the 256-px queue threshold), well inside a 640 x 480 image, at
    depths 2-3 m; 9 views that shift the camera by a few centimetres.  Returns verts [P,3F,3] fp32, faces, K [9,3,3],
    pose [9,3,4]."""
    Fn, P, B, H, W = (SLIVER[k] for k in ("faces", "persons", "views", "H", "W"))
    f, cx, cy = 500.0, W / 2 + 0.25, H / 2 - 0.35
    g = np.random.default_rng(2048)
    u0 = g.uniform(30, W - 90, (P, Fn))
    v0 = g.uniform(30, H - 40, (P, Fn))
    L = g.uniform(40, 46, (P, Fn))
    h = g.uniform(4.0, 6.0, (P, Fn))
    wd = g.uniform(0.6, 1.5, (P, Fn))
    scr = np.stack([np.stack([u0, v0], -1), np.stack([u0 + L, v0 + h], -1), np.stack([u0 + L, v0 + h + wd], -1)], 2)
    za, zb = g.uniform(2.0, 3.0, (2, P, Fn))
    z = np.stack([za, zb, zb], -1)                       # the short edge at one depth: no sliver is seen edge-on
    cam = np.stack([(scr[..., 0] - cx) * z / f, (scr[..., 1] - cy) * z / f, z], -1)   # [P,F,3,3]
    tri = orient_front(scr.reshape(-1, 3, 2))
    flip = ~np.all(tri == scr.reshape(-1, 3, 2), axis=(1, 2))
    cam = cam.reshape(-1, 3, 3)
    cam[flip] = cam[flip][:, [0, 2, 1]]
    verts = cam.reshape(P, 3 * Fn, 3).astype(np.float32)
    faces = np.arange(3 * Fn).reshape(Fn, 3)
    K = np.tile(np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]]), (B, 1, 1))
    pose = np.zeros((B, 3, 4))
    pose[:, :, :3] = np.eye(3)
    pose[:, 0, 3] = 0.004 * np.arange(B)
    pose[:, 1, 3] = -0.003 * np.arange(B)
    return verts, faces, K, pose


def queued_counts(verts, faces, K, pose, H, W):
    """Per view, the (person, face) pairs the raster kernel sends to the queue: front-facing, in front of the near
    plane, box over BIG_AREA px (fp64 on the fp32 vertices), and the smallest and largest such box."""
    counts, amin, amax = [], math.inf, 0
    v = torch.as_tensor(np.asarray(verts, np.float64))
    for b in range(len(K)):
        R, t = torch.as_tensor(pose[b, :, :3]), torch.as_tensor(pose[b, :, 3])
        p = (v @ R.T + t)[:, torch.as_tensor(faces)].reshape(-1, 3, 3)
        n = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=-1)
        keep = ((n * p[:, 0]).sum(-1) < 0) & (p[..., 2].amin(1) >= render_ref.ZNEAR)
        x0, x1, y0, y1 = render_ref._bbox(p[keep], torch.as_tensor(K[b]), W, H)
        area = ((x1 - x0 + 1) * (y1 - y0 + 1)).numpy()
        counts.append(int((area > BIG_AREA).sum()) if keep.all() else -1)
        amin, amax = min(amin, int(area.min())), max(amax, int(area.max()))
    return counts, amin, amax
