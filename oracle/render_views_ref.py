"""fp64 restatement of the demo's extra views on top of oracle/render_ref.py: meshes of several topologies in one
z-buffer (the persons plus the camera glyph's props), the reference's `lookAt` (utils/render.py:329-363), the
side-view poses of `render_side_views` (utils/render.py:407-448) and the orbit poses of `create_rotating_video`
(demo.py:160-241) expressed as camera poses.

Orbit: the reference rotates the vertices about c = the first person's vertex mean, x' = (x - c) R^T + c, with R a
rotation about y (or x) by angle_range i / (n_frames - 1) degrees.  The light sits at the camera, so this is the
camera pose [R | c - R c] applied to the unrotated vertices.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.render_ref import _BIG, ZFAR, ZNEAR, _bbox, _edge_planes, composite, shade, vertex_normals  # noqa: F401

CV2GL = np.diag([1.0, -1.0, -1.0, 1.0])


def look_at(eye, target):
    """utils/render.py:lookAt: up (0, -1, 0), v / (|v| + 1e-13), then OPENCV_TO_OPENGL @ view; returns 4x4."""
    def normalize(v):
        n = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) + 1e-13
        return [v[0] / n, v[1] / n, v[2] / n]

    def cross(a, b):
        return [a[1] * b[2] - b[1] * a[2], a[2] * b[0] - b[2] * a[0], a[0] * b[1] - b[0] * a[1]]

    up = [0, -1, 0]
    z = normalize((target[0] - eye[0], target[1] - eye[1], target[2] - eye[2]))
    x = normalize(cross(z, up))
    y = cross(x, z)
    z = [-z[0], -z[1], -z[2]]
    dot = lambda a, b: a[0] * b[0] + a[1] * b[1] + a[2] * b[2]
    view = np.asarray([[*x, -dot(x, eye)], [*y, -dot(y, eye)], [*z, -dot(z, eye)], [0, 0, 0, 1]], np.float64)
    return CV2GL @ view


def side_poses(pelvis_z):
    """[3,3,4] world -> camera poses of the displaced, side and bird's-eye views for the persons' pelvis depths."""
    zt = float(np.median(np.asarray(pelvis_z, np.float64)))
    H = [look_at([2.0, -1, -2], [0, 0, 3]), look_at([2.2 * zt, 0, zt], [0, 0, zt]),
         look_at([0.0, -2 * zt, zt - 0.001], [0, 0, zt])]
    return np.stack([h[:3, :4] for h in H])


def orbit_rotation(angle_deg, axis):
    th = np.deg2rad(angle_deg)
    c, s = np.cos(th), np.sin(th)
    if axis == "y":
        return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def orbit_poses(first_verts, n_frames, angle_range):
    """[3 n_frames, 3, 4]: sweeps y by +range, y by -range, x by +range about the vertex mean of `first_verts`."""
    c = np.asarray(first_verts, np.float64).mean(0)
    out = []
    for rng, axis in ((angle_range, "y"), (-angle_range, "y"), (angle_range, "x")):
        for i in range(n_frames):
            R = orbit_rotation(rng * i / (n_frames - 1), axis)
            out.append(np.concatenate([R, (c - R @ c)[:, None]], 1))
    return np.stack(out)


def rasterize_meshes(l_verts, l_faces, K, H: int, W: int, R=None, t=None, normals=None, colors=None, intensity=3.0,
                     metallic=0.0, roughness=0.5, smooth=True, device="cpu", chunk_pairs=1 << 22) -> dict:
    """render_ref.rasterize for meshes of several topologies in one z-buffer: mesh i has vertices l_verts[i] [V_i,3]
    and faces l_faces[i]; the key's face field is sized for the largest face count, ties go to the smaller
    (mesh, face) and 'index' holds the mesh.  Same outputs as render_ref.rasterize."""
    dt = torch.float64
    dev = torch.device(device)
    l_verts = [torch.as_tensor(np.asarray(v), dtype=dt).to(dev) for v in l_verts]
    l_faces = [torch.as_tensor(np.asarray(f)).long().to(dev) for f in l_faces]
    K = torch.as_tensor(np.asarray(K), dtype=dt).to(dev)
    R = torch.eye(3, dtype=dt, device=dev) if R is None else torch.as_tensor(np.asarray(R), dtype=dt).to(dev)
    t = torch.zeros(3, dtype=dt, device=dev) if t is None else torch.as_tensor(np.asarray(t), dtype=dt).reshape(3).to(dev)
    P = len(l_verts)
    fbits = max(1, int(max(f.shape[0] for f in l_faces) - 1).bit_length())
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    HW = H * W
    z1 = torch.full((HW,), math.inf, dtype=dt, device=dev)
    id1 = torch.full((HW,), _BIG, dtype=torch.int64, device=dev)
    z2 = torch.full((HW,), math.inf, dtype=dt, device=dev)
    edge = torch.full((HW,), math.inf, dtype=dt, device=dev)
    for pi in range(P):
        faces = l_faces[pi]
        pc = l_verts[pi] @ R.T + t
        p = pc[faces]
        n = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=-1)
        keep = ((n * p[:, 0]).sum(-1) < 0) & (p[..., 2].amax(1) >= ZNEAR) & (p[..., 2].amin(1) <= ZFAR)
        fid = torch.nonzero(keep).flatten()
        if fid.numel() == 0:
            continue
        x0, x1, y0, y1 = _bbox(p[fid], K, W, H)
        bw, bh = (x1 - x0 + 1).clamp_min(0), (y1 - y0 + 1).clamp_min(0)
        cnt = bw * bh
        m_all = _edge_planes(p[fid])
        n_all = n[fid]
        np0_all = (n_all * p[fid, 0]).sum(-1)
        cross_near = p[fid, :, 2].amin(1) < ZNEAR
        csum = torch.cumsum(cnt, 0)
        start = 0
        while start < fid.numel():
            base = csum[start - 1] if start > 0 else torch.zeros((), dtype=csum.dtype, device=dev)
            end = max(int(torch.searchsorted(csum, base + chunk_pairs, right=True)), start + 1)
            sl = slice(start, end)
            c = cnt[sl]
            tot = int(c.sum())
            start = end
            if tot == 0:
                continue
            owner = torch.repeat_interleave(torch.arange(c.numel(), device=dev), c)
            off = torch.arange(tot, device=dev) - torch.repeat_interleave(torch.cumsum(c, 0) - c, c)
            w_ = bw[sl][owner]
            xs = x0[sl][owner] + off % w_
            ys = y0[sl][owner] + off // w_
            dx = (xs.to(dt) + 0.5 - cx) / fx
            dy = (ys.to(dt) + 0.5 - cy) / fy
            m = m_all[sl][owner]
            e = m[..., 0] * dx[:, None] + m[..., 1] * dy[:, None] + m[..., 2]
            gx, gy = m[..., 0] / fx, m[..., 1] / fy
            dist = e / torch.sqrt(gx * gx + gy * gy).clamp_min(1e-300)
            own = (m[..., 0] > 0) | ((m[..., 0] == 0) & (m[..., 1] > 0))
            inside = ((e > 0) | ((e == 0) & own)).all(1)
            s = e.sum(1)
            pp = p[fid[sl]][owner]
            z = (e * pp[..., 2]).sum(1) / s
            nn = n_all[sl][owner]
            g = nn[:, 0] * dx + nn[:, 1] * dy + nn[:, 2] - np0_all[sl][owner] / ZNEAR
            gdist = (g / torch.sqrt((nn[:, 0] / fx) ** 2 + (nn[:, 1] / fy) ** 2).clamp_min(1e-300)).abs()
            near_line = torch.where(cross_near[sl][owner], gdist, torch.full_like(gdist, math.inf))
            margin = dist.amin(1)
            pix = ys * W + xs
            rel = margin > -1e-2
            ed = torch.minimum(dist.abs().amin(1), near_line)
            edge.scatter_reduce_(0, pix[rel], ed[rel], "amin")
            cov = inside & (s > 0) & (z >= ZNEAR) & (z <= ZFAR)
            pix, z = pix[cov], z[cov]
            ids = (pi << fbits) | fid[sl][owner][cov]
            have = torch.isfinite(z1)
            cp = torch.cat([pix, have.nonzero().flatten(), torch.isfinite(z2).nonzero().flatten()])
            cz = torch.cat([z, z1[have], z2[torch.isfinite(z2)]])
            cid = torch.cat([ids, id1[have], torch.full((int(torch.isfinite(z2).sum()),), _BIG + 1,
                                                        dtype=torch.int64, device=dev)])
            nz1 = torch.full((HW,), math.inf, dtype=dt, device=dev).scatter_reduce_(0, cp, cz, "amin")
            at1 = cz == nz1[cp]
            nid1 = torch.full((HW,), _BIG, dtype=torch.int64, device=dev).scatter_reduce_(0, cp[at1], cid[at1], "amin")
            win = at1 & (cid == nid1[cp])
            nz2 = torch.full((HW,), math.inf, dtype=dt, device=dev).scatter_reduce_(0, cp[~win], cz[~win], "amin")
            z1, id1, z2 = nz1, nid1, nz2
    fg = torch.isfinite(z1)
    out_depth = torch.where(fg, z1, torch.zeros_like(z1))
    person = torch.where(fg, id1 >> fbits, torch.full_like(id1, -1))
    face = torch.where(fg, id1 & ((1 << fbits) - 1), torch.full_like(id1, -1))
    rgb = torch.zeros(HW, 3, dtype=torch.uint8, device=dev)
    for mi in torch.unique(person[fg]).tolist():
        pix = (fg & (person == mi)).nonzero().flatten()
        faces = l_faces[mi]
        xs, ys = pix % W, pix // W
        dx = (xs.to(dt) + 0.5 - cx) / fx
        dy = (ys.to(dt) + 0.5 - cy) / fy
        fv = faces[face[pix]]
        p = (l_verts[mi] @ R.T + t)[fv]
        m = _edge_planes(p)
        e = m[..., 0] * dx[:, None] + m[..., 1] * dy[:, None] + m[..., 2]
        lam = e / e.sum(1, keepdim=True)
        if smooth:
            vn = normals[mi] if normals is not None else vertex_normals(l_verts[mi], faces)
            vn = torch.as_tensor(np.asarray(vn) if not torch.is_tensor(vn) else vn, dtype=dt).to(dev)
            nrm = (lam[..., None] * vn[fv]).sum(1) @ R.T
        else:
            nrm = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=-1)
        nrm = nrm / nrm.norm(dim=-1, keepdim=True).clamp_min(1e-300)
        zz = out_depth[pix]
        pos = torch.stack([dx * zz, dy * zz, zz], 1)
        view = -pos / pos.norm(dim=-1, keepdim=True)
        cols = torch.as_tensor(np.asarray(colors[mi], np.float64)[:3], dtype=dt).to(dev).expand(pix.numel(), 3)
        rgb[pix] = torch.round(shade(nrm, view, cols, intensity, metallic, roughness) * 255.0).to(torch.uint8)
    gap = torch.where(fg, (z2 - z1) / z1.where(fg, torch.ones_like(z1)), torch.full_like(z1, math.inf))
    cpu = lambda a, *s: a.reshape(*s).cpu().numpy()
    return {"rgb": cpu(rgb, H, W, 3), "depth": cpu(out_depth, H, W), "index": cpu(person, H, W).astype(np.int32),
            "face": cpu(face, H, W).astype(np.int32), "edge_dist": cpu(edge, H, W), "depth_gap": cpu(gap, H, W)}


# ---------------------------------------------------------------------------------------------- pyvista / trimesh
# [3P-memory] restatement of what pyvista (VTK sources) returns for utils/render.py:236-274, written from the VTK
# sources' construction, independently of multihmr_b200.render.camera_glyph: float32 points as VTK outputs them,
# polygons fan-triangulated by `triangulate()`, and trimesh's merge of coincident points on construction.

def _rot_axis(axis, deg):
    """Rodrigues rotation about `axis` by `deg` degrees (vtkTransform.RotateWXYZ)."""
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    th = np.deg2rad(deg)
    Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def vtk_cone(height, radius, resolution, center=(0, 0, 0), direction=(1, 0, 0)):
    """vtkConeSource, capped: point 0 the apex at (h/2, 0, 0), points 1..res the base ring at x = -h/2, angle
    2 pi i / res in the (y, z) plane; the base polygon (ring reversed) then the side triangles (0, i, i+1); rotated
    180 degrees about (direction + |direction| x) / 2 (direction with x < 0: about (d - |d| x) / 2, then 180 about y)
    and moved to `center`.  Returns (points, polygons)."""
    ang = 2 * np.pi / resolution
    pts = [(height / 2, 0.0, 0.0)] + [(-height / 2, radius * np.cos(i * ang), radius * np.sin(i * ang))
                                       for i in range(resolution)]
    polys = [[resolution - i for i in range(resolution)]]
    polys += [[0, i + 1, (i + 1) % resolution + 1] for i in range(resolution)]
    P = np.asarray(pts)
    d = np.asarray(direction, np.float64)
    if not (d[0] == 1 and d[1] == 0 and d[2] == 0):
        n = np.linalg.norm(d)
        if d[0] < 0:
            R = _rot_axis(((d[0] - n) / 2, d[1] / 2, d[2] / 2), 180) @ _rot_axis((0, 1, 0), 180)
        else:
            R = _rot_axis(((d[0] + n) / 2, d[1] / 2, d[2] / 2), 180)
        P = P @ R.T
    return (P + np.asarray(center, np.float64)).astype(np.float32), polys


def vtk_cylinder(height, radius, resolution):
    """vtkCylinderSource along y, centred, capped: side points (bottom / top per angle, x = r cos a, z = -r sin a),
    side quads, then each cap's own ring of points and polygon."""
    pts, polys = [], []
    for i in range(resolution):
        a = 2 * np.pi * i / resolution
        x, z = radius * np.cos(a), -radius * np.sin(a)
        pts += [(x, 0.5 * height, z), (x, -0.5 * height, z)]
    for i in range(resolution):
        j = (i + 1) % resolution
        polys.append([2 * i, 2 * i + 1, 2 * j + 1, 2 * j])
    base = len(pts)
    for i in range(resolution):
        a = 2 * np.pi * i / resolution
        pts.append((radius * np.cos(a), 0.5 * height, -radius * np.sin(a)))
    polys.append([base + i for i in range(resolution)])
    base2 = len(pts)
    for i in range(resolution):
        a = 2 * np.pi * i / resolution
        pts.append((radius * np.cos(a), -0.5 * height, -radius * np.sin(a)))
    polys.append([base2 + resolution - 1 - i for i in range(resolution)])
    return np.asarray(pts, np.float64), polys


def vtk_arrow(tip_length=0.25, tip_radius=0.1, tip_resolution=20, shaft_radius=0.05, shaft_resolution=20):
    """vtkArrowSource: the cylinder turned -90 degrees about z onto x and moved to ((1 - tip) / 2, 0, 0), then the cone
    tip centred at (1 - tip / 2, 0, 0), appended."""
    cp, cpoly = vtk_cylinder(1.0 - tip_length, shaft_radius, shaft_resolution)
    cp = cp @ _rot_axis((0, 0, 1), -90).T + [(1.0 - tip_length) / 2, 0, 0]
    tp, tpoly = vtk_cone(tip_length, tip_radius, tip_resolution, center=(1.0 - tip_length / 2, 0, 0))
    polys = cpoly + [[k + len(cp) for k in p] for p in tpoly]
    return np.concatenate([cp, tp.astype(np.float64)]).astype(np.float32), polys


class PolyData:
    """What the reference reads of a pyvista mesh: points, `faces` (flat [n, i0, .. in-1, ...]), n_faces,
    extract_surface(), triangulate() (fan per polygon)."""

    def __init__(self, points, polys):
        self.points, self._polys = np.asarray(points), [list(p) for p in polys]

    @property
    def n_faces(self):
        return len(self._polys)

    @property
    def faces(self):
        return np.asarray([v for p in self._polys for v in [len(p)] + p], np.int64)

    def extract_surface(self):
        return self

    def triangulate(self):
        return PolyData(self.points, [[p[0], p[k], p[k + 1]] for p in self._polys for k in range(1, len(p) - 1)])


def _outward(points, polys, parts):
    """Winds each polygon of the closed convex parts (lists of polygon indices) away from the part's centroid."""
    P = np.asarray(points, np.float64)
    polys = [list(p) for p in polys]
    for part in parts:
        c = P[sorted({v for i in part for v in polys[i]})].mean(0)
        for i in part:
            q = P[polys[i]]
            n = sum(np.cross(q[k], q[(k + 1) % len(q)]) for k in range(len(q)))
            if n @ (q.mean(0) - c) < 0:
                polys[i] = polys[i][::-1]
    return polys


def pyvista_cone(center=(0.0, 0.0, 0.0), direction=(1.0, 0.0, 0.0), height=1.0, radius=0.5, resolution=6):
    p, polys = vtk_cone(height, radius, resolution, center, direction)
    return PolyData(p, _outward(p, polys, [range(len(polys))]))


def pyvista_box(bounds=(-1.0, 1.0, -1.0, 1.0, -1.0, 1.0)):
    """vtkTessellatedBoxSource, level 0, quads, duplicated shared points: 4 points per face."""
    x0, x1, y0, y1, z0, z1 = bounds
    faces = [[(x0, y0, z0), (x0, y1, z0), (x0, y1, z1), (x0, y0, z1)], [(x1, y0, z0), (x1, y0, z1), (x1, y1, z1),
                                                                           (x1, y1, z0)],
             [(x0, y0, z0), (x0, y0, z1), (x1, y0, z1), (x1, y0, z0)], [(x0, y1, z0), (x1, y1, z0), (x1, y1, z1),
                                                                           (x0, y1, z1)],
             [(x0, y0, z0), (x1, y0, z0), (x1, y1, z0), (x0, y1, z0)], [(x0, y0, z1), (x0, y1, z1), (x1, y1, z1),
                                                                           (x1, y0, z1)]]
    pts = np.asarray([c for f in faces for c in f], np.float32)
    polys = [[4 * i + k for k in range(4)] for i in range(6)]
    return PolyData(pts, _outward(pts, polys, [range(6)]))


def pyvista_arrow(start=(0.0, 0.0, 0.0), direction=(1.0, 0.0, 0.0), tip_length=0.25, tip_radius=0.1,
                  tip_resolution=20, shaft_radius=0.05, shaft_resolution=20, scale=None):
    """pyvista.Arrow: vtkArrowSource, then pyvista's `translate` (x onto `direction`, the frame's z = x cross (0,1,0),
    or cross (0,0,1) when x is along y) and `points *= scale`."""
    p, polys = vtk_arrow(tip_length, tip_radius, tip_resolution, shaft_radius, shaft_resolution)
    ns = len(polys) - (tip_resolution + 1)
    polys = _outward(p, polys, [range(ns), range(ns, len(polys))])
    nx = np.asarray(direction, np.float64) / np.linalg.norm(direction)
    ny_tmp = np.array([0.0, 0.0, 1.0]) if np.allclose(abs(nx[1]), 1.0) else np.array([0.0, 1.0, 0.0])
    nz = np.cross(nx, ny_tmp)
    nz = nz / np.linalg.norm(nz)
    ny = np.cross(nz, nx)
    M = np.stack([nx, ny, nz], 1)
    pts = (p.astype(np.float64) @ M.T + np.asarray(start)).astype(np.float32)
    if scale is not None:
        pts = pts * np.float32(scale)
    return PolyData(pts, polys)


def merge_vertices(verts, faces):
    """trimesh's `process=True` on construction: coincident points merged (first occurrence keeps its place),
    faces re-indexed [3P-memory]."""
    v = np.asarray(verts, np.float64)
    key = {}
    remap = np.empty(len(v), np.int64)
    keep = []
    for i, p in enumerate(map(tuple, np.round(v, 8))):
        if p not in key:
            key[p] = len(keep)
            keep.append(i)
        remap[i] = key[p]
    return v[keep], remap[np.asarray(faces, np.int64)]


def glyph_meshes():
    """The camera glyph as the reference builds it (utils/render.py:242-274) from this restatement of pyvista, after
    trimesh's merge: (verts list, faces list, colours list) for cone, box and the x / y / z arrows."""
    def faces_of(x):
        return x.faces.astype(np.uint32).reshape((x.n_faces, 4))[:, 1:]

    height, radius, size, scale = 0.2, 0.1, 0.1, 0.2
    cone = pyvista_cone(center=(0.0, 0.0, -height / 2), direction=(0.0, 0.0, -1.0), height=height,
                        radius=radius).extract_surface().triangulate()
    zmin = cone.points[:, -1].min()
    box = pyvista_box(bounds=(-size, size, -size, size, zmin - 3 * size, zmin)).extract_surface().triangulate()
    out = [merge_vertices(cone.points, faces_of(cone)), merge_vertices(box.points, faces_of(box))]
    for d in [(1, 0, 0), (0, 1, 0), (0, 0, 1)]:
        a = pyvista_arrow(direction=d, scale=scale).extract_surface().triangulate()
        out.append(merge_vertices(a.points + np.asarray([[2 * scale, 0.0, -scale]]), faces_of(a)))
    colors = [(0.5, 0.5, 0.5), (0.5, 0.5, 0.5), (1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)]
    return [v for v, _ in out], [f for _, f in out], colors


def views(verts, faces, K, H, W, photo, alpha, colors, pelvis_z, n_frames=None, angle_range=None, side=False,
          device="cpu"):
    """One image's demo views: {'overlay': (raster, composite), 'orbit': [...], 'side': [...]} with each raster the
    rasterize_meshes dict of that view plus 'overlay'.  verts [P,V,3] in list order (first = orbit centre)."""
    P = len(verts)
    white = np.full_like(photo, 255)
    out = {}

    def one(R, t, img, a, with_glyph):
        lv, lf, lc = list(verts), [faces] * P, list(colors)
        if with_glyph:
            gv, gf, gc = glyph_meshes()
            lv, lf, lc = lv + gv, lf + gf, lc + gc
        r = rasterize_meshes(lv, lf, K, H, W, R=R, t=t, colors=lc, device=device)
        r["overlay"] = composite(r["rgb"], r["depth"], img, a)
        return r

    out["overlay"] = one(None, None, photo, alpha, False)
    if n_frames:
        out["orbit"] = [one(q[:, :3], q[:, 3], white, alpha, False) for q in orbit_poses(verts[0], n_frames,
                                                                                           angle_range)]
    if side:
        # render_side_views blends over a float64 white (utils/render.py:418-420), which sets numpy's promotion
        out["side"] = [one(q[:, :3], q[:, 3], white.astype(np.float64), 1.0, True) for q in side_poses(pelvis_z)]
    return out
