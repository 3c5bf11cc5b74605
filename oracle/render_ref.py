"""fp64 restatement of the mesh overlay (reference utils/render.py:175 `render_meshes` through pyrender / trimesh),
vectorised over faces, for small images.  Items marked [3P-memory] restate pyrender / trimesh from memory: neither
package is installed here.

1. Camera: world -> camera [R|t] (OpenCV), u = fx x/z + cx, v = fy y/z + cy, y down; near 0.05 / far 100
   (pyrender IntrinsicsCamera defaults [3P-memory]); a triangle crossing the near plane is clipped.
2. Coverage: one sample at each pixel centre (x+0.5, y+0.5), edge functions with the top-left rule.  pyrender's
   framebuffer may multisample [3P-memory]; this restatement does not.
3. Culling: GL's default counter-clockwise front face, back faces culled (material not doubleSided) [3P-memory].
4. Visibility: camera z interpolated perspective-correctly, nearest wins, ties to the smaller (person, face).
5. Normals: trimesh vertex normals = unit face normals weighted by corner angle, normalised [3P-memory]; or face
   normals with smooth=False.
6. Shading: pyrender's metallic-roughness fragment shader (glTF reference BRDF: Schlick Fresnel with F0 0.04,
   Smith-GGX occlusion with k = (r+1)^2/8, GGX distribution), one white directional light along the view direction,
   ambient 0.3 x base colour, pow(c, 1/2.2), clamped, rounded to uint8 [3P-memory].  Background 0, depth 0.
7. Composite: the reference's own 3x3 foreground smoothing and alpha blend (utils/render.py:297-311).

Besides the images, `rasterize` reports per pixel the distance of the pixel centre to the nearest edge (or near-plane
clip line) of any triangle covering or almost covering it, in pixels, and the relative depth gap to the second
nearest surface: pixels where float32 arithmetic may legitimately decide differently.
"""
from __future__ import annotations

import math

import numpy as np
import torch

ZNEAR, ZFAR = 0.05, 100.0
AMBIENT = 0.3
MIN_ROUGHNESS = 0.04
_BIG = 1 << 62


def face_normals(v: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """Unit normals of cross(v1 - v0, v2 - v0); zero for a degenerate face."""
    p = v[faces]
    n = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=-1)
    ln = n.norm(dim=-1, keepdim=True)
    return torch.where(ln > 0, n / ln.clamp_min(1e-300), torch.zeros_like(n))


def vertex_normals(v: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """trimesh `vertex_normals` [3P-memory]: face normals weighted by the face's angle at the vertex, normalised."""
    p = v[faces]                                                       # [F,3,3]
    fn = face_normals(v, faces)
    out = torch.zeros_like(v)
    for c in range(3):
        u = p[:, (c + 1) % 3] - p[:, c]
        w = p[:, (c + 2) % 3] - p[:, c]
        ang = torch.atan2(torch.cross(u, w, dim=-1).norm(dim=-1), (u * w).sum(-1))
        out.index_add_(0, faces[:, c], fn * ang[:, None])
    ln = out.norm(dim=-1, keepdim=True)
    return torch.where(ln > 0, out / ln.clamp_min(1e-300), torch.zeros_like(out))


def shade(n: torch.Tensor, v: torch.Tensor, base: torch.Tensor, intensity: float, metallic: float,
          roughness: float) -> torch.Tensor:
    """Item 6 for unit normals n [N,3] and view vectors v [N,3] (camera space), base colours [N,3]; returns the
    gamma-corrected colour in [0, 1]."""
    r = min(max(roughness, MIN_ROUGHNESS), 1.0)
    m = min(max(metallic, 0.0), 1.0)
    l = torch.tensor([0.0, 0.0, -1.0], dtype=n.dtype, device=n.device).expand_as(n)
    h = l + v
    h = h / h.norm(dim=-1, keepdim=True)
    nl = (n * l).sum(-1).clamp(0.001, 1.0)[:, None]
    nv = (n * v).sum(-1).abs().clamp(0.001, 1.0)[:, None]
    nh = (n * h).sum(-1).clamp(0.0, 1.0)[:, None]
    vh = (v * h).sum(-1).clamp(0.0, 1.0)[:, None]
    f0 = MIN_ROUGHNESS + (base - MIN_ROUGHNESS) * m
    c_diff = base * (1.0 - MIN_ROUGHNESS) * (1.0 - m)
    F = f0 + (1.0 - f0) * (1.0 - vh).clamp(0.0, 1.0) ** 5
    k = (r + 1.0) ** 2 / 8.0
    G = nv / (nv * (1.0 - k) + k) * (nl / (nl * (1.0 - k) + k))
    a2 = (r * r) ** 2
    fd = nh * nh * (a2 - 1.0) + 1.0
    D = a2 / (math.pi * fd * fd)
    col = nl * intensity * ((1.0 - F) * c_diff / math.pi + F * G * D / (4.0 * nl * nv + 0.001)) + AMBIENT * base
    return col.clamp_min(0.0).pow(1.0 / 2.2).clamp(0.0, 1.0)


def _edge_planes(p: torch.Tensor) -> torch.Tensor:
    """m[:, k] = p_j x p_i for the edge (i, j) = (k+1, k+2) opposite vertex k; e_k = d . m_k > 0 inside a front face."""
    return torch.stack([torch.cross(p[:, (k + 2) % 3], p[:, (k + 1) % 3], dim=-1) for k in range(3)], 1)


def _bbox(p: torch.Tensor, K: torch.Tensor, W: int, H: int):
    """Pixel box of the near-clipped triangles (conservative by one pixel)."""
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    pts, ok = [], []
    for k in range(3):
        a, b = p[:, k], p[:, (k + 1) % 3]
        ina, inb = a[:, 2] >= ZNEAR, b[:, 2] >= ZNEAR
        pts.append(a)
        ok.append(ina)
        s = ((ZNEAR - a[:, 2]) / (b[:, 2] - a[:, 2]).where(ina != inb, torch.ones_like(a[:, 2])))[:, None]
        q = a + s * (b - a)
        pts.append(q)
        ok.append(ina != inb)
    P = torch.stack(pts, 1)
    O = torch.stack(ok, 1)
    z = P[..., 2].where(O, torch.ones_like(P[..., 2]))
    u = (fx * P[..., 0] / z + cx).where(O, torch.full_like(z, math.inf))
    v = (fy * P[..., 1] / z + cy).where(O, torch.full_like(z, math.inf))
    umin, vmin = u.amin(1), v.amin(1)
    umax = u.where(O, torch.full_like(u, -math.inf)).amax(1)
    vmax = v.where(O, torch.full_like(v, -math.inf)).amax(1)
    x0 = (umin.clamp(-2, W + 2) - 0.5).floor().long() - 1
    x1 = (umax.clamp(-2, W + 2) - 0.5).ceil().long() + 1
    y0 = (vmin.clamp(-2, H + 2) - 0.5).floor().long() - 1
    y1 = (vmax.clamp(-2, H + 2) - 0.5).ceil().long() + 1
    return x0.clamp_min(0), x1.clamp_max(W - 1), y0.clamp_min(0), y1.clamp_max(H - 1)


def rasterize(verts, faces, K, H: int, W: int, R=None, t=None, normals=None, colors=None, intensity=3.0,
              metallic=0.0, roughness=0.5, smooth=True, device="cpu", chunk_pairs=1 << 22) -> dict:
    """Renders persons `verts` [P,V,3] (faces [F,3] shared) into one H x W view.  Returns numpy arrays: 'rgb' uint8
    [H,W,3] (0 = background), 'depth' [H,W] (0 = background), 'index' [H,W] person (-1), 'face' [H,W] (-1),
    'edge_dist' [H,W] px, 'depth_gap' [H,W] relative.  `normals` [P,V,3] overrides the smooth vertex normals
    (the pyrender shim passes trimesh's); `colors` [P,3] in [0,1]."""
    dt = torch.float64
    dev = torch.device(device)
    verts = torch.as_tensor(np.asarray(verts), dtype=dt).to(dev)
    faces = torch.as_tensor(np.asarray(faces)).long().to(dev)
    K = torch.as_tensor(np.asarray(K), dtype=dt).to(dev)
    R = torch.eye(3, dtype=dt, device=dev) if R is None else torch.as_tensor(np.asarray(R), dtype=dt).to(dev)
    t = torch.zeros(3, dtype=dt, device=dev) if t is None else torch.as_tensor(np.asarray(t), dtype=dt).reshape(3).to(dev)
    P, F = verts.shape[0], faces.shape[0]
    fbits = max(1, int(F - 1).bit_length())
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    HW = H * W
    z1 = torch.full((HW,), math.inf, dtype=dt, device=dev)
    id1 = torch.full((HW,), _BIG, dtype=torch.int64, device=dev)
    z2 = torch.full((HW,), math.inf, dtype=dt, device=dev)
    edge = torch.full((HW,), math.inf, dtype=dt, device=dev)
    for pi in range(P):
        pc = verts[pi] @ R.T + t
        p = pc[faces]                                                       # [F,3,3]
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
            end = int(torch.searchsorted(csum, base + chunk_pairs, right=True))
            end = max(end, start + 1)
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
            m = m_all[sl][owner]                                               # [N,3,3]
            e = m[..., 0] * dx[:, None] + m[..., 1] * dy[:, None] + m[..., 2]
            gx, gy = m[..., 0] / fx, m[..., 1] / fy
            dist = e / torch.sqrt(gx * gx + gy * gy).clamp_min(1e-300)        # signed, px
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
            # merge with the running (nearest, its id, second nearest) of each pixel
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
    pix = fg.nonzero().flatten()
    if pix.numel():
        pp_, ff = person[pix], face[pix]
        xs, ys = pix % W, pix // W
        dx = (xs.to(dt) + 0.5 - cx) / fx
        dy = (ys.to(dt) + 0.5 - cy) / fy
        pc = torch.einsum("pvc,dc->pvd", verts, R) + t                     # [P,V,3] camera space
        fv = faces[ff]                                                      # [N,3]
        p = pc[pp_[:, None], fv]                                            # [N,3,3]
        m = _edge_planes(p)
        e = m[..., 0] * dx[:, None] + m[..., 1] * dy[:, None] + m[..., 2]
        lam = e / e.sum(1, keepdim=True)
        if smooth:
            vn = normals if normals is not None else torch.stack([vertex_normals(verts[i], faces) for i in range(P)])
            vn = torch.as_tensor(np.asarray(vn) if not torch.is_tensor(vn) else vn, dtype=dt).to(dev)
            nrm = (lam[..., None] * vn[pp_[:, None], fv]).sum(1) @ R.T
        else:
            nrm = torch.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=-1)
        nrm = nrm / nrm.norm(dim=-1, keepdim=True).clamp_min(1e-300)
        zz = out_depth[pix]
        pos = torch.stack([dx * zz, dy * zz, zz], 1)
        view = -pos / pos.norm(dim=-1, keepdim=True)
        cols = torch.as_tensor(np.asarray(colors), dtype=dt).to(dev)[pp_]
        c = shade(nrm, view, cols, intensity, metallic, roughness)
        rgb[pix] = torch.round(c * 255.0).to(torch.uint8)
    gap = torch.where(fg, (z2 - z1) / z1.where(fg, torch.ones_like(z1)), torch.full_like(z1, math.inf))
    cpu = lambda a, *s: a.reshape(*s).cpu().numpy()
    return {"rgb": cpu(rgb, H, W, 3), "depth": cpu(out_depth, H, W), "index": cpu(person, H, W).astype(np.int32),
            "face": cpu(face, H, W).astype(np.int32), "edge_dist": cpu(edge, H, W), "depth_gap": cpu(gap, H, W)}


def composite(rgb, depth, img, alpha):
    """Item 7, the reference's smoothing and blend (utils/render.py:297-311): fg = depth > 0, a 3x3 box of weight 2/9
    with bias -1 and zero padding, times fg, clamped at 0; then fg (alpha rgb + (1 - alpha) img) + (1 - fg) img in
    numpy's promotion of the reference's operands, truncated to uint8."""
    rgb = np.asarray(rgb)[:, :, :3].astype(np.float32)
    fg = torch.from_numpy((np.asarray(depth) > 0).astype(np.float32))[None]
    kern = 2.0 * torch.ones((1, 1, 3, 3)) / 9
    fg = torch.clamp_min(torch.nn.functional.conv2d(fg, weight=kern, bias=-torch.ones(1), padding=1) * fg, 0.0)
    fg = fg.permute(1, 2, 0).numpy()
    blend = alpha * rgb + (1.0 - alpha) * img
    return (fg * blend + (1 - fg) * img).astype(np.uint8)


def render_meshes(img, verts, faces, K, R=None, t=None, colors=None, alpha=1.0, intensity=3.0, metallic=0.0,
                  roughness=0.5, smooth=True, device="cpu") -> dict:
    """Items 1-7 for one view: the `rasterize` outputs plus 'overlay' uint8 [H,W,3]."""
    H, W = np.asarray(img).shape[:2]
    out = rasterize(verts, faces, K, H, W, R=R, t=t, colors=colors, intensity=intensity, metallic=metallic,
                    roughness=roughness, smooth=smooth, device=device)
    out["overlay"] = composite(out["rgb"], out["depth"], np.asarray(img), alpha)
    return out
