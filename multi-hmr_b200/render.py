"""Mesh overlay on the device (`mhmr_render_*`, csrc/render.cu): the reference's `utils/render.py:175 render_meshes`
without pyrender / OpenGL, for any body model's faces (SMPL-X `model.smpl_layer['neutral_10'].bm_x.faces`, Anny
`model.body_model.faces`).

    Renderer(faces, device).render(verts, K, images, ...)   tensor in / tensor out, B views per call
    Renderer.render_outputs(t, images, K)                   straight from `Model.forward_raw`'s output dict
    render_meshes(img, l_mesh, l_face, cam_param, ...)      the reference's signature and numpy return

Arithmetic (what the kernels and `oracle/render_ref.py` implement): camera `[R|t]` world -> camera in the OpenCV
convention, `u = fx x/z + cx`, `v = fy y/z + cy`, near / far planes 0.05 / 100; one sample at each pixel centre with
the top-left fill rule; back faces culled; nearest depth wins, ties to the smaller (person, face); pyrender's
metallic-roughness shading under a white directional light at the camera plus ambient 0.3, gamma 2.2, rounded to
uint8; then the reference's 3x3 foreground smoothing and alpha blend, truncated to uint8.  pyrender may multisample
its framebuffer; this renderer does not, so silhouette pixels can differ from a pyrender run.
"""
from __future__ import annotations

import colorsys
import ctypes
import hashlib
from ctypes import c_int, c_void_p

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr

ZNEAR, ZFAR = 0.05, 100.0


def _palette(n: int = 40) -> list[tuple[float, float, float]]:
    """This package's person colours: hues a golden-ratio step apart, alternating two saturation / value levels."""
    out = []
    for i in range(n):
        h = (0.58 + 0.6180339887 * i) % 1.0
        s, v = (0.55, 0.95) if i % 2 == 0 else (0.75, 0.8)
        out.append(tuple(round(c, 4) for c in colorsys.hsv_to_rgb(h, s, v)))
    return out


PALETTE = _palette()


def _stream(dev):
    return c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _faces(faces) -> torch.Tensor:
    f = torch.as_tensor(np.asarray(faces) if not torch.is_tensor(faces) else faces)
    if f.ndim != 2 or f.shape[1] != 3 or f.shape[0] < 1:
        raise ValueError(f"faces must be [F,3], got {tuple(f.shape)}")
    if f.dtype.is_floating_point:
        raise ValueError("faces must be integers")
    return f.to(torch.int64).cpu()


def _orient_out(v: np.ndarray, f: np.ndarray) -> np.ndarray:
    """Winds every face of a convex closed component so that cross(v1 - v0, v2 - v0) points away from its centroid."""
    p = v[f]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    flip = (n * (p.mean(1) - v[np.unique(f)].mean(0))).sum(-1) < 0
    f = f.copy()
    f[flip] = f[flip][:, [0, 2, 1]]
    return f


def _ring(n, radius, x):
    a = 2 * np.pi * np.arange(n) / n
    return np.stack([np.full(n, x), radius * np.cos(a), radius * np.sin(a)], 1)


def _fan(ids):
    return [[ids[0], ids[i], ids[i + 1]] for i in range(1, len(ids) - 1)]


def _vtk_cone(height, radius, res, center=(0.0, 0.0, 0.0), direction=(1.0, 0.0, 0.0)):
    """vtkConeSource, capped: apex at x = +h/2, a ring of `res` points at x = -h/2 shared by the sides and the cap,
    then the source's 180-degree turn of +x onto `direction` and the shift to `center` [3P-memory]."""
    v = np.concatenate([[[height / 2, 0.0, 0.0]], _ring(res, radius, -height / 2)])
    f = [[0, 1 + i, 1 + (i + 1) % res] for i in range(res)] + _fan(list(range(1, res + 1)))
    d = np.asarray(direction, np.float64)
    if not np.array_equal(d, [1.0, 0.0, 0.0]):
        m = np.linalg.norm(d)
        rot = lambda a: 2 * np.outer(a, a) / (a @ a) - np.eye(3)  # 180 degrees about a
        if d[0] < 0:
            R = rot(np.array([(d[0] - m) / 2, d[1] / 2, d[2] / 2])) @ rot(np.array([0.0, 1.0, 0.0]))
        else:
            R = rot(np.array([(d[0] + m) / 2, d[1] / 2, d[2] / 2]))
        v = v @ R.T
    return v + np.asarray(center), _orient_out(v, np.asarray(f))


def _vtk_arrow(tip_length=0.25, tip_radius=0.1, tip_res=20, shaft_radius=0.05, shaft_res=20):
    """vtkArrowSource along +x from 0 to 1: a capped cylinder shaft to 1 - tip_length and a capped cone tip, two closed
    components [3P-memory]."""
    shaft = np.concatenate([_ring(shaft_res, shaft_radius, 0.0), _ring(shaft_res, shaft_radius, 1.0 - tip_length)])
    sf = []
    for i in range(shaft_res):
        j = (i + 1) % shaft_res
        sf += [[i, j, shaft_res + j], [i, shaft_res + j, shaft_res + i]]
    sf += _fan(list(range(shaft_res))) + _fan(list(range(shaft_res, 2 * shaft_res)))
    sf = _orient_out(shaft, np.asarray(sf))
    tv, tf = _vtk_cone(tip_length, tip_radius, tip_res, center=(1.0 - tip_length / 2, 0.0, 0.0))
    return np.concatenate([shaft, tv]), np.concatenate([sf, tf + len(shaft)])


def _pyvista_direction(direction):
    """pyvista's `translate` frame: columns normx, normy, normz with normz = normx x (0,1,0) (or (0,0,1) when
    collinear) [3P-memory]."""
    nx = np.asarray(direction, np.float64) / np.linalg.norm(direction)
    tmp = np.array([0.0, 1.0, 0.0]) if not np.isclose(abs(nx @ [0.0, 1.0, 0.0]), 1.0) else np.array([0.0, 0.0, 1.0])
    nz = np.cross(nx, tmp)
    nz /= np.linalg.norm(nz)
    return np.stack([nx, np.cross(nz, nx), nz], 1)


def camera_glyph():
    """The camera glyph of reference utils/render.py:236-274 (`show_camera=True`), in world coordinates: pyvista's
    Cone(center (0,0,-0.1), direction -z, height 0.2, radius 0.1, resolution 6, capped), the Box of +-0.1 in x and y
    from zmin(cone) - 0.3 to zmin(cone), and Arrow(direction x / y / z, scale 0.2) shifted by (0.4, 0, -0.2), each
    `extract_surface().triangulate()`d, with coincident points merged as trimesh does on construction [3P-memory:
    pyvista and trimesh are not installed].  Returns (topologies [faces], meshes [(topology, verts [V,3] fp64,
    colour)]): grey 0.5 cone and box, red / green / blue arrows."""
    cv, cf = _vtk_cone(0.2, 0.1, 6, center=(0.0, 0.0, -0.1), direction=(0.0, 0.0, -1.0))
    z0 = cv[:, 2].min()
    s = 0.1
    bv = np.array([[x, y, z] for z in (z0 - 3 * s, z0) for y in (-s, s) for x in (-s, s)])
    quads = [[0, 1, 3, 2], [4, 5, 7, 6], [0, 1, 5, 4], [2, 3, 7, 6], [0, 2, 6, 4], [1, 3, 7, 5]]
    bf = _orient_out(bv, np.asarray([t for q in quads for t in _fan(q)]))
    av, af = _vtk_arrow()
    meshes = [(0, cv, (0.5, 0.5, 0.5)), (1, bv, (0.5, 0.5, 0.5))]
    for d, col in zip(np.eye(3), [(1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)]):
        meshes.append((2, (av @ _pyvista_direction(d).T) * 0.2 + [0.4, 0.0, -0.2], col))
    return [cf, bf, af], meshes


class Renderer:
    """A renderer for one face array [F,3] (int, indices < num_verts) on one CUDA device.  The handle builds the
    vertex -> face table of the normal pass once and owns the depth-key buffer (8 B per pixel per view).
    `topologies`: extra face arrays (each over max index + 1 vertices) that `render(props=...)` draws in the same
    z-buffer as the persons, e.g. `camera_glyph()`'s."""

    def __init__(self, faces, device="cuda", num_verts: int | None = None, topologies=None):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("the renderer runs on a CUDA device (no CPU fallback)")
        f = _faces(faces)
        V = int(num_verts) if num_verts is not None else int(f.max()) + 1
        self.device, self.num_faces, self.num_verts = dev, int(f.shape[0]), V
        self.faces = f.to(torch.int32).cpu().contiguous()
        topo = [_faces(t).to(torch.int32) for t in (topologies or [])]
        self.topologies = topo
        self.topology_verts = [int(t.max()) + 1 for t in topo]
        self._lib = _lib.load()
        h = c_void_p()
        with torch.cuda.device(dev):
            if topo:
                tf = torch.cat(topo).contiguous()
                nf = torch.tensor([t.shape[0] for t in topo], dtype=torch.int32)
                nv = torch.tensor(self.topology_verts, dtype=torch.int32)
                check(self._lib.mhmr_render_create_topologies(ptr(self.faces), self.num_faces, V, len(topo), ptr(tf),
                                                              ptr(nf), ptr(nv), _stream(dev), ctypes.byref(h)),
                      "mhmr_render_create_topologies")
            else:
                check(self._lib.mhmr_render_create(ptr(self.faces), self.num_faces, V, _stream(dev),
                                                   ctypes.byref(h)), "mhmr_render_create")
        self._h = h
        self._glyph = self._palette = None
        fb = c_int()
        check(self._lib.mhmr_render_info(h, None, None, ctypes.byref(fb)), "mhmr_render_info")
        self.face_bits = fb.value

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            self._lib.mhmr_render_destroy(h)
            self._h = None

    def render(self, verts, K, images, person_image=None, count=None, view_image=None, pose=None, colors=None,
               alpha: float = 1.0, intensity: float = 3.0, metallic: float = 0.0, roughness: float = 0.5,
               smooth: bool = True, depth: bool = False, index: bool = False, props=None, prop_visible=None,
               view_alpha=None, view_background=None) -> dict:
        """Renders the persons `verts` [P,V,3] into B = K.shape[0] views and returns {'overlay' [B,H,W,3] uint8,
        'depth' [B,H,W] fp32 (0 = background) if `depth`, 'index' [B,H,W] int32 (-1 = background) if `index`}.

        images: uint8 [N,H,W,3] backgrounds on the device.  view_image: background image of each view (host list /
        array, default 0..B-1).  person_image [P] int32 on the device: person p is drawn into every view whose image
        is person_image[p] (default: all in image 0).  count: device int32 [1] read by the kernels (no host sync) or
        an int (default P).  pose: [B,3,4] world -> camera [R|t] (OpenCV), default identity.  colors [P,3] in [0,1]
        (default `PALETTE`)."""
        dev = self.device
        verts = self._dev(verts, torch.float32)
        if verts.ndim != 3 or verts.shape[1] != self.num_verts or verts.shape[2] != 3:
            raise ValueError(f"verts must be [P,{self.num_verts},3], got {tuple(verts.shape)}")
        P = int(verts.shape[0])
        K = self._dev(K, torch.float32)
        if K.ndim != 3 or K.shape[1:] != (3, 3):
            raise ValueError(f"K must be [B,3,3], got {tuple(K.shape)}")
        B = int(K.shape[0])
        if not torch.is_tensor(images) or images.dtype != torch.uint8 or images.ndim != 4 or images.shape[3] != 3:
            raise ValueError("images must be a uint8 tensor [N,H,W,3]")
        images = images.to(dev).contiguous()
        N, H, W = int(images.shape[0]), int(images.shape[1]), int(images.shape[2])
        vi = np.arange(B) if view_image is None else np.asarray(
            view_image.cpu() if torch.is_tensor(view_image) else view_image).reshape(-1)
        if vi.shape[0] != B or (vi.size and (vi.min() < 0 or vi.max() >= N)):
            raise ValueError(f"view_image must hold {B} image indices in [0, {N})")
        vi = torch.as_tensor(vi.astype(np.int32)).to(dev)
        if pose is not None:
            pose = self._dev(pose, torch.float32)
            if pose.shape != (B, 3, 4):
                raise ValueError(f"pose must be [B,3,4], got {tuple(pose.shape)}")
        Pm = max(P, 1)
        if person_image is None:
            person_image = torch.zeros(Pm, dtype=torch.int32, device=dev)
        person_image = self._dev(person_image, torch.int32)
        if person_image.ndim != 1 or person_image.shape[0] < P:
            raise ValueError(f"person_image must be [P] = [{P}]")
        if count is None or not torch.is_tensor(count):
            n = P if count is None else int(count)
            if not 0 <= n <= P:
                raise ValueError(f"count {n} outside [0, {P}]")
            count = torch.full((1,), n, dtype=torch.int32, device=dev)
        count = self._dev(count, torch.int32)
        if colors is None:
            colors = torch.tensor([PALETTE[i % len(PALETTE)] for i in range(Pm)], dtype=torch.float32)
        colors = self._dev(colors, torch.float32)
        if colors.ndim != 2 or colors.shape[1] != 3 or colors.shape[0] < P:
            raise ValueError(f"colors must be [P,3] = [{P},3]")
        if P == 0:  # nothing to draw: the blend returns the photos
            verts = torch.zeros(1, self.num_verts, 3, device=dev)
            count = torch.zeros(1, dtype=torch.int32, device=dev)
        extra = None
        if props is not None or view_alpha is not None or view_background is not None:
            extra = self._extra(B, N, props or [], prop_visible, view_alpha, view_background)
        return self._launch(B, H, W, images, vi, K, pose, verts, Pm, person_image, count, colors, alpha, intensity,
                            metallic, roughness, smooth, depth, index, extra)

    def _launch(self, B, H, W, images, vi, K, pose, verts, Pm, person_image, count, colors, alpha, intensity,
                metallic, roughness, smooth, depth, index, extra):
        dev = self.device
        out = {"overlay": torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev),
               "depth": torch.empty(B, H, W, dtype=torch.float32, device=dev) if depth else None,
               "index": torch.empty(B, H, W, dtype=torch.int32, device=dev) if index else None}
        args = _lib.RenderArgs(B, H, W, images.data_ptr(), vi.data_ptr(), K.data_ptr(),
                               pose.data_ptr() if pose is not None else None, verts.data_ptr(), Pm,
                               person_image.data_ptr(), count.data_ptr(), colors.data_ptr(), float(alpha),
                               float(intensity), float(metallic), float(roughness), int(bool(smooth)),
                               out["overlay"].data_ptr(), out["depth"].data_ptr() if depth else None,
                               out["index"].data_ptr() if index else None)
        with torch.cuda.device(dev):
            if extra is None:
                check(self._lib.mhmr_render_forward(self._h, ctypes.byref(args), _stream(dev)),
                      "mhmr_render_forward")
            else:
                check(self._lib.mhmr_render_forward_extra(self._h, ctypes.byref(args), ctypes.byref(extra[0]),
                                                          _stream(dev)), "mhmr_render_forward_extra")
        return {k: v for k, v in out.items() if v is not None}

    def _extra(self, B, N, props, prop_visible, view_alpha, view_background):
        """(RenderExtra, tensors it points to).  props: [(topology, verts [V_t,3], colour)]."""
        dev = self.device
        n = len(props)
        keep = []
        topo = torch.tensor([int(p[0]) for p in props] or [0], dtype=torch.int32)
        for t in topo[:n].tolist():
            if not 0 <= t < len(self.topologies):
                raise ValueError(f"prop topology {t} outside [0, {len(self.topologies)})")
        pv = pc = vis = None
        if n:
            parts = [self._dev(p[1], torch.float32) for p in props]
            for (t, _, _), v in zip(props, parts):
                if v.shape != (self.topology_verts[t], 3):
                    raise ValueError(f"prop verts must be [{self.topology_verts[t]},3], got {tuple(v.shape)}")
            pv = torch.cat(parts).contiguous()
            pc = torch.stack([self._dev(p[2], torch.float32).reshape(3) for p in props]).contiguous()
            if prop_visible is not None:
                vis = self._dev(prop_visible, torch.uint8)
                if vis.shape != (B, n):
                    raise ValueError(f"prop_visible must be [B, props] = [{B},{n}], got {tuple(vis.shape)}")
        va = vb = None
        if view_alpha is not None:
            va = self._dev(view_alpha, torch.float32).reshape(-1)
            if va.shape[0] != B:
                raise ValueError(f"view_alpha must hold {B} values")
        if view_background is not None:
            vb = self._dev(view_background, torch.int32).reshape(-1)
            if vb.shape[0] != B:
                raise ValueError(f"view_background must hold {B} image indices")
        keep += [topo, pv, pc, vis, va, vb]
        p = lambda t: t.data_ptr() if t is not None else None
        return _lib.RenderExtra(n, topo.data_ptr(), p(pv), p(pc), p(vis), p(va), p(vb)), keep

    def glyph_props(self):
        """The device props of `camera_glyph()` for a renderer created with its topologies (the first three)."""
        if self._glyph is None:
            topo, meshes = camera_glyph()
            if len(self.topologies) < 3 or any(not np.array_equal(self.topologies[i].numpy(), topo[i])
                                               for i in range(3)):
                raise ValueError("this renderer was not created with camera_glyph()'s topologies")
            self._glyph = [(t, torch.as_tensor(v, dtype=torch.float32).to(self.device),
                            torch.tensor(c, dtype=torch.float32).to(self.device)) for t, v, c in meshes]
            self._palette = torch.tensor(PALETTE, dtype=torch.float32).to(self.device)
        return self._glyph

    def render_views(self, t: dict, photos_u8, K, *, orbit=None, side: bool = False, alpha: float = 0.8,
                     colors=None, closest_first: bool = False, intensity: float = 3.0, metallic: float = 0.0,
                     roughness: float = 0.5, smooth: bool = True, depth: bool = False, index: bool = False) -> dict:
        """The demo's views of a `forward_raw` output dict `t` (v3d, det_idx, count, transl_pelvis; with
        `closest_first` also transl, Anny's order) over B photos (uint8 [B,H,W,3]) with their intrinsics K [B,3,3],
        from one pose launch and one render call, without reading anything back.  Returns device tensors:
        'overlay' [B,H,W,3] (the photos, demo.py overlay_human_meshes at `alpha`); with orbit=(n_frames,
        angle_range) 'orbit' [B, 3 n_frames, H, W, 3] (sweeps y +range, y -range, x +range over white, demo.py:160-241)
        and 'frame_order', the frames of `create_rotating_video` as indices into [overlay] + orbit frames; with
        `side`, 'side' [B,3,H,W,3] (displaced, side and bird's-eye views with the camera glyph at alpha 1 over white,
        utils/render.py:407); 'nonempty' [B] uint8 (an image without persons has no rotating video and plain
        white side views); 'pose' [B, views per image, 3, 4]; 'rank' [P] (position in the image's person list, whose
        palette colour the person gets unless `colors` [P,3] is given); with `depth` / `index`, those maps of every
        view [B, views per image, H, W] (index: person p, or P + j for glyph part j)."""
        dev = self.device
        if side and len(self.topologies) < 3:
            raise ValueError("side views draw the camera glyph: create the Renderer with camera_glyph()'s topologies")
        if not torch.is_tensor(photos_u8) or photos_u8.dtype != torch.uint8 or photos_u8.ndim != 4 \
                or photos_u8.shape[3] != 3:
            raise ValueError("photos_u8 must be a uint8 tensor [B,H,W,3]")
        B, H, W = (int(s) for s in photos_u8.shape[:3])
        K = self._dev(K, torch.float32)
        if K.shape != (B, 3, 3):
            raise ValueError(f"K must be [B,3,3] = [{B},3,3], got {tuple(K.shape)}")
        nf, ar = 0, 0.0
        if orbit is not None:
            nf, ar = int(orbit[0]), float(orbit[1])
            if nf < 2:
                raise ValueError(f"n_frames must be at least 2, got {nf}")
        verts = self._dev(t["v3d"], torch.float32)
        P = int(verts.shape[0])
        if verts.ndim != 3 or verts.shape[1:] != (self.num_verts, 3):
            raise ValueError(f"v3d must be [P,{self.num_verts},3], got {tuple(verts.shape)}")
        Pm = max(P, 1)
        if P == 0:
            verts = torch.zeros(1, self.num_verts, 3, device=dev)
        person_image = self._dev(t["det_idx"][0] if P else torch.zeros(1), torch.int32)
        count = self._dev(t["count"], torch.int32) if P else torch.zeros(1, dtype=torch.int32, device=dev)
        tp = self._dev(t["transl_pelvis"], torch.float32).reshape(-1, 3) if P and side else None
        tr = self._dev(t["transl"], torch.float32).reshape(-1, 3) if P and closest_first else None
        vpi = 1 + 3 * nf + (3 if side else 0)
        pose = torch.empty(B, vpi, 3, 4, dtype=torch.float32, device=dev)
        nonempty = torch.empty(B, dtype=torch.uint8, device=dev)
        rank = torch.empty(Pm, dtype=torch.int32, device=dev)
        if side and P and tp is None:
            raise ValueError("the side views need t['transl_pelvis']")
        pa = _lib.RenderPoseArgs(B, Pm, self.num_verts, count.data_ptr(), person_image.data_ptr(), verts.data_ptr(),
                                 tp.data_ptr() if tp is not None else None, tr.data_ptr() if tr is not None else None,
                                 nf, ar, int(bool(side)), pose.data_ptr(), nonempty.data_ptr(), rank.data_ptr())
        with torch.cuda.device(dev):
            check(self._lib.mhmr_render_view_poses(ctypes.byref(pa), _stream(dev)), "mhmr_render_view_poses")
        if colors is None:
            if self._palette is None:
                self._palette = torch.tensor(PALETTE, dtype=torch.float32).to(dev)
            colors = self._palette[rank.clamp_min(0).long() % len(PALETTE)]
        colors = self._dev(colors, torch.float32)
        if colors.shape != (Pm, 3) and not (P == 0 and colors.shape[1:] == (3,)):
            raise ValueError(f"colors must be [P,3] = [{P},3]")
        photos = photos_u8.to(dev)
        images = torch.cat([photos, torch.full((1, H, W, 3), 255, dtype=torch.uint8, device=dev)]).contiguous()
        views = B * vpi
        vi = torch.arange(B, dtype=torch.int32, device=dev).repeat_interleave(vpi)
        kind = torch.arange(vpi, device=dev).repeat(B)                       # 0 overlay, 1..3nf orbit, then side
        background = torch.where(kind == 0, vi, torch.full_like(vi, B))
        view_alpha = torch.where(kind > 3 * nf, torch.ones(views, device=dev), torch.full((views,), float(alpha),
                                                                                           device=dev))
        props, vis = [], None
        if side:
            props = self.glyph_props()
            vis = ((kind > 3 * nf) & (nonempty.repeat_interleave(vpi) > 0)).to(torch.uint8)[:, None]
            vis = vis.expand(views, len(props)).contiguous()
        extra = self._extra(views, B + 1, props, vis, view_alpha, background)
        Kv = K.repeat_interleave(vpi, 0).contiguous()
        out = self._launch(views, H, W, images, vi, Kv, pose.reshape(views, 3, 4), verts, Pm, person_image, count,
                           colors.contiguous(), alpha, intensity, metallic, roughness, smooth, depth, index, extra)
        o = out["overlay"].reshape(B, vpi, H, W, 3)
        res = {"overlay": o[:, 0], "nonempty": nonempty, "pose": pose, "rank": rank}
        for k in ("depth", "index"):
            if k in out:
                res[k] = out[k].reshape(B, vpi, H, W)
        if nf:
            res["orbit"] = o[:, 1:1 + 3 * nf]
            c = [0] * (nf // 4)
            sweeps = [[1 + s * nf + i for i in range(nf)] for s in range(3)]
            res["frame_order"] = (c + sweeps[0] + sweeps[0][::-1][1:-1] + c + sweeps[1] + sweeps[1][::-1][1:-1] + c
                                  + sweeps[2] + sweeps[2][::-1][1:-1] + c)
        if side:
            res["side"] = o[:, 1 + 3 * nf:]
        return res

    def render_outputs(self, t: dict, images, K, colors=None, **kw) -> dict:
        """Renders the persons of one `Model.forward_raw` / `ModelAnny.forward_raw` output dict `t` into their own
        images (uint8 [B,H,W,3] with intrinsics K [B,3,3] for that resolution): vertices `t['v3d']`, images
        `t['det_idx'][0]`, count `t['count']` read on the device, so this can be enqueued right behind the forward."""
        return self.render(t["v3d"], K, images, person_image=t["det_idx"][0], count=t["count"], colors=colors, **kw)

    def _dev(self, x, dtype):
        x = torch.as_tensor(x)
        return x.to(self.device, dtype=dtype).contiguous()


_CACHE: dict = {}


def _np_faces(f) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(f.cpu() if torch.is_tensor(f) else f).astype(np.int32))


def renderer_for(faces, num_verts: int, device="cuda", topologies=()) -> Renderer:
    """A cached Renderer per (faces, vertex count, extra topologies, device)."""
    f = _np_faces(faces)
    topo = [_np_faces(t) for t in topologies]
    key = (hashlib.sha1(f.tobytes()).hexdigest(), f.shape, int(num_verts), str(torch.device(device)),
           tuple((hashlib.sha1(t.tobytes()).hexdigest(), t.shape) for t in topo))
    r = _CACHE.get(key)
    if r is None:
        if len(_CACHE) >= 8:
            _CACHE.pop(next(iter(_CACHE)))
        r = _CACHE[key] = Renderer(f, device, num_verts=num_verts, topologies=topo or None)
    return r


def _as_u8_image(img) -> np.ndarray:
    a = np.asarray(img)
    if a.ndim != 3 or a.shape[2] != 3:
        raise ValueError(f"img must be [H,W,3], got {a.shape}")
    if a.dtype == np.uint8:
        return a
    if not np.issubdtype(a.dtype, np.floating) and not np.issubdtype(a.dtype, np.integer):
        raise ValueError(f"unsupported image dtype {a.dtype}")
    if not (np.all(a == np.round(a)) and a.min() >= 0 and a.max() <= 255):
        raise ValueError("a non-uint8 image must hold integral values in [0, 255]")
    return a.astype(np.uint8)


def render_meshes(img, l_mesh, l_face, cam_param, color=None, alpha=1.0, show_camera=False, intensity=3.0,
                  metallicFactor=0., roughnessFactor=0.5, smooth=True, device="cuda"):
    """reference utils/render.py:175: the meshes `l_mesh` (list of [V,3], numpy or torch) with faces `l_face` (one
    face array per mesh) rendered with `cam_param` {'focal', 'princpt', optional 'R', 't'} and blended over `img`
    [H,W,3]; returns uint8 [H,W,3] (numpy).  `color=None` draws random colours as the reference does.  Meshes with
    the first mesh's faces are drawn as persons, the others (at most 16) as props of their own topology.
    `show_camera=True` raises NotImplementedError here: the camera glyph is drawn by `render_side_views` (and
    `Renderer.render_views(side=True)`), whose poses place it as the reference does."""
    if show_camera:
        raise NotImplementedError("show_camera: the camera glyph is drawn by render_side_views / "
                                  "Renderer.render_views(side=True)")
    base = _as_u8_image(img)
    n = len(l_mesh)
    cols = []
    for i in range(n):
        if color is None:
            cols.append((np.random.choice(range(1, 225)) / 255, np.random.choice(range(1, 225)) / 255,
                         np.random.choice(range(1, 225)) / 255))
        elif isinstance(color, list):
            cols.append(color[i])
        elif isinstance(color, tuple):
            cols.append(color)
        else:
            raise NotImplementedError
    if n == 0:
        return base.copy()
    f0 = _np_faces(l_face[0])
    nv0 = int(np.asarray(l_mesh[0].shape)[0])
    persons, topo, props = [], [], []
    for i in range(n):
        fi = _np_faces(l_face[i])
        if np.array_equal(fi, f0) and int(l_mesh[i].shape[0]) == nv0:
            persons.append(i)
            continue
        k = next((j for j, t in enumerate(topo) if np.array_equal(t, fi)), None)
        if k is None:
            topo.append(fi)
            k = len(topo) - 1
        props.append((k, i))
    dev = torch.device(device)
    verts = torch.stack([torch.as_tensor(l_mesh[i]).to(dev, torch.float32) for i in persons])
    r = renderer_for(f0, verts.shape[1], dev, topo)
    prop_list = [(k, torch.as_tensor(l_mesh[i]).to(dev, torch.float32), cols[i]) for k, i in props] or None
    cols = [cols[i] for i in persons]
    focal, princpt = np.asarray(cam_param["focal"], np.float64), np.asarray(cam_param["princpt"], np.float64)
    K = torch.tensor([[[focal[0], 0, princpt[0]], [0, focal[1], princpt[1]], [0, 0, 1]]], dtype=torch.float32)
    pose = None
    if "R" in cam_param or "t" in cam_param:
        pose = np.zeros((1, 3, 4))
        pose[0, :, :3] = np.asarray(cam_param["R"]) if "R" in cam_param else np.eye(3)
        pose[0, :, 3] = np.asarray(cam_param["t"]).reshape(3) if "t" in cam_param else 0.0
    out = r.render(verts, K, torch.from_numpy(np.ascontiguousarray(base))[None].to(dev), pose=pose,
                   colors=torch.tensor(np.asarray(cols, np.float64), dtype=torch.float32), alpha=alpha,
                   intensity=intensity, metallic=metallicFactor, roughness=roughnessFactor, smooth=smooth,
                   props=prop_list)
    return out["overlay"][0].cpu().numpy()


def _humans_dict(humans, dev, name="v3d"):
    """One image's person list (Model.forward / ModelAnny.forward) as a forward_raw-like dict, list order kept, with
    the vertices of key `name`."""
    P = len(humans)
    t = {"v3d": torch.stack([torch.as_tensor(h[name]).to(dev, torch.float32) for h in humans]),
         "det_idx": torch.zeros(3, P, dtype=torch.int32, device=dev),
         "count": torch.full((1,), P, dtype=torch.int32, device=dev)}
    if all("transl_pelvis" in h for h in humans):
        t["transl_pelvis"] = torch.stack([torch.as_tensor(h["transl_pelvis"]).to(dev, torch.float32).reshape(3)
                                          for h in humans])
    return t


def _person_colors(_color, n):
    if isinstance(_color, tuple):
        return [_color] * n
    if isinstance(_color, list):
        return [_color[i] for i in range(n)]
    raise NotImplementedError


def render_side_views(img_array, _color, humans, model, K, faces, device="cuda"):
    """reference utils/render.py:407: the displaced, side and bird's-eye views of one image's persons (list of
    dicts with 'v3d' and 'transl_pelvis') with the camera glyph, over white at alpha 1, with the focal and principal
    point of K[0].  Returns three uint8 [H,W,3] arrays; without persons, the reference's three white float arrays."""
    img_array = np.asarray(img_array)
    if len(humans) == 0:
        bg = 1 + 0. * img_array.copy()
        return 255.0 * bg.copy(), 255.0 * bg.copy(), 255.0 * bg.copy()
    dev = torch.device(device)
    H, W = img_array.shape[:2]
    t = _humans_dict(humans, dev)
    topo, _ = camera_glyph()
    r = renderer_for(faces, t["v3d"].shape[1], dev, topo)
    cols = torch.tensor(np.asarray(_person_colors(_color, len(humans)), np.float64)[:, :3], dtype=torch.float32)
    white = torch.full((1, H, W, 3), 255, dtype=torch.uint8, device=dev)
    out = r.render_views(t, white, torch.as_tensor(K)[:1], side=True, alpha=1.0, colors=cols)
    s = out["side"][0].cpu().numpy()
    return s[0], s[1], s[2]
