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


class Renderer:
    """A renderer for one face array [F,3] (int, indices < num_verts) on one CUDA device.  The handle builds the
    vertex -> face table of the normal pass once and owns the depth-key buffer (8 B per pixel per view)."""

    def __init__(self, faces, device="cuda", num_verts: int | None = None):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("the renderer runs on a CUDA device (no CPU fallback)")
        f = torch.as_tensor(np.asarray(faces) if not torch.is_tensor(faces) else faces)
        if f.ndim != 2 or f.shape[1] != 3 or f.shape[0] < 1:
            raise ValueError(f"faces must be [F,3], got {tuple(f.shape)}")
        if f.dtype.is_floating_point:
            raise ValueError("faces must be integers")
        f = f.to(torch.int64)
        V = int(num_verts) if num_verts is not None else int(f.max()) + 1
        self.device, self.num_faces, self.num_verts = dev, int(f.shape[0]), V
        self.faces = f.to(torch.int32).cpu().contiguous()
        self._lib = _lib.load()
        h = c_void_p()
        with torch.cuda.device(dev):
            check(self._lib.mhmr_render_create(ptr(self.faces), self.num_faces, V, _stream(dev), ctypes.byref(h)),
                  "mhmr_render_create")
        self._h = h
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
               smooth: bool = True, depth: bool = False, index: bool = False) -> dict:
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
            check(self._lib.mhmr_render_forward(self._h, ctypes.byref(args), _stream(dev)), "mhmr_render_forward")
        return {k: v for k, v in out.items() if v is not None}

    def render_outputs(self, t: dict, images, K, colors=None, **kw) -> dict:
        """Renders the persons of one `Model.forward_raw` / `ModelAnny.forward_raw` output dict `t` into their own
        images (uint8 [B,H,W,3] with intrinsics K [B,3,3] for that resolution): vertices `t['v3d']`, images
        `t['det_idx'][0]`, count `t['count']` read on the device, so this can be enqueued right behind the forward."""
        return self.render(t["v3d"], K, images, person_image=t["det_idx"][0], count=t["count"], colors=colors, **kw)

    def _dev(self, x, dtype):
        x = torch.as_tensor(x)
        return x.to(self.device, dtype=dtype).contiguous()


_CACHE: dict = {}


def renderer_for(faces, num_verts: int, device="cuda") -> Renderer:
    """A cached Renderer per (faces, vertex count, device)."""
    f = np.ascontiguousarray(np.asarray(faces.cpu() if torch.is_tensor(faces) else faces).astype(np.int32))
    key = (hashlib.sha1(f.tobytes()).hexdigest(), f.shape, int(num_verts), str(torch.device(device)))
    r = _CACHE.get(key)
    if r is None:
        if len(_CACHE) >= 8:
            _CACHE.pop(next(iter(_CACHE)))
        r = _CACHE[key] = Renderer(f, device, num_verts=num_verts)
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
    face array shared by all meshes) rendered with `cam_param` {'focal', 'princpt', optional 'R', 't'} and blended
    over `img` [H,W,3]; returns uint8 [H,W,3] (numpy).  `color=None` draws random colours as the reference does."""
    if show_camera:
        raise NotImplementedError("show_camera draws pyvista glyphs, which this renderer does not provide")
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
    f0 = np.asarray(l_face[0].cpu() if torch.is_tensor(l_face[0]) else l_face[0])
    for f in l_face[1:n]:
        if not np.array_equal(np.asarray(f.cpu() if torch.is_tensor(f) else f), f0):
            raise ValueError("render_meshes here takes one face array shared by every mesh")
    dev = torch.device(device)
    verts = torch.stack([torch.as_tensor(m).to(dev, torch.float32) for m in l_mesh])
    r = renderer_for(f0, verts.shape[1], dev)
    focal, princpt = np.asarray(cam_param["focal"], np.float64), np.asarray(cam_param["princpt"], np.float64)
    K = torch.tensor([[[focal[0], 0, princpt[0]], [0, focal[1], princpt[1]], [0, 0, 1]]], dtype=torch.float32)
    pose = None
    if "R" in cam_param or "t" in cam_param:
        pose = np.zeros((1, 3, 4))
        pose[0, :, :3] = np.asarray(cam_param["R"]) if "R" in cam_param else np.eye(3)
        pose[0, :, 3] = np.asarray(cam_param["t"]).reshape(3) if "t" in cam_param else 0.0
    out = r.render(verts, K, torch.from_numpy(np.ascontiguousarray(base))[None].to(dev), pose=pose,
                   colors=torch.tensor(np.asarray(cols, np.float64), dtype=torch.float32), alpha=alpha,
                   intensity=intensity, metallic=metallicFactor, roughness=roughnessFactor, smooth=smooth)
    return out["overlay"][0].cpu().numpy()
