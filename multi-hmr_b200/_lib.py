"""ctypes binding of libmhmr_sm90.so (the C-ABI declared in include/mhmr.h).

The library is built in-tree by build.py.  Importing this module never falls back to another
implementation: if the shared object is missing it is (re)built, and if that fails the import raises.
"""
from __future__ import annotations

import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmhmr_sm90.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "mhmr.h")

c_void_p, c_int, c_int64, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float

_lib = None


class MhmrError(RuntimeError):
    pass


def declared_symbols() -> list[str]:
    """Function names declared in include/mhmr.h (used by the export test)."""
    text = open(HEADER_PATH).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mhmr_[a-z0-9_]+)\s*\(", text)))


def load() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        import importlib.util

        spec = importlib.util.spec_from_file_location("_mhmr_build", os.path.join(_HERE, "build.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.build()
    lib = ctypes.CDLL(LIB_PATH)
    lib.mhmr_last_error.restype = ctypes.c_char_p
    lib.mhmr_last_error.argtypes = []
    _declare_render(lib)
    _lib = lib
    return lib


class RenderArgs(ctypes.Structure):
    """`mhmr_render_args` of include/mhmr.h."""

    _fields_ = [("views", c_int), ("H", c_int), ("W", c_int), ("images", c_void_p), ("view_image", c_void_p),
                ("K", c_void_p), ("pose", c_void_p), ("verts", c_void_p), ("max_persons", c_int),
                ("person_image", c_void_p), ("count", c_void_p), ("colors", c_void_p), ("alpha", c_float),
                ("intensity", c_float), ("metallic", c_float), ("roughness", c_float), ("smooth", c_int),
                ("overlay", c_void_p), ("depth", c_void_p), ("person", c_void_p)]


class RenderExtra(ctypes.Structure):
    """`mhmr_render_extra` of include/mhmr.h."""

    _fields_ = [("num_props", c_int), ("prop_topology", c_void_p), ("prop_verts", c_void_p),
                ("prop_colors", c_void_p), ("prop_visible", c_void_p), ("view_alpha", c_void_p),
                ("view_background", c_void_p)]


class RenderPoseArgs(ctypes.Structure):
    """`mhmr_render_pose_args` of include/mhmr.h."""

    _fields_ = [("images", c_int), ("max_persons", c_int), ("num_verts", c_int), ("count", c_void_p),
                ("person_image", c_void_p), ("verts", c_void_p), ("transl_pelvis", c_void_p), ("transl", c_void_p),
                ("n_frames", c_int), ("angle_range", ctypes.c_double), ("side", c_int), ("pose", c_void_p),
                ("nonempty", c_void_p), ("rank", c_void_p)]


def _declare_render(lib) -> None:
    P = ctypes.POINTER
    lib.mhmr_render_create.argtypes = [c_void_p, c_int, c_int, c_void_p, P(c_void_p)]
    lib.mhmr_render_create_topologies.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                                  c_void_p, P(c_void_p)]
    lib.mhmr_render_destroy.argtypes = [c_void_p]
    lib.mhmr_render_info.argtypes = [c_void_p, P(c_int), P(c_int), P(c_int)]
    lib.mhmr_render_forward.argtypes = [c_void_p, P(RenderArgs), c_void_p]
    lib.mhmr_render_forward_extra.argtypes = [c_void_p, P(RenderArgs), P(RenderExtra), c_void_p]
    lib.mhmr_render_view_poses.argtypes = [P(RenderPoseArgs), c_void_p]
    for f in (lib.mhmr_render_create, lib.mhmr_render_create_topologies, lib.mhmr_render_destroy,
              lib.mhmr_render_info, lib.mhmr_render_forward, lib.mhmr_render_forward_extra,
              lib.mhmr_render_view_poses):
        f.restype = c_int


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().mhmr_last_error().decode("utf-8", "replace")
        exc = MhmrError if rc != -2 else AssertionError
        raise exc(f"{what} failed (code {rc}): {msg}")


def ptr(t) -> c_void_p:
    """Device (or host) pointer of a torch tensor / None."""
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def stream_ptr() -> c_void_p:
    import torch

    return c_void_p(torch.cuda.current_stream().cuda_stream)
