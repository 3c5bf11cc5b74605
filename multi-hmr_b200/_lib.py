"""ctypes binding of libmhmr_sm90.so, derived from the C-ABI declared in include/mhmr.h.

The header is parsed once: every prototype gets exact `argtypes` / `restype`, and every `typedef struct` becomes a
ctypes structure with the header's field names, types and order.  `call(name, *args)` is the checked way in; the typed
library of `load()` stays reachable for callers that want a raw status code.  The names of the hand-written binding this
replaced (`check`, `ptr` and the ctypes scalar types) still work against the typed library.

The library is built in-tree by build.py.  Loading never falls back to another implementation: if the shared object
is missing it is (re)built, and if that fails, or the header declares a C type this binding cannot map, load() raises.
"""
from __future__ import annotations

import ctypes
import os
import re
from ctypes import c_float, c_int, c_int64, c_void_p  # noqa: F401  (the previous binding's names)

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmhmr_sm90.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "mhmr.h")

# entries whose return value is a result, not a status code
VALUE_RETURNS = frozenset(("mhmr_last_error", "mhmr_last_launch_count", "mhmr_record_floats",
                           "mhmr_record_block_bytes"))
_SCALARS = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "float": ctypes.c_float, "double": ctypes.c_double}
_RETURNS = {("int", 0): ctypes.c_int, ("int64_t", 0): ctypes.c_int64, ("char", 1): ctypes.c_char_p}

_lib = None
_header = None


class MhmrError(RuntimeError):
    pass


class Pointer:
    """The argtype of every pointer parameter that is not a pointer to one of the header's structs: data, opaque
    handles, `handle**` and `int*` out-params, `void* stream`.  Takes None, an address, a torch tensor (its
    data_ptr()) or whatever c_void_p takes (ctypes arrays, byref(), c_void_p, bytes) except str."""

    @classmethod
    def from_param(cls, obj):
        if isinstance(obj, torch.Tensor):
            obj = obj.data_ptr()
        elif isinstance(obj, str):
            raise TypeError("a str is not a pointer (pass bytes)")
        return ctypes.c_void_p.from_param(obj)


class Struct(ctypes.Structure):
    """Base of the structs generated from the header: built by keyword, unknown field names are an error, pointer
    fields take a torch tensor (its data_ptr()), an address or None.  Positional values follow the header's field
    order, as in any ctypes structure."""

    def __init__(self, *values, **fields):
        types = dict(self._fields_)
        unknown = sorted(set(fields) - set(types))
        if unknown:
            raise TypeError(f"{type(self).__name__} has no field {', '.join(unknown)}")
        super().__init__(*values, **{k: v.data_ptr() if isinstance(v, torch.Tensor) and types[k] is ctypes.c_void_p
                                     else v for k, v in fields.items()})

    @classmethod
    def field_names(cls) -> tuple[str, ...]:
        return tuple(n for n, _ in cls._fields_)


def _declarators(decl: str, what: str) -> list[tuple[str, int, str]]:
    """A C declaration -> [(base type, pointer depth, name)], one per declarator: `int views, H, W` gives three,
    `const float* bias` gives ('float', 1, 'bias')."""
    m = re.fullmatch(r"\s*(?:const\s+)?(\w+)(.*?)\s*", decl, re.S)
    out = []
    for d in (m.group(2).split(",") if m else [None]):
        dm = d is not None and re.fullmatch(r"\s*(\**)\s*(?:const\s+)?(\w+)\s*", d)
        if not dm:
            raise TypeError(f"{what}: cannot parse the C declaration {decl.strip()!r}")
        out.append((m.group(1), len(dm.group(1)), dm.group(2)))
    return out


def _ctype(base: str, depth: int, structs: dict, what: str, field: bool = False):
    if depth == 0 and base in _SCALARS:
        return _SCALARS[base]
    if depth and field:
        return ctypes.c_void_p
    if depth == 1 and base in structs:
        return ctypes.POINTER(structs[base])
    if depth:
        return Pointer
    raise TypeError(f"{what}: no ctypes type for the C type {base!r}")


def _parse():
    """({struct name: Struct subclass}, {function name: (restype, argtypes)}) of include/mhmr.h."""
    global _header
    if _header is None:
        text = re.sub(r"/\*.*?\*/|//[^\n]*", "", open(HEADER_PATH).read(), flags=re.S)
        text = re.sub(r"^\s*#.*$", "", text, flags=re.M)
        struct_re = r"typedef\s+struct\s+\w+\s*\{([^}]*)\}\s*(\w+)\s*;"
        structs = {}
        for body, name in re.findall(struct_re, text):
            fields = [(n, _ctype(b, d, structs, name, field=True))
                      for decl in body.split(";") if decl.strip() for b, d, n in _declarators(decl, name)]
            structs[name] = type(name, (Struct,), {"_fields_": fields})
        protos = {}
        for stmt in re.split(r"[;{}]", re.sub(struct_re, "", text)):
            if "(" not in stmt:
                continue
            m = re.fullmatch(r"([^()]*)\(([^()]*)\)\s*", stmt)
            if m is None:
                raise TypeError(f"cannot parse the declaration {stmt.strip()!r}")
            [(rbase, rdepth, name)] = _declarators(m.group(1), "prototype")
            if (rbase, rdepth) not in _RETURNS:
                raise TypeError(f"{name}: no ctypes type for its return type")
            params = [] if m.group(2).strip() in ("", "void") else [
                _ctype(*_declarators(p, name)[0][:2], structs, name) for p in m.group(2).split(",")]
            protos[name] = (_RETURNS[rbase, rdepth], params)
        _header = structs, protos
    return _header


def declared_symbols() -> list[str]:
    """Function names declared in include/mhmr.h."""
    return sorted(_parse()[1])


def structs() -> dict:
    """{name: Struct subclass} of the header's `typedef struct`s."""
    return _parse()[0]


def struct(name: str, **fields) -> Struct:
    """An instance of the header's struct `name` (e.g. 'mhmr_config'), built by keyword."""
    return structs()[name](**fields)


def load() -> ctypes.CDLL:
    """The library with every declared function typed from the header."""
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
    for name, (restype, argtypes) in _parse()[1].items():
        f = getattr(lib, name)
        f.restype, f.argtypes = restype, argtypes
    _lib = lib
    return lib


def call(name: str, *args):
    """Calls the entry `name` with exactly its declared arguments.  A status code != 0 raises: AssertionError for
    MHMR_ERR_ARG (as the reference asserts on bad arguments), MhmrError otherwise, with mhmr_last_error()'s message.
    The entries of VALUE_RETURNS return their value unchecked."""
    f = getattr(load(), name)
    if len(args) != len(f.argtypes):
        raise TypeError(f"{name} takes {len(f.argtypes)} arguments ({len(args)} given)")
    rc = f(*args)
    if name not in VALUE_RETURNS:
        check(rc, name)
    return rc


def check(rc: int, what: str = "") -> None:
    """Raises for a status code != 0: AssertionError for MHMR_ERR_ARG, MhmrError otherwise."""
    if rc != 0:
        msg = load().mhmr_last_error().decode("utf-8", "replace")
        raise (AssertionError if rc == -2 else MhmrError)(f"{what} failed (code {rc}): {msg}")


def ptr(t) -> c_void_p:
    """The address of a torch tensor (or NULL for None) as a c_void_p."""
    return c_void_p(0 if t is None else t.data_ptr())


def stream(device=None) -> int:
    """The `void* stream` argument of the current torch CUDA stream of `device` (default: the current device)."""
    return torch.cuda.current_stream(device).cuda_stream
