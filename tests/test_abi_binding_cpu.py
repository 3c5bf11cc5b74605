"""CPU: the ctypes binding derived from include/mhmr.h.  Every prototype is typed with the header's arity and types,
every generated struct has the C compiler's size and field offsets, and wrong calls fail in Python before anything
reaches the library."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from multihmr_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCALARS = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "float": ctypes.c_float, "double": ctypes.c_double}


def _prototypes():
    """{name: [parameter declarations]} read from the header with a plain regex, independently of _lib's parser."""
    text = re.sub(r"/\*.*?\*/", "", open(_lib.HEADER_PATH).read(), flags=re.S)
    out = {}
    for name, params in re.findall(r"\b(mhmr_\w+)\s*\(([^)]*)\)\s*;", text):
        out[name] = [] if params.strip() == "void" else [p.strip() for p in params.split(",")]
    return out


def test_every_prototype_is_typed_from_the_header():
    lib = _lib.load()
    structs = _lib.structs()
    protos = _prototypes()
    assert sorted(protos) == _lib.declared_symbols() and len(protos) >= 60
    for name, params in protos.items():
        f = getattr(lib, name)
        assert len(f.argtypes) == len(params), name
        for decl, t in zip(params, f.argtypes):
            base = re.sub(r"\bconst\b|\*|\w+$", "", decl).strip()
            if "*" not in decl:
                assert t is SCALARS[base], (name, decl)
            elif base in structs and decl.count("*") == 1:
                assert t is ctypes.POINTER(structs[base]), (name, decl)
            else:
                assert t is _lib.Pointer, (name, decl)
        want = {"mhmr_last_error": ctypes.c_char_p, "mhmr_record_block_bytes": ctypes.c_int64}.get(name, ctypes.c_int)
        assert f.restype is want, name


def test_structs_match_the_c_compiler(tmp_path):
    structs = _lib.structs()
    assert set(structs) == {"mhmr_config", "mhmr_outputs", "mhmr_anny_outputs", "mhmr_render_args",
                            "mhmr_render_extra", "mhmr_render_pose_args"}
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "mhmr.h"', "int main(void) {"]
    for name, cls in structs.items():
        lines.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        lines += [f'  printf("{name}.{f} %zu\\n", offsetof({name}, {f}));' for f, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    (tmp_path / "probe.c").write_text("\n".join(lines) + "\n")
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a host C compiler is needed (nvcc needs one to build the library)"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(tmp_path / "probe.c"), "-o", str(tmp_path / "probe")],
                   check=True)
    got = dict(line.split() for line in subprocess.run([str(tmp_path / "probe")], check=True, capture_output=True,
                                                       text=True).stdout.splitlines())
    want = {}
    for name, cls in structs.items():
        want[name] = str(ctypes.sizeof(cls))
        want.update({f"{name}.{f}": str(getattr(cls, f).offset) for f, _ in cls._fields_})
    assert got == want
    assert ctypes.sizeof(structs["mhmr_render_args"]) == 136 and len(structs["mhmr_render_args"]._fields_) == 20


@pytest.mark.parametrize("decl, match", [("int mhmr_extra(unsigned int n);", "mhmr_extra"),
                                         ("char mhmr_extra(int n);", "mhmr_extra"),
                                         ("int mhmr_extra(int32_t n);", "mhmr_extra"),
                                         ("int mhmr_extra(void (*cb)(int));", "mhmr_extra")])
def test_an_unmappable_declaration_is_refused(decl, match, tmp_path, monkeypatch):
    header = tmp_path / "mhmr.h"
    header.write_text(open(_lib.HEADER_PATH).read().replace("#ifdef __cplusplus\n}", decl + "\n#ifdef __cplusplus\n}"))
    monkeypatch.setattr(_lib, "HEADER_PATH", str(header))
    monkeypatch.setattr(_lib, "_header", None)
    with pytest.raises(TypeError, match=match):
        _lib._parse()


def test_struct_constructor_takes_keywords_and_tensors_only_for_known_fields():
    t = torch.zeros(4)
    o = _lib.struct("mhmr_outputs", count=t, v2d=None, z=1234)
    assert o.count == t.data_ptr() and o.v2d is None and o.z == 1234 and o.v3d is None
    with pytest.raises(TypeError, match="img_sise"):
        _lib.struct("mhmr_config", img_sise=896)


def test_calls_fail_loudly_before_the_library_runs():
    lib = _lib.load()
    with pytest.raises(TypeError, match="takes 1 argument"):
        _lib.call("mhmr_destroy")
    with pytest.raises(TypeError, match="takes 6 argument"):
        _lib.call("mhmr_body_info", None, None, None, None, None, None, None)
    with pytest.raises(ctypes.ArgumentError):
        _lib.call("mhmr_record_floats", 10.0, 10475)
    with pytest.raises(ctypes.ArgumentError):
        lib.mhmr_record_floats(10, 10475.0)
    with pytest.raises(ctypes.ArgumentError):
        lib.mhmr_body_info(1.5, None, None, None, None, None)
    with pytest.raises(ctypes.ArgumentError):
        lib.mhmr_body_info("not a pointer", None, None, None, None, None)


def test_pointers_take_tensors_none_and_ints():
    lib = _lib.load()
    n = torch.full((1,), -7, dtype=torch.int32)
    h = torch.zeros(1, dtype=torch.int64)
    for args in ((None, n, 0, None, None, None), (0, None, None, None, None, n)):
        assert lib.mhmr_body_info(*args) == -2
    with pytest.raises(AssertionError, match=r"mhmr_body_info failed \(code -2\): .*null body model"):
        _lib.call("mhmr_body_info", None, n, None, None, None, None)
    assert n.item() == -7
    cfg = _lib.struct("mhmr_config", arch=2, img_size=900, max_batch=1, max_persons=8, xat_depth=2, xat_num_heads=8,
                      num_betas=10, person_center_idx=15, num_verts=10475)
    with pytest.raises(AssertionError, match="img size"):
        _lib.call("mhmr_create", cfg, h)
    assert lib.mhmr_create(ctypes.byref(cfg), h) == -2 and h.item() == 0


def test_value_returns_are_unchecked_and_int64_is_not_truncated():
    R = _lib.call("mhmr_record_floats", 10, 10475)
    assert R == 179 + 10 + 3 * 10475 + 381 + 254
    cap = 100_000
    assert _lib.call("mhmr_record_block_bytes", 10, 10475, cap) == 4 * (8 + cap * R) > 2 ** 31


def test_only_the_binding_declares_ctypes_signatures():
    pattern = re.compile(r"\b(argtypes|restype|_fields_)\b")
    files = [os.path.join(d, f) for top in ("multi-hmr_b200", "tests")
             for d, _, fs in os.walk(os.path.join(ROOT, top)) for f in fs if f.endswith(".py")]
    skip = {os.path.join(ROOT, "multi-hmr_b200", "_lib.py"), os.path.abspath(__file__)}
    offenders = [f for f in files if f not in skip and pattern.search(open(f).read())]
    assert not offenders, offenders
