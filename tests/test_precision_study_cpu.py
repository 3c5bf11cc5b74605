"""The CPU precision studies (tools/precision_study.py) on a ViT-S golden case: the default rounding-point mode and
the FP8-MLP study both run end to end and report what DESIGN.md §3 records for that case."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import precision_study as ps  # noqa: E402


def test_default_mode_reports_the_emulated_engine_error():
    res = ps.run("s_224_S_forced", lambda sd: iter([("all-rounded", ps.Emu(sd)), ("none", ps.Emu(sd, default="n"))]))
    assert set(res) == {"all-rounded", "none"}
    v3d_rounded, v3d_fp32 = res["all-rounded"]["v3d"][0], res["none"]["v3d"][0]
    assert v3d_fp32 < 1e-5                   # no rounding point: the oracle itself
    assert 1e-5 < v3d_rounded < 1e-3         # fp16 operands: a measurable error inside the 1e-3 contract


def test_fp8_study_reports_fp16_and_fp8_with_and_without_refinement():
    res = ps.fp8_study("s_224_S_forced")
    assert set(res) == {(v, r) for v in ps.FP8_VARIANTS for r in (False, True)}
    assert all(persons == 5 and same for persons, same, _ in res.values())
    v3d = {key: e["v3d"] for key, (_, _, e) in res.items()}
    assert v3d[("fp16", True)] < 1e-4 < v3d[("fp8 fc1+fc2", True)] < v3d[("fp8 fc1+fc2", False)]
    # DESIGN.md §3 table: 4.6e-3 with MKL's AVX-512 kernels.  Its SSE4.2 and AVX2 kernels sum the fp32 products in
    # other orders, which flips some e4m3 roundings: 4.77e-3 and 4.91e-3.  The band holds all three with ~6% margin.
    assert 4.3e-3 < v3d[("fp8 fc1+fc2", True)] < 5.2e-3
