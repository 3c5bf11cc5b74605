"""The premises of the bulk-pass accuracy rule (tests/vit_bulk_util.py), checked on the CPU at ViT-S 224: the rounding
model is the exact forward once its roundings are switched off, another accumulation order of it passes the rule, and
each planted mistake fails it."""
import pytest
import torch

import vit_bulk_util as vb

NAME = "dinov2_vits14"
TAPS = (1, 6, 12)


def _reference(case_name):
    torch.set_num_threads(min(16, torch.get_num_threads()))
    case, sd, _, x = vb.build(case_name, 224, 1)
    sd64 = vb.backbone64(sd, 224)
    x64 = x.double()
    with torch.no_grad():
        ex = vb.exact(x64, sd64, NAME, TAPS)
        emu = vb.emulate(x64, sd64, NAME, "fold", TAPS)
    return x, sd64, ex, emu


@pytest.fixture(scope="module")
def refs():
    return {c: _reference(c) for c in ("s_224_S_forced", "s_224_S_outliers")}


@pytest.fixture(scope="module")
def ref(refs):
    return refs["s_224_S_forced"]


def _pairs(got, ex):
    """(label, got, exact) for the stream taps and the final features."""
    return [(f"after {l} blocks", got[0][l], ex[0][l]) for l in TAPS] + [("features", got[1], ex[1])]


@pytest.mark.parametrize("mode", ["fold", "sep"])
def test_model_without_rounding_is_the_exact_forward(ref, mode):
    """With no rounding point left the folded LayerNorm (centred W', b + W beta, statistics of the raw stream) is the
    same algebra as dinov2_ref: the two agree to fp64 noise."""
    x, sd64, ex, _ = ref
    with torch.no_grad(), vb.rounding_off():
        got = vb.emulate(x.double(), sd64, NAME, mode, TAPS)
    for label, g, e in _pairs(got, ex):
        err = (g - e).abs().max().item()
        print(f"  {mode} {label}: max |model - exact| {err:.2e}")
        assert err < 1e-10, (label, err)


def test_fp32_accumulation_of_the_model_passes_the_rule(ref):
    """The same rounding model summed in fp32 by the CPU's BLAS, in its own order, stands in for the engine."""
    x, sd64, ex, emu = ref
    sd32 = {k: v.float() for k, v in sd64.items()}
    with torch.no_grad():
        got = vb.emulate(x, sd32, NAME, "fold", TAPS)
    for (label, g, e), (_, m, _) in zip(_pairs(got, ex), _pairs(emu, ex)):
        r, glob = vb.row_ratios(g, m, e)
        vb.describe(f"fp32 model, {label}", r, glob)
        assert vb.passes(r, glob), label


def test_outlier_rows_break_the_premise_of_the_per_row_rule(refs):
    """At the outlier weights the model accumulated in fp32 is itself outside the per-row rule on a few rows (their
    error is made of a handful of fp16 roundings of the outlier channels), while its median and global ratios stay at
    1: on that case the engine is held to the median and global ratios, its per-row maximum is an open finding
    (test_vit_bulk_gpu.py)."""
    x, sd64, ex, emu = refs["s_224_S_outliers"]
    sd32 = {k: v.float() for k, v in sd64.items()}
    with torch.no_grad():
        got = vb.emulate(x, sd32, NAME, "fold", TAPS)
    outside = []
    for (label, g, e), (_, m, _) in zip(_pairs(got, ex), _pairs(emu, ex)):
        r, glob = vb.row_ratios(g, m, e)
        vb.describe(f"fp32 model, outliers, {label}", r, glob)
        outside.append(r.max().item() > vb.R_MAX)
        assert vb.R_GLOBAL[0] <= glob <= vb.R_GLOBAL[1] and r.median().item() < 1.05, label
    assert any(outside)


# (case, mistake).  The planted mistakes that no weights here make fail the rule are listed with vit_bulk_util.MISTAKES.
MISTAKE_CASES = [("s_224_S_forced", "no_lo_plane"), ("s_224_S_outliers", "no_lo_plane"),
                 ("s_224_S_forced", "cls_without_pos0"), ("s_224_S_outliers", "cls_without_pos0")]


@pytest.mark.parametrize("case_name,mistake", MISTAKE_CASES)
def test_planted_mistakes_fail_the_rule(refs, case_name, mistake):
    """Each mistake fails the rule on the final features (the cls one, which the features drop, on the stream after
    the last block); the rounding-sized mistake of dropping the lo plane puts even the median row outside it at every
    tap."""
    x, sd64, ex, emu = refs[case_name]
    got = vb.planted_model(x, sd64, NAME, mistake, TAPS)
    last = None
    for (label, g, e), (_, m, _) in zip(_pairs(got, ex), _pairs(emu, ex)):
        r, glob = vb.row_ratios(g, m, e)
        vb.describe(f"{case_name} {mistake}, {label}", r, glob)
        if mistake == "no_lo_plane":
            assert r.median().item() > vb.R_MAX, label
        if label != "features" or mistake != "cls_without_pos0":
            last = (label, vb.passes(r, glob))
    assert last[1] is False, last
