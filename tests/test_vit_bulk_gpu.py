"""The composed bulk pass (engine.cu::vit_forward: patch embedding, the blocks chained with programmatic dependent
launch, the final norm) against fp64, row by row, through the stage entry mhmr_op_vit_stream:

  (a) the stream after the patch embedding, per element, against its fp64 value and bound;
  (b) the stream after 1, depth/2 and depth blocks and the final features, each token row against the accuracy of
      the engine's own rounding model (tests/vit_bulk_util.py: R_r = rms_r(engine - exact) / rms_r(model - exact));
  (c) bit-equality of a batch position, of stale rows, of images next to a non-finite one, and with PDL off.

The fp32 refinement of the detected tokens (DESIGN.md §3) overwrites their bulk rows, so an error confined to some
rows, layers or images of the bulk pass can pass every output-level test: these check the bulk pass itself."""
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import vit_bulk_util as vb

pytestmark = pytest.mark.gpu

DEPTH = {"dinov2_vits14": 12, "dinov2_vitb14": 12, "dinov2_vitl14": 24}
BIT_CASES = {"S_224": ("s_224_S_forced", 224), "L_896": ("dinov2_vitl14", 896)}


def _taps(name):
    d = DEPTH[name]
    return (1, d // 2, d)


def _pairs(eng, ref, taps):
    return [(f"after {l} blocks", eng[l], ref[0][l]) for l in taps] + [("features", eng["features"], ref[1])]


# Open finding.  At the outlier weights a few token rows of the engine (tokens 88 and 198 of image 0 among them, the same
# rows run after run) are up to 2.1x less accurate than the fp64 rounding model after 6 and 12 blocks, while the median
# and global ratios stay at 1.00-1.01.  The model accumulated in fp32 reaches ~1.7 on such rows (test_vit_bulk_cpu.py):
# part of it is the rule's premise failing on rows whose error is a handful of roundings, but the gap from 1.7 to 2.1 is
# not explained.  Only the per-row maximum is expected to fail there; strict, so that a fix shows up.
_OUTLIER_ROW_MAX = pytest.mark.xfail(raises=vb.RowMaxExceeded, strict=True,
                                     reason="outlier-channel rows up to 2.1x the model's error, 1.7x for its fp32 "
                                            "accumulation; the gap is unexplained (open finding)")
ROW_CASES = [pytest.param(k, "fold", marks=_OUTLIER_ROW_MAX) if k == "s_224_S_outliers" else (k, "fold")
             for k in vb.CASES] + [("s_224_S_forced", "sep"), ("s_280_L_forced", "sep")]


@pytest.mark.parametrize("key,mode", ROW_CASES)
def test_bulk_pass_rows_against_fp64(cuda_device, monkeypatch, key, mode):
    weights, S, B, max_batch = vb.CASES[key]
    case, sd, bm, x = vb.build(weights, S, B)
    name = case["backbone"]
    taps = _taps(name)
    if mode == "sep":
        monkeypatch.setenv("MHMR_LN_FOLD", "0")      # read at mhmr_finalize
    m = vb.engine(case, sd, bm, max_batch)
    monkeypatch.delenv("MHMR_LN_FOLD", raising=False)
    eng = vb.taps_and_features(m, x, (0,) + taps)
    vb.release(m)
    sd64 = vb.backbone64(sd, S, cuda_device)
    x64 = x.to(cuda_device, torch.float64)

    # the path the engine built: the folded one stores the stream as hi + lo, the separate-LayerNorm one in fp32
    two_term = vb.is_two_term(eng[0])
    assert bool(two_term.all()) == (mode == "fold"), (mode, two_term.float().mean().item())

    # (a) the patch embedding, every element of every image
    ref0, tol0 = vb.patch_embed_bound(x64, sd64)
    err0 = (eng[0].double() - ref0).abs()
    worst = (err0 / tol0).max().item()
    print(f"\n{key} [{mode}] B={B}/{max_batch}: patch embedding worst err/tol {worst:.3f}")
    assert torch.isfinite(eng[0]).all() and worst <= 1.0, worst

    # (b) every token row of the taps and the features against the rounding model's accuracy: the global ratio and
    # the median row at 1, then the worst row
    with torch.no_grad():
        ex = vb.exact(x64, sd64, name, taps)
        emu = vb.emulate(x64, sd64, name, mode, taps)
    off, rows = [], []
    for (label, g, e), (_, mm, _) in zip(_pairs(eng, ex, taps), _pairs({**emu[0], "features": emu[1]}, ex, taps)):
        r, glob = vb.row_ratios(g, mm, e)
        vb.describe(f"  {key} [{mode}] {label}", r, glob)
        med = r.median().item()
        if not (vb.R_GLOBAL[0] <= glob <= vb.R_GLOBAL[1] and abs(med - 1.0) <= 0.05):
            off.append((label, glob, med))
        if r.max().item() > vb.R_MAX:
            rows.append((label, r.max().item(), int(r.argmax())))
    assert not off, off
    if rows:
        raise vb.RowMaxExceeded(rows)


@pytest.mark.parametrize("mistake", ["no_lo_plane", "cls_without_pos0"])
def test_planted_mistakes_fail_at_vit_l(cuda_device, mistake):
    """At ViT-L depth (fp64 is cheap on the device) the planted mistakes of test_vit_bulk_cpu.py still fail the rule:
    dropping the lo plane even for the median row, the cls row without pos[0] on its own row."""
    case, sd, _, x = vb.build("s_280_L_forced", 280, 2)
    name, taps = case["backbone"], _taps(case["backbone"])
    sd64 = vb.backbone64(sd, 280, cuda_device)
    x64 = x.to(cuda_device, torch.float64)
    with torch.no_grad():
        ex = vb.exact(x64, sd64, name, taps)
        emu = vb.emulate(x64, sd64, name, "fold", taps)
    got = vb.planted_model(x64, sd64, name, mistake, taps)
    last = None
    for (label, g, e), (_, mm, _) in zip(_pairs({**got[0], "features": got[1]}, ex, taps),
                                         _pairs({**emu[0], "features": emu[1]}, ex, taps)):
        r, glob = vb.row_ratios(g, mm, e)
        vb.describe(f"  {mistake} {label}", r, glob)
        if mistake == "no_lo_plane":
            assert r.median().item() > vb.R_MAX, label
        if label != "features" or mistake != "cls_without_pos0":
            last = (label, vb.passes(r, glob))
    assert last[1] is False, last


# ---- (c) bit-equality
_WEIGHTS = {}


def _bit_inputs(key):
    if key not in _WEIGHTS:
        weights, S = BIT_CASES[key]
        case, sd, bm, _ = vb.build(weights, S, 1)
        _WEIGHTS[key] = (case, sd, bm)
    case, sd, bm = _WEIGHTS[key]
    from multihmr_b200 import synth

    S = case["img_size"]
    return case, sd, bm, synth.make_images(4, S, seed=11), synth.make_images(1, S, seed=12)


def _same(a, b, what):
    for k in a:
        assert a[k].shape == b[k].shape, (what, k)
        assert torch.equal(a[k], b[k]), (what, k, (a[k] - b[k]).abs().max().item())


def _rows(out, sl):
    return {k: v[sl] for k, v in out.items()}


@pytest.mark.parametrize("key", list(BIT_CASES))
def test_batch_position_and_stale_rows_are_bit_exact(cuda_device, key):
    """Image i alone equals row block i of a 4-image call, and so do 2- and 3-image calls at other positions (every
    GEMM row and attention tile is computed from its own image only, whatever M_run < M the plans run at).  A 1-image
    call after a 4-image call on other images equals the same call on a fresh engine."""
    case, sd, bm, x4, y = _bit_inputs(key)
    taps = _taps(case["backbone"])
    m = vb.engine(case, sd, bm, 4)
    ref = vb.taps_and_features(m, x4, taps)
    for i in range(4):
        _same(vb.taps_and_features(m, x4[i:i + 1], taps), _rows(ref, slice(i, i + 1)), f"image {i} alone")
    _same(vb.taps_and_features(m, x4[2:4], taps), _rows(ref, slice(2, 4)), "images 2-3")
    _same(vb.taps_and_features(m, x4[1:4], taps), _rows(ref, slice(1, 4)), "images 1-3")
    vb.taps_and_features(m, x4, taps)
    after = vb.taps_and_features(m, y, taps)
    fresh_m = vb.engine(case, sd, bm, 4)
    fresh = vb.taps_and_features(fresh_m, y, taps)
    vb.release(m, fresh_m)
    _same(after, fresh, "1 image after 4")


@pytest.mark.parametrize("key", list(BIT_CASES))
def test_non_finite_image_stays_in_its_rows(cuda_device, key):
    """One NaN pixel in image 3 of 4: images 0-2 are bit-equal to the clean run (the GEMM and attention tiles that
    straddle an image boundary do not mix rows), image 3 comes out non-finite."""
    case, sd, bm, x4, _ = _bit_inputs(key)
    taps = _taps(case["backbone"])
    m = vb.engine(case, sd, bm, 4)
    clean = vb.taps_and_features(m, x4, taps)
    xn = x4.clone()
    xn[3, 1, 100, 37] = float("nan")
    got = vb.taps_and_features(m, xn, taps)
    vb.release(m)
    _same(_rows(got, slice(0, 3)), _rows(clean, slice(0, 3)), "images 0-2 next to a NaN")
    res = case["img_size"] // 14
    z3 = got["features"][3]
    bad_rows = (~torch.isfinite(z3)).any(-1)
    print(f"\n{key}: image 3 has {int(bad_rows.sum())} / {z3.shape[0]} non-finite feature rows")
    assert bad_rows[(100 // 14) * res + 37 // 14], "the NaN pixel's own patch row is finite"
    assert bad_rows.all()                    # attention spreads it over the whole image


_CHILD = r'''
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import torch
import test_vit_bulk_gpu as t
torch.save(t._pdl_outputs(), sys.argv[1])
'''


def _pdl_outputs():
    case, sd, bm, x4, _ = _bit_inputs("L_896")
    m = vb.engine(case, sd, bm, 4)
    out = {str(k): v.cpu() for k, v in vb.taps_and_features(m, x4[:2], _taps(case["backbone"])).items()}
    vb.release(m)
    return out


def test_pdl_off_is_bit_exact(cuda_device):
    """The blocks chain their kernels with programmatic dependent launch; a read before griddep_wait or a write racing
    the previous grid only shows there.  With MHMR_PDL=0 (read once per process, hence a child process) the stream
    taps and the features of ViT-L 896 x 2 are the same bits."""
    here = os.path.dirname(os.path.abspath(__file__))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "pdl_off.pt")
        env = dict(os.environ, MHMR_PDL="0")
        r = subprocess.run([sys.executable, "-c", _CHILD % (os.path.dirname(here), here), path], env=env,
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (r.stdout[-1000:], r.stderr[-3000:])
        off = torch.load(path)
    on = _pdl_outputs()
    _same(on, off, "PDL on vs off")
