"""The training loss and its gradient on the device (mhmr_train_loss) against the fp64 autograd of the oracle's head
post-processing, the placed SMPL-X layer and the statement of loss.py (train_loss_util), at production sizes: B = 8,
res 64 (896 px), SMPL-X with 11 betas, P in {1, 16, 17, 48, 128}.  Every gradient element within its rounding bound,
each planted mistake outside it; the edge cases of the loss; guard bands; bitwise repeatability; Loss and
Model.training_loss."""
import argparse
import types

import pytest
import torch

import parity_util as pu
import train_loss_util as tl

pytestmark = pytest.mark.gpu
SENTINEL = 12345.0


@pytest.fixture(scope="module")
def engine(cuda_device):
    from multihmr_b200 import synth
    from multihmr_b200.model import Model

    sd = synth.make_state_dict("dinov2_vits14", 896, num_betas=11, seed=3)
    m = Model(backbone="dinov2_vits14", img_size=896, num_betas=11, max_batch=8, max_persons=128,
              body_model=synth.make_body_model(3))
    m.load_state_dict(sd, strict=False)
    m.finalize()
    return m


def _args(start_2d_epoch=10):
    return types.SimpleNamespace(**{"alpha_" + k: v for k, v in tl.WEIGHTS.items()}, start_2d_epoch=start_2d_epoch)


def _engine_inputs(m, case):
    """The engine's own fp32 outputs for the case's decoder rows: person post-processing and the SMPL-X layer."""
    from multihmr_b200 import ops

    dev, P, B = m.device, case["dec"].shape[0], case["K"].shape[0]
    f = lambda t: t.to(dev, torch.float32).contiguous()
    dec, off, K = f(case["dec"]), f(case["offset"]), f(case["K"])
    det = torch.stack([case["b"], case["cells"][:, 1], case["cells"][:, 0]]).to(dev, torch.int32)
    count = torch.tensor([P], device=dev, dtype=torch.int32)
    fn = m.img_size / (2 * __import__("math").tan(__import__("math").radians(30)))
    o = ops.person_post(dec, m.num_betas, off, K, det[0].contiguous(), det[1].contiguous(), det[2].contiguous(), count,
                        P, fn)
    body = m._smplx_forward(o["rotvec"], o["shape"], o["loc"], o["dist"], o["K_det"], o["expression"])
    s = torch.sigmoid(case["logit"]).clamp(tl.LO, tl.HI).to(dev, torch.float32).contiguous()
    t = dict(scores_map=s, count=count, det_idx=det, det_score=torch.zeros(P, device=dev), offset=off, loc=o["loc"],
             dist_pp=o["dist_pp"], dist=o["dist"], rotmat=o["rotmat"], rotvec=o["rotvec"], shape=o["shape"],
             expression=o["expression"], transl=body["transl"], transl_pelvis=body["transl_pelvis"][:, 0].contiguous(),
             v3d=body["v3d"], v2d=body["v2d"], j3d=body["j3d"], j2d=body["j2d"], dec=dec)
    return t, K


def _run(m, case, use_2d=True, guard=False):
    """mhmr_train_loss on the case: (loss [11], d_logits, d_offset, d_dec); with guard, the outputs are views into
    buffers one row / 64 cells larger filled with a sentinel, returned as the last element."""
    from multihmr_b200 import _lib
    from multihmr_b200._lib import call, stream

    t, K = _engine_inputs(m, case)
    dev, P, B = m.device, case["dec"].shape[0], case["K"].shape[0]
    y = {k: v.to(dev, torch.float32).contiguous() for k, v in case["targets"].items()}
    from multihmr_b200.loss import TARGETS, WEIGHTS

    tg = torch.tensor([y[k].data_ptr() for k in TARGETS], dtype=torch.int64)
    w = torch.tensor([tl.WEIGHTS[k] for k in WEIGHTS], dtype=torch.float32)
    BN, nd = B * m.res * m.res, 318 + m.num_betas + 13
    bufs = [torch.full((n,), SENTINEL, device=dev) for n in (BN + 64, (P + 1) * 2, (P + 1) * nd)]
    loss = torch.empty(11, device=dev)
    call("mhmr_train_loss", m._handle, B, P, K, _lib.struct("mhmr_outputs", **t), tg, y["shape"].shape[1], w,
         1 if use_2d else 0, loss,
         bufs[0], bufs[1], bufs[2], stream(dev))
    torch.cuda.synchronize()
    out = (loss, bufs[0][:BN].reshape(B, m.res, m.res), bufs[1][:P * 2].reshape(P, 2), bufs[2][:P * nd].reshape(P, nd))
    return out + ((bufs, BN, P * 2, P * nd),) if guard else out


def _ratios(got, case, ref, ref_abs, n, flips=0):
    """max err / bound of d_logits, d_dec and d_offset.  flips: sign flips of single vertex differences allowed on
    top of the rounding bound, each worth 2 / V of the person's |upstream| gradient sum."""
    tol = tl.logit_tolerance(ref[0].cpu(), case["logit"].cpu(), tl.bce_coef(case)) + 1e-30
    r_log = ((got[1].double().cpu() - ref[0].cpu()).abs() / tol).max().item()
    out = [r_log]
    for a, r, ra in ((got[3], ref[1], ref_abs[1]), (got[2], ref[2], ref_abs[2])):
        tol = tl.tolerance(r, ra, n)
        if flips:
            row = ra.abs().reshape(ra.shape[0], -1).amax(1).reshape((-1,) + (1,) * (ra.dim() - 1))
            tol = tol + flips * 2.0 / 10475 * row
        out.append(((a.double().reshape(r.shape) - r.to(a.device)).abs() / tol.to(a.device)).max().item())
    return out


def _case_on(case, dev):
    c = dict(case)
    for k in ("logit", "dec", "offset", "cells", "K_det"):
        c[k] = case[k].to(dev)
    c["targets"] = {k: v.to(dev) for k, v in case["targets"].items()}
    return c


def _check_terms(got_loss, terms, L, rtol=1e-4):
    vals = [L] + [terms[k] for k in tl.TERMS]
    for i, v in enumerate(vals):
        assert abs(got_loss[i].item() - v) <= rtol * abs(v) + 1e-6, (i, got_loss[i].item(), v)


@pytest.mark.parametrize("P", [1, 16, 17, 48, 128])
def test_loss_and_gradient_vs_fp64(engine, cuda_device, P):
    m = engine
    case = tl.make_case(m, P, 8, seed=40 + P)
    got = _run(m, case)
    terms, L, ref, ref_abs, case_cb = tl.reference(m._bm, _case_on(case, cuda_device))
    _check_terms(got[0], terms, L)
    r = _ratios(got, case, ref, ref_abs, tl.n_seq(m.num_verts))
    print(f"P={P} worst err/tol logits {r[0]:.3f} dec {r[1]:.3f} offset {r[2]:.3f}")
    assert max(r) <= 1.0, r
    assert all(torch.isfinite(t).all() for t in got[1:])


@pytest.mark.parametrize("mistake", ["no_pelvis", "mask_per_person", "no_inv_p", "clamp_grad", "gs_t"])
def test_planted_mistakes_fall_outside_the_bound(engine, cuda_device, mistake):
    m = engine
    case = tl.make_case(m, 16, 8, seed=7)
    got = _run(m, case)
    kw = {mistake: False} if mistake == "clamp_grad" else {mistake: True}
    _, _, wrong, _, _ = tl.reference(m._bm, _case_on(case, cuda_device), **kw)
    _, _, ref, ref_abs, case_cb = tl.reference(m._bm, _case_on(case, cuda_device))
    n = tl.n_seq(m.num_verts)
    assert max(_ratios(got, case, ref, ref_abs, n)) <= 1.0
    r = max(_ratios(got, case, wrong, ref_abs, n))
    print(f"{mistake}: err/tol {r:.3g}")
    assert r > 1.0


@pytest.mark.parametrize("edge", ["no_pos", "no_2d", "nan_shape", "dist_clamp", "before_2d"])
def test_edge_cases(engine, cuda_device, edge):
    m = engine
    case = tl.make_case(m, 17, 8, seed=11, edge=None if edge == "before_2d" else edge)
    use_2d = edge != "before_2d"
    got = _run(m, case, use_2d=use_2d)
    terms, L, ref, ref_abs, case_cb = tl.reference(m._bm, _case_on(case, cuda_device), use_2d=use_2d)
    _check_terms(got[0], terms, L)
    assert max(_ratios(got, case, ref, ref_abs, tl.n_seq(m.num_verts))) <= 1.0
    if edge == "no_2d":
        assert got[0][9].item() == 0.0 and got[0][10].item() == 0.0
    if edge == "nan_shape":
        assert got[0][4].item() == 0.0
    if edge == "before_2d":
        assert got[0][9].item() > 0 and got[0][10].item() > 0  # reported, not in the total


def test_fewer_betas_than_the_target(cuda_device):
    """An engine with 10 betas against 11-beta targets compares the first 10 (loss.py:55-56)."""
    case, sd, bm, x, K, idx = pu.build_inputs("s_224_S_forced")
    m = pu.build_engine(case, sd, bm, max_persons=16)
    c = tl.make_case(m, 5, 3, seed=2, nb_gt=11)
    got = _run(m, c)
    terms, L, ref, ref_abs, case_cb = tl.reference(m._bm, _case_on(c, cuda_device))
    _check_terms(got[0], terms, L)
    assert max(_ratios(got, c, ref, ref_abs, tl.n_seq(m.num_verts))) <= 1.0


def test_guard_bands_and_bitwise_repeat(engine):
    m = engine
    case = tl.make_case(m, 48, 8, seed=5)
    a = _run(m, case, guard=True)
    bufs, nl, no, nd = a[4]
    assert (bufs[0][nl:] == SENTINEL).all() and (bufs[1][no:] == SENTINEL).all() and (bufs[2][nd:] == SENTINEL).all()
    b = _run(m, case)
    assert all(torch.equal(x, y) for x, y in zip(a[:4], b))


def test_training_loss_and_loss_module(engine, cuda_device):
    """Model.training_loss and Loss.forward on a forward of the model give the kernel's values for the forward's
    outputs; the gradients come with the shapes of the head's last Linears."""
    from multihmr_b200 import synth
    from multihmr_b200.loss import Loss

    m = engine
    B, P = 2, 5
    x = synth.make_images(B, m.img_size, 1)
    K = synth.make_cameras(B, m.img_size, jitter=True, seed=1)
    idx = synth.make_forced_idx(B, m.res, [3, 2], 1)
    y_hat = m(x, idx=idx, K=K, is_training=True)
    g = torch.Generator().manual_seed(0)
    rnd = lambda t: (t + 0.05 * torch.randn(t.shape, generator=g).to(t.device)).contiguous()
    y = {k: rnd(y_hat[k].detach()) for k in ("offset", "rotmat", "transl", "j3d", "v3d", "j2d", "v2d")}
    y["shape"] = torch.cat([rnd(y_hat["shape"]), torch.zeros(P, 11 - m.num_betas, device=cuda_device)], 1)
    y["dist_postprocessed"] = rnd(y_hat["dist_postprocessed"][:, 0])
    y["transl_pelvis"] = rnd(y_hat["transl_pelvis"][:, 0])
    y["scores"] = torch.zeros(B, m.res, m.res, device=cuda_device)
    y["scores"][idx[0], idx[1], idx[2]] = 1.0
    y.update(idx=idx, K=K)
    parser = Loss.add_specific_args(argparse.ArgumentParser())
    args = parser.parse_args([])
    loss = Loss(args)
    total, d = loss(y_hat, y, epoch=12, img_size=m.img_size)
    total2, d2, grads = m.training_loss(x, y, 12, args)
    assert torch.equal(total, total2) and all(torch.equal(d[k], d2[k]) for k in d)
    assert all(torch.equal(loss.last_grads[k], grads[k]) for k in grads)
    assert grads["scores_logits"].shape == (B, m.res, m.res) and grads["offset"].shape == (P, 2)
    assert grads["dec"].shape == (P, 318 + m.num_betas + 13)
    assert torch.isfinite(total) and total.item() > 0
    with pytest.raises(TypeError):
        loss(dict(y_hat), y, epoch=0, img_size=m.img_size)


@pytest.fixture(scope="module")
def golden_engine(cuda_device):
    from multihmr_b200 import synth
    from multihmr_b200.model import Model

    m = Model(backbone="dinov2_vits14", img_size=224, num_betas=10, max_batch=3, max_persons=8,
              body_model=synth.make_body_model(tl.GOLDEN_SEED))
    m.load_state_dict(synth.make_state_dict("dinov2_vits14", 224, seed=tl.GOLDEN_SEED), strict=False)
    m.finalize()
    return m, pu.load_golden("train_loss_224_S")


@pytest.mark.parametrize("epoch", [12, 0])
def test_engine_matches_the_reference_golden(golden_engine, cuda_device, epoch):
    """The kernel on the reference model's head outputs and the reference's targets (tests/golden/train_loss_224_S,
    oracle/make_golden_train.py) against the reference's own Loss.forward and autograd gradients.  The targets are not
    kept away from the predictions here, so a rounding may flip the sign of a difference within fp32 rounding of 0:
    up to 4 vertex flips per person are allowed on top of the bound."""
    m, gold = golden_engine
    case = tl.golden_case(gold)
    got = _run(m, case, use_2d=epoch >= 10)
    want = gold[f"loss_e{epoch}"]
    for i in range(11):
        assert abs(got[0][i].item() - float(want[i])) <= 1e-4 * abs(float(want[i])) + 1e-6, (i, got[0][i].item(), want[i])
    _, _, _, ref_abs, _ = tl.reference(m._bm, _case_on(case, cuda_device), use_2d=epoch >= 10)
    ref = [gold[f"{k}_e{epoch}"].to(cuda_device, torch.float64) for k in ("d_logits", "d_dec", "d_offset")]
    r = _ratios(got, case, ref, ref_abs, tl.n_seq(m.num_verts), flips=4)
    print(f"golden epoch {epoch}: worst err/tol logits {r[0]:.3f} dec {r[1]:.3f} offset {r[2]:.3f}")
    assert max(r) <= 1.0, r


def test_prepare_train_targets_matches_the_reference(golden_engine, cuda_device):
    """metrics.prepare_train_targets on the golden's batch (two persons on one head patch, a person at the border, an
    image without persons) against the reference's Trainer.prepare_gt: indices and heat map exactly, the rest within
    the fp32 parity tolerances."""
    from multihmr_b200 import metrics, synth

    _, gold = golden_engine
    y = {k: gold[k].to(cuda_device) for k in ("K", "valid_humans", "smplx_root_pose", "smplx_body_pose",
                                              "smplx_jaw_pose", "smplx_leye_pose", "smplx_reye_pose",
                                              "smplx_left_hand_pose", "smplx_right_hand_pose", "smplx_shape",
                                              "smplx_transl")}
    bodies = {"smplx": metrics.BodyModel(synth.make_body_model(tl.GOLDEN_SEED), "smplx", 11, 8, cuda_device)}
    t = metrics.prepare_train_targets(y, bodies, img_size=224)
    idx = torch.stack([i.long() for i in t["idx"]]).cpu()
    assert torch.equal(idx, gold["gt_idx"].long())
    assert torch.equal(t["scores"].cpu(), gold["gt_scores"])
    tol = dict(loc=2e-2, j2d=2e-2, v2d=2e-2, offset=2e-2 / 14)
    for k in ("scores", "offset", "rotmat", "rotvec", "shape", "dist", "dist_postprocessed", "transl", "transl_pelvis",
              "j3d", "v3d", "j2d", "v2d", "loc"):
        a, b = t[k].float().cpu(), gold["gt_" + k].float()
        assert a.shape == b.shape, (k, a.shape, b.shape)
        err = (a - b).abs().max().item()
        assert err <= tol.get(k, 1e-4), (k, err)
