"""The fp64 restatement of the training step (train_loss_util: head post-processing, placed SMPL-X layer, loss.py)
against the reference's own `Loss.forward` and autograd gradients (tests/golden/train_loss_224_S.npz, written by
oracle/make_golden_train.py from the unmodified reference): the eleven loss values and the gradients at the outputs
of mlp_classif, mlp_offset and the dec* Linears, with the 2-D terms in the total (epoch 12) and before
start_2d_epoch (epoch 0)."""
import pytest
import torch

import parity_util as pu
import train_loss_util as tl


@pytest.fixture(scope="module")
def golden():
    from multihmr_b200 import synth

    return pu.load_golden("train_loss_224_S"), synth.make_body_model(tl.GOLDEN_SEED)


@pytest.mark.parametrize("epoch", [12, 0])
def test_restatement_matches_the_reference(golden, epoch):
    gold, bm = golden
    case = tl.golden_case(gold)
    terms, L, ref, _, _ = tl.reference(bm, case, use_2d=epoch >= 10)
    got = [L] + [terms[k] for k in tl.TERMS]
    want = gold[f"loss_e{epoch}"]
    assert all(abs(a - float(b)) <= 1e-9 * (1 + abs(float(b))) for a, b in zip(got, want)), (got, want)
    for r, k in zip(ref, ("d_logits", "d_dec", "d_offset")):
        w = gold[f"{k}_e{epoch}"].to(torch.float64)
        err = (r.reshape(w.shape) - w).abs().max().item()
        assert err <= 1e-9 * (1 + w.abs().max().item()), (k, err)


def test_golden_covers_its_cases(golden):
    gold, _ = golden
    assert gold["gt_idx"].shape[1] == 4  # five annotated persons, one sharing a head patch
    assert not bool(gold["valid_humans"][2].any()) and float(gold["gt_scores"][2].sum()) == 0.0
    v2d = gold["gt_v2d"]
    inside = ((v2d > 0) & (v2d < 224)).all(-1)
    assert 0 < int(inside.sum()) < inside.numel()  # some 2-D targets leave the image
    assert float(gold["loss_e12"][0]) != float(gold["loss_e0"][0])
