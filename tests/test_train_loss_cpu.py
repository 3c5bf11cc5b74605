"""Premises of the training-loss kernels (csrc/train_loss.cu), checked in fp64 without a GPU: the rotation chain needs
only the body model's gradient with respect to each R (exp(log(R)) = R); torch restatements of the formulas the kernel
uses for the Gram-Schmidt backward and the focal derivative agree with autograd (the kernel itself is tested on the
GPU); Loss's arguments."""
import argparse

import torch

import train_loss_util as tl
from oracle import multihmr_ref, roma_ref


def _gs_grad(x, G):
    """csrc/train_loss.cu gram_schmidt_grad, restated in torch: x [n, 6], G [n, 3, 3] -> dx [n, 6]."""
    a, b = x[:, :3], x[:, 3:]
    na = a.norm(dim=1, keepdim=True)
    e1 = a / na
    dp = (e1 * b).sum(1, keepdim=True)
    bp = b - dp * e1
    nb = bp.norm(dim=1, keepdim=True)
    e2 = bp / nb
    g1, g2, g3 = G[:, :, 0], G[:, :, 1], G[:, :, 2]
    ge1 = g1 + torch.cross(e2, g3, dim=1)
    ge2 = g2 + torch.cross(g3, e1, dim=1)
    gbp = (ge2 - (ge2 * e2).sum(1, keepdim=True) * e2) / nb
    q = (e1 * gbp).sum(1, keepdim=True)
    db = gbp - q * e1
    ge1 = ge1 - (dp * gbp + q * b)
    da = (ge1 - (ge1 * e1).sum(1, keepdim=True) * e1) / na
    return torch.cat([da, db], 1)


def _rot6d(n, g):
    x = torch.randn(n, 6, generator=g, dtype=torch.float64) * 0.5
    return x + torch.tensor([1.0, 0, 0, 0, 1.0, 0], dtype=torch.float64)


def test_gram_schmidt_backward_matches_autograd():
    g = torch.Generator().manual_seed(0)
    x = _rot6d(500, g).requires_grad_()
    G = torch.randn(500, 3, 3, generator=g, dtype=torch.float64)
    R = multihmr_ref.rot6d_to_rotmat(x)
    (ref,) = torch.autograd.grad((R * G).sum(), x)
    got = _gs_grad(x.detach(), G)
    assert (got - ref).abs().max() < 1e-12
    # the transposed derivative (a planted mistake of the GPU tests) is far off
    assert (_gs_grad(x.detach(), G.transpose(1, 2)) - ref).abs().max() > 1e-2


def test_rotation_chain_needs_only_the_gradient_of_R():
    """d/dx <G, exp(log(GS(x)))> = d/dx <G, GS(x)>: the derivative of rotmat_to_rotvec is never needed, also near
    angle pi where it is singular."""
    g = torch.Generator().manual_seed(1)
    x = _rot6d(400, g)
    # rotations close to angle pi: a = e1, b = e2 of R(pi - 1e-3 about a random axis)
    ax = torch.nn.functional.normalize(torch.randn(50, 3, generator=g, dtype=torch.float64), dim=1)
    Rpi = roma_ref.rotvec_to_rotmat(ax * (torch.pi - 1e-3))
    x[:50] = torch.cat([Rpi[:, :, 0], Rpi[:, :, 1]], 1)
    x.requires_grad_()
    G = torch.randn(400, 3, 3, generator=g, dtype=torch.float64)
    R = multihmr_ref.rot6d_to_rotmat(x)
    (direct,) = torch.autograd.grad((R * G).sum(), x, retain_graph=True)
    R2 = roma_ref.rotvec_to_rotmat(roma_ref.rotmat_to_rotvec(R))
    (chain,) = torch.autograd.grad((R2 * G).sum(), x)
    assert (chain[50:] - direct[50:]).abs().max() < 1e-9
    assert (chain[:50] - direct[:50]).abs().max() < 1e-5 * (1 + direct[:50].abs().max())


def test_focal_derivative_as_the_kernel_writes_it():
    g = torch.Generator().manual_seed(2)
    logit = torch.randn(4000, generator=g, dtype=torch.float64) * 4
    logit[:50] = -30.0
    logit[50:60] = 30.0
    gt = (torch.rand(4000, generator=g) < 0.05).to(torch.float64)
    for gt_ in (gt, torch.zeros_like(gt)):
        lg = logit.clone().requires_grad_()
        s = tl.scores_from_logits(lg)
        pos = torch.log(s + 1e-7) * (1 - s) ** 2 * gt_
        neg = torch.log(1 - s + 1e-7) * s ** 2 * (1 - gt_)
        npos = gt_.sum()
        L = -neg.sum() if npos == 0 else -(pos.sum() + neg.sum()) / npos
        (ref,) = torch.autograd.grad(L, lg)
        sd = s.detach()
        q = 1 - sd
        ds = torch.where(gt_ >= 1, q * q / (sd + 1e-7) - 2 * q * torch.log(sd + 1e-7),
                         -(sd * sd) / (q + 1e-7) + 2 * sd * torch.log(q + 1e-7))
        coef = -1.0 if npos == 0 else -1.0 / npos
        on = (sd.float() != tl.LO) & (sd.float() != tl.HI)
        got = torch.where(on, coef * ds * sd * q, torch.zeros_like(sd))
        assert (got - ref).abs().max() <= 1e-12 * (1 + ref.abs().max())
        assert (ref[:60] == 0).all()


def test_loss_arguments_and_defaults():
    from multihmr_b200.loss import TERMS, Loss

    args = Loss.add_specific_args(argparse.ArgumentParser()).parse_args([])
    assert {k: getattr(args, "alpha_" + k) for k in tl.WEIGHTS} == tl.WEIGHTS
    assert args.start_2d_epoch == 10
    assert TERMS == ("total",) + tl.TERMS
