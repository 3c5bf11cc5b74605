"""Training loss of the SMPL-X head on the device (reference loss.py): the same `Loss(parser_args)` constructor,
`add_specific_args` and `forward(y_hat, y, epoch, img_size) -> (total, dict_loss)`, computed with its gradient by
`mhmr_train_loss` (csrc/train_loss.cu, DESIGN.md §10).  `y_hat` is what `Model.forward(..., is_training=True)`
returns, `y` what `metrics.prepare_train_targets` returns.  After a forward, `Loss.last_grads` holds the gradient of
the total with respect to the head's last Linears (see `Model.training_loss`)."""
from __future__ import annotations

from argparse import ArgumentParser

import torch

from . import _lib
from ._lib import call, stream

TERMS = ("total", "bce", "offset", "rotmat", "shape", "dist", "transl", "j3d", "v3d", "j2d", "v2d")
WEIGHTS = ("bce", "offset", "rotmat", "shape", "dist", "transl", "j3d", "v3d", "j2d", "v2d")
# the targets in the order of mhmr_train_loss's address table
TARGETS = ("scores", "offset", "rotmat", "shape", "dist_postprocessed", "transl", "transl_pelvis", "j3d", "v3d", "j2d",
           "v2d")
DEFAULT_WEIGHTS = dict(zip(WEIGHTS, (10.0, 1.0, 0.1, 1.0, 1.0, 1.0, 100.0, 100.0, 1.0, 1.0)))


def run_train_loss(model, t: dict, P: int, K, y: dict, epoch: int, args):
    """`mhmr_train_loss` on the raw outputs `t` of a forced-index forward of `model` with P persons (v2d and dec
    requested) and the targets `y`.  Returns (total, dict_loss, grads) on the device."""
    dev = model.device
    f32 = lambda v: v.to(dev, torch.float32).contiguous()
    tg = [f32(y[k]) for k in TARGETS]
    tg[4] = tg[4].reshape(-1)
    # the kernel reads the targets at raw addresses: every shape is checked here
    B, V, nb_gt = int(tg[0].shape[0]), model.num_verts, int(tg[3].shape[-1]) if tg[3].dim() == 2 else -1
    want = dict(scores=(B, model.res, model.res), offset=(P, 2), rotmat=(P, 53, 3, 3), shape=(P, nb_gt),
                dist_postprocessed=(P,), transl=(P, 3), transl_pelvis=(P, 3), j3d=(P, 127, 3), v3d=(P, V, 3),
                j2d=(P, 127, 2), v2d=(P, V, 2))
    for k, t_ in zip(TARGETS, tg):
        if tuple(t_.shape) != want[k] or nb_gt < 1:
            raise ValueError(f"target {k!r} has shape {tuple(t_.shape)}, expected {want[k]} for {P} forced persons")
    if B != int(K.shape[0]) or B > model.max_batch:
        raise ValueError(f"scores cover {B} images, the forward {int(K.shape[0])}")
    targets = torch.tensor([t.data_ptr() for t in tg], dtype=torch.int64)
    weights = torch.tensor([float(getattr(args, "alpha_" + k)) for k in WEIGHTS], dtype=torch.float32)
    loss = torch.empty(len(TERMS), device=dev)
    grads = {"scores_logits": torch.empty(B, model.res, model.res, device=dev),
             "offset": torch.empty(P, 2, device=dev), "dec": torch.empty(P, 318 + model.num_betas + 13, device=dev)}
    use_2d = 1 if epoch >= args.start_2d_epoch else 0
    with torch.cuda.device(dev):
        call("mhmr_train_loss", model._handle, B, P, f32(K), _lib.struct("mhmr_outputs", **t), targets,
             int(tg[3].shape[1]), weights, use_2d, loss, grads["scores_logits"], grads["offset"], grads["dec"],
             stream(dev))
    dict_loss = {k: loss[i] for i, k in enumerate(TERMS)}
    return dict_loss["total"], dict_loss, grads


class Loss(torch.nn.Module):
    """reference loss.py:42-141."""

    def __init__(self, parser_args, *args, **kwargs):
        super().__init__()
        self.parser_args = parser_args
        self.last_grads = None

    def forward(self, y_hat, y, epoch=None, img_size=None):
        raw = getattr(y_hat, "raw", None)
        if raw is None:
            raise TypeError("Loss.forward takes the outputs of Model.forward(..., is_training=True) of this package")
        model, t, P, K = raw
        if img_size is not None and int(img_size) != model.img_size:
            raise ValueError(f"img_size {img_size} differs from the model's {model.img_size}")
        total, dict_loss, self.last_grads = run_train_loss(model, t, P, K, y, epoch, self.parser_args)
        return total, dict_loss

    @staticmethod
    def add_specific_args(parent_parser):
        """loss.py:117-141: --alpha_<term> for the ten terms and --start_2d_epoch, with the reference's defaults."""
        parser = ArgumentParser(parents=[parent_parser], add_help=False)
        for k in WEIGHTS:
            parser.add_argument(f"--alpha_{k}", type=float, default=DEFAULT_WEIGHTS[k])
        parser.add_argument("--start_2d_epoch", type=int, default=10)
        return parser
