"""Writes tests/golden/train_loss_224_S.npz from the reference's OWN training step: `Trainer.prepare_gt`, the forced-index
forward of `Model` (model.py, is_training=True) and `Loss.forward` (loss.py) with its autograd gradients.

Runs ONLY in the build container (needs /root/reference).  It imports /root/reference/train.py, model.py and loss.py
UNMODIFIED, with the shims of oracle/make_golden.py (roma, smplx.create for the model's SMPL-X layer, the torch.hub
DINOv2) and of oracle/make_golden_eval.py (tensorboard, render-only imports, the datasets package):
  * a `Trainer` made with `Trainer.__new__` (its `smplx_neutral_11` the 11-beta SMPL-X shim) runs `prepare_gt` on a
    seeded BEDLAM-style batch of three images: two persons sharing a head patch (the second is dropped), a person at
    the image border (2-D targets leaving the image) and an image without persons;
  * the reference model (ViT-S, 224 px, 10 betas, synthetic weights of multihmr_b200.synth) is converted to fp64 and
    run at gt['idx'] / gt['K']; forward hooks make the outputs of mlp_classif, mlp_offset and the four dec* Linears
    leaves of the graph, so that `Loss.forward(...)` followed by `backward()` gives the gradients there;
  * the loss is taken at epoch 12 (2-D terms in the total) and at epoch 0 (before start_2d_epoch, default 10).
The npz holds the batch, the reference's targets, the head outputs (logits [B, res, res], offset [P, 2], the decoder
rows dec = pose6 | betas | cam | expression with the inits added, as the engine's decoder writes them) and, per epoch,
the eleven loss values and the gradients (fp64).

Usage:  python -m oracle.make_golden_train            (from the repo root)
"""
import argparse
import os
import sys
import tempfile
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
REFERENCE = "/root/reference"

from multihmr_b200 import synth  # noqa: E402
from oracle import eval_bench_ref, make_golden, make_golden_eval  # noqa: E402

SEED = 21
IMG_SIZE = 224
TERMS = ("total", "bce", "offset", "rotmat", "shape", "dist", "transl", "j3d", "v3d", "j2d", "v2d")
EPOCHS = (12, 0)


def make_batch(seed=SEED):
    """BEDLAM-style batch in the reference's collate_fn format: 3 images, up to 3 persons each."""
    g = torch.Generator().manual_seed(seed)
    B, H = 3, 3
    K = eval_bench_ref._camera(IMG_SIZE).repeat(B, 1, 1)
    valid = torch.tensor([[1, 1, 1], [1, 1, 0], [0, 0, 0]], dtype=torch.float32)
    transl = torch.stack([torch.randn(B, H, generator=g) * 0.3, torch.randn(B, H, generator=g) * 0.1,
                          5.0 + torch.rand(B, H, generator=g)], -1)
    transl[0, 1] = transl[0, 0] + torch.tensor([0.0005, 0.0, 0.0])  # same head patch as person 0: dropped
    transl[1, 1] = torch.tensor([1.55, 0.2, 4.5])  # at the image border: part of the 2-D targets leave the image
    p = eval_bench_ref._smplx_params(g, B * H)
    for v in p.values():
        v[1] = v[0]  # person 1 of image 0: the body of person 0, 0.5 mm to the side
    r = lambda t, n: t.reshape(B, H, n, 3) if n > 1 else t.reshape(B, H, 1, 3)
    return dict(K=K, valid_humans=valid, smplx_root_pose=r(p["root"], 1), smplx_body_pose=r(p["body"], 21),
                smplx_jaw_pose=r(p["jaw"], 1), smplx_leye_pose=r(p["leye"], 1), smplx_reye_pose=r(p["reye"], 1),
                smplx_left_hand_pose=r(p["lhand"], 15), smplx_right_hand_pose=r(p["rhand"], 15),
                smplx_shape=p["betas"].reshape(B, H, 11), smplx_transl=transl)


def main():
    assert os.path.isdir(REFERENCE), "make_golden_train needs the reference checkout (build container only)"
    make_golden_eval.install_shims()
    make_golden.install_shims()  # the model's smplx.create and roma over the evaluation's
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count())
    case = dict(backbone="dinov2_vits14", img_size=IMG_SIZE)
    sd = synth.make_state_dict(case["backbone"], IMG_SIZE, seed=SEED)
    bm = synth.make_body_model(SEED)
    mean = synth.make_mean_params(SEED)
    model = make_golden.build_reference_model(case, sd, bm, mean)
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    ds = types.ModuleType("datasets")
    ds.__path__ = [os.path.join(REFERENCE, "datasets")]
    sys.modules["datasets"] = ds
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp(prefix="mhmr_train_"))
    try:
        import train  # the reference, unmodified
        from loss import Loss  # the reference, unmodified
    finally:
        os.chdir(cwd)

    y = make_batch()
    train.args = argparse.Namespace(person_center="head", img_size=IMG_SIZE, amp=0)
    t = train.Trainer.__new__(train.Trainer)
    t.device, t.args, t.model = torch.device("cpu"), train.args, model
    t.smplx_neutral_11 = eval_bench_ref.SMPLXFullShim(bm, num_betas=11)
    with torch.no_grad():
        gt = t.prepare_gt({k: v.clone() for k, v in y.items()})
    P = int(gt["idx"][0].shape[0])
    assert P == 4, P  # five annotated persons, one dropped

    model = model.double()
    # embedd_camera builds its token grid with `.float()` (model.py:164-175): integer pixel centres, exact in fp32; cast
    # them to the fp64 intrinsics at the one call that mixes the two
    ref_model = sys.modules[type(model).__module__]
    ipp = ref_model.inverse_perspective_projection
    ref_model.inverse_perspective_projection = lambda pts, K, dist: ipp(pts.to(K.dtype), K, dist.to(K.dtype))
    leaves = {}

    def leaf(name):
        def hook(mod, inp, out):
            lv = out.detach().requires_grad_()
            leaves[name] = lv
            return lv * 1.0  # the model's in-place sigmoid_ must not touch the leaf
        return hook

    h = model.x_attention_head
    mods = dict(classif=model.mlp_classif, offset=model.mlp_offset, decpose=h.decpose, decshape=h.decshape,
                deccam=h.deccam, decexpression=h.decexpression)
    for n, mod in mods.items():
        mod.register_forward_hook(leaf(n))
    x = synth.make_images(3, IMG_SIZE, SEED).double()
    gt64 = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in gt.items()}
    parser = Loss.add_specific_args(argparse.ArgumentParser(add_help=False))
    largs = parser.parse_args([])
    gold = {k: v.numpy() for k, v in y.items()}
    for k in ("scores", "offset", "rotmat", "shape", "dist_postprocessed", "transl", "transl_pelvis", "j3d", "v3d",
              "j2d", "v2d", "loc", "dist", "rotvec"):
        gold["gt_" + k] = gt[k].float().numpy()
    gold["gt_idx"] = torch.stack([i.long() for i in gt["idx"]]).numpy()
    res = IMG_SIZE // 14
    torch.set_default_dtype(torch.float64)  # tensors the model creates on the fly (camera rays, grids) in fp64 too
    for epoch in EPOCHS:
        leaves.clear()
        pred = model(x, is_training=True, idx=gt["idx"], K=gt64["K"])
        total, d = Loss(largs)(pred, gt64, epoch=epoch, img_size=IMG_SIZE)
        total.backward()
        gold[f"loss_e{epoch}"] = np.array([float(d[k]) for k in TERMS])
        gold[f"d_logits_e{epoch}"] = leaves["classif"].grad.reshape(3, res, res).numpy()
        gold[f"d_offset_e{epoch}"] = leaves["offset"].grad.numpy()
        gold[f"d_dec_e{epoch}"] = torch.cat([leaves[n].grad.reshape(P, -1) for n in
                                             ("decpose", "decshape", "deccam", "decexpression")], 1).numpy()
    inits = [h.init_body_pose, h.init_betas, h.init_cam, h.init_expression]
    gold["logits"] = leaves["classif"].detach().reshape(3, res, res).numpy()
    gold["offset"] = leaves["offset"].detach().numpy()
    gold["dec"] = torch.cat([leaves[n].detach().reshape(P, -1) + i.detach().reshape(1, -1) for n, i in
                             zip(("decpose", "decshape", "deccam", "decexpression"), inits)], 1).numpy()
    out = os.path.join(REPO, "tests", "golden", "train_loss_224_S.npz")
    np.savez_compressed(out, **gold)
    print(f"train_loss_224_S: P={P}, loss e12 {gold['loss_e12'].round(4).tolist()}, e0 total {gold['loss_e0'][0]:.4f}")


if __name__ == "__main__":
    main()
