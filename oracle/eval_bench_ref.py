"""CPU restatement of the three evaluation protocols of the reference's `Trainer.prepare_gt` / `Trainer.evaluate`
(train.py:58-182, :336-482): 3DPW (SMPL ground truth, SMPL-X -> SMPL transfer, MPJPE on 14 H36M joints), EHF (SMPL-X
vertices, J_regressor joints) and BEDLAM (SMPL-X parameters, 11 betas).  Plain torch fp32, every step cites the lines
it follows; the body models restate `smplx.SMPL` / `smplx.SMPLX` forward with a full pose and `transl` on top of
oracle/smplx_ref.lbs.  Pinned against the reference's OWN train.py by oracle/make_golden_eval.py
(tests/golden/eval_{3dpw,ehf,bedlam}.npz).  The seeded evaluation cases (inputs) live here too, so that the golden
script, the CPU tests and the GPU tests regenerate the same ones.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import math

import numpy as np
import torch

from . import eval_ref, smplx_ref

H36M_TO_J17 = [6, 5, 4, 1, 2, 3, 16, 15, 14, 11, 12, 13, 8, 10, 0, 7, 9]   # train.py:402
H36M_TO_J14 = H36M_TO_J17[:14]                                             # train.py:403
METERS = ["pve", "pa_pve", "precision", "recall", "f1_score", "mpjpe", "pa_mpjpe"]  # train.py:341-343


class SMPLShim(torch.nn.Module):
    """`smplx.create(SMPLX_DIR, 'smpl', gender=...)` stand-in (train.py:42-43) built from an SMPL body-model dict
    (multihmr_b200.synth.make_smpl_body_model): smplx.SMPL.forward = lbs over [global_orient | body_pose] (24 joints),
    joints = [24 LBS joints | 21 vertex-picked joints (vertex_ids['smplh'])], then + transl."""

    def __init__(self, bm: dict, num_betas: int = 10):
        super().__init__()
        self.bm = {k: v for k, v in bm.items() if isinstance(v, torch.Tensor)}
        self.num_betas = num_betas
        self.faces = bm["faces"].numpy()

    def forward(self, global_orient, body_pose, betas, transl):
        b = self.bm
        full_pose = torch.cat([global_orient.reshape(-1, 3), body_pose.reshape(-1, 69)], dim=1)
        verts, joints = smplx_ref.lbs(betas, full_pose, b["v_template"].float(),
                                      b["shapedirs"][..., : self.num_betas].float(), b["posedirs"].float(),
                                      b["J_regressor"].float(), b["parents"].long(), b["lbs_weights"].float())
        joints = torch.cat([joints, verts[:, b["extra_joints_idxs"].long()]], dim=1)
        return smplx_ref.Output(verts + transl.unsqueeze(1), joints + transl.unsqueeze(1))


class SMPLXFullShim(smplx_ref.SMPLXShim):
    """`smplx.create(SMPLX_DIR, 'smplx', gender='neutral', use_pca=False, flat_hand_mean=True, num_betas=11)` as
    Trainer.prepare_gt calls it (train.py:41, :98-109): global orient, eyes and `transl` are call arguments."""

    def forward(self, betas, global_orient, body_pose, left_hand_pose, right_hand_pose, jaw_pose, expression=None,
                leye_pose=None, reye_pose=None, transl=None):
        B = betas.shape[0]
        z3 = torch.zeros(B, 3)
        out = super().forward(betas, global_orient, body_pose, left_hand_pose, right_hand_pose, jaw_pose,
                              expression if expression is not None else torch.zeros(B, 10),
                              leye_pose if leye_pose is not None else z3, reye_pose if reye_pose is not None else z3)
        t = (transl if transl is not None else z3).unsqueeze(1)
        return smplx_ref.Output(out.vertices + t, out.joints + t)


def perspective_projection(x, K):
    """utils/camera.py:14-27."""
    y = x / x[:, :, -1].unsqueeze(-1)
    y = torch.einsum("bij,bkj->bki", K, y)
    return y[:, :, :2]


def prepare_gt(y, models, person_center_idx=15, img_size=448, patch_size=14):
    """train.py:58-182, the keys evaluate reads (K, j2d, v3d, transl_pelvis).  models: smplx, smpl_male,
    smpl_female shims."""
    valid_h = y["valid_humans"]
    idx_h = torch.where(valid_h)                                                     # :64-65
    nhv = int(valid_h.sum())
    K = y["K"][idx_h[0]]                                                             # :67
    if "smplx_vertices" in y:                                                        # :70-73
        verts = y["smplx_vertices"].reshape(1, -1, 3)
        jts = models["smplx"].J_regressor @ verts
    elif "smpl_root_pose" in y:                                                      # :74-94
        kw = dict(global_orient=y["smpl_root_pose"][idx_h[0], idx_h[1]].reshape(-1, 3),
                  body_pose=y["smpl_body_pose"][idx_h[0], idx_h[1]].reshape(-1, 23 * 3),
                  betas=y["smpl_shape"][idx_h[0], idx_h[1]].reshape(-1, 10),
                  transl=y["smpl_transl"][idx_h[0], idx_h[1]].reshape(-1, 3))
        out = models["smpl_male"](**kw)
        verts, jts = out.vertices.reshape(nhv, -1, 3), out.joints.reshape(nhv, -1, 3)
        if int(y["smpl_gender_id"].max()) == 2:
            out_f = models["smpl_female"](**kw)
            idx = torch.where(y["smpl_gender_id"] == 2)[1]
            verts[idx] = out_f.vertices.reshape(nhv, -1, 3)[idx]
            jts[idx] = out_f.joints.reshape(nhv, -1, 3)[idx]
    elif "smplx_root_pose" in y:                                                     # :95-110
        s = lambda k, n: y[k][idx_h[0], idx_h[1]].reshape(-1, n)
        out = models["smplx"](global_orient=s("smplx_root_pose", 3), body_pose=s("smplx_body_pose", 63),
                              jaw_pose=s("smplx_jaw_pose", 3), leye_pose=s("smplx_leye_pose", 3),
                              reye_pose=s("smplx_reye_pose", 3), left_hand_pose=s("smplx_left_hand_pose", 45),
                              right_hand_pose=s("smplx_right_hand_pose", 45), betas=s("smplx_shape", 11),
                              transl=s("smplx_transl", 3), expression=torch.zeros(nhv, 10))
        verts, jts = out.vertices.reshape(nhv, -1, 3), out.joints.reshape(nhv, -1, 3)
    else:
        return None
    j2d = perspective_projection(jts, K)                                             # :113
    n_patch = img_size // patch_size                                                 # :137
    pk_loc = perspective_projection(jts[:, person_center_idx].unsqueeze(1), K).squeeze(1)   # :138-139
    pk_idx = torch.clamp((pk_loc // patch_size).int(), 0, n_patch - 1)             # :140-141
    taken, vis = set(), []
    for k in range(nhv):                                                             # :147-156
        cell = (int(idx_h[0][k]), int(pk_idx[k, 1]), int(pk_idx[k, 0]))
        vis.append(cell not in taken)
        taken.add(cell)
    keep = torch.tensor([k for k in range(nhv) if vis[k]], dtype=torch.long)        # :169-180
    return dict(K=y["K"], j2d=j2d[keep], v3d=verts[keep], transl_pelvis=jts[:, 0][keep], j3d=jts[keep])


@torch.no_grad()  # train.py:336
def evaluate(cases, models, smplx2smpl, j_regressor_h36m, dataset, img_size):
    """train.py:336-482 over (x, y, persons) cases (batch size 1).  smplx2smpl: torch (sparse or dense) [6890, 10475].
    Returns (final meter averages, per-pair values per meter)."""
    vals = {k: [] for k in ("pve", "pa_pve", "mpjpe", "pa_mpjpe")}
    count = miss = fp = 0
    for x, y, pred in cases:
        gt = prepare_gt(y, models, img_size=img_size)
        kp_gt = gt["j2d"].numpy()                                                    # :360-362
        kp_pred = np.asarray([h["j2d"].numpy()[: kp_gt.shape[1]] for h in pred])
        best, fps, misses = eval_ref.match_2d_greedy(kp_pred, kp_gt, np.ones_like(kp_gt[..., 0]).astype(np.bool_))
        count += len(kp_gt)                                                          # :365-367
        miss += len(misses)
        fp += len(fps)
        for pid, gid in best:                                                        # :371-429
            v3d_ctx = gt["v3d"][gid] - gt["transl_pelvis"][gid].reshape(1, 3)
            v3d_hat_ctx = pred[pid]["v3d"] - pred[pid]["transl_pelvis"].reshape(1, 3)
            if v3d_ctx.shape[0] == 6890:
                v3d_hat_ctx = smplx2smpl @ v3d_hat_ctx
            e, pe = eval_ref.points_errors(v3d_hat_ctx, v3d_ctx)
            vals["pve"].append(e.item())
            vals["pa_pve"].append(pe.item())
            if dataset == "3dpw":
                h = j_regressor_h36m @ v3d_ctx
                hh = j_regressor_h36m @ v3d_hat_ctx
                h, hh = (h - h[[0]])[H36M_TO_J14], (hh - hh[[0]])[H36M_TO_J14]
                e, pe = eval_ref.points_errors(hh, h)
                vals["mpjpe"].append(e.item())
                vals["pa_mpjpe"].append(pe.item())
    precision, recall, f1 = eval_ref.compute_prf1(count, miss, fp)                  # :473
    avg = lambda v: float(np.mean(v)) if len(v) else 0.0
    meters = dict(pve=avg(vals["pve"]), pa_pve=avg(vals["pa_pve"]), precision=float(precision), recall=float(recall),
                  f1_score=float(f1), mpjpe=avg(vals["mpjpe"]), pa_mpjpe=avg(vals["pa_mpjpe"]))
    return meters, {k: np.asarray(v, dtype=np.float64) for k, v in vals.items()}


# ------------------------------------------------------------------------------------------------------------------
# Seeded evaluation cases
# ------------------------------------------------------------------------------------------------------------------
IMG_SIZE = 448
DATASETS = ("3dpw", "ehf", "bedlam")


def eval_assets(seed=0):
    """Body-model dicts and regressors of the evaluation (synthetic, seeded)."""
    from multihmr_b200 import synth

    return dict(smplx=synth.make_body_model(seed), smpl_male=synth.make_smpl_body_model(seed, "male"),
                smpl_female=synth.make_smpl_body_model(seed, "female"), smplx2smpl=synth.make_smplx2smpl(seed),
                j_regressor_h36m=synth.make_j_regressor_h36m(seed))


def shim_models(assets):
    return dict(smplx=SMPLXFullShim(assets["smplx"], num_betas=11), smpl_male=SMPLShim(assets["smpl_male"]),
                smpl_female=SMPLShim(assets["smpl_female"]))


def _camera(img_size):
    f = img_size / (2 * math.tan(math.radians(60) / 2))
    K = torch.tensor([[f, 0.0, img_size / 2], [0.0, f, img_size / 2], [0.0, 0.0, 1.0]])
    return K.unsqueeze(0)


def _smplx_params(g, n, pose_std=0.15):
    r = lambda *s, std=pose_std: torch.randn(*s, generator=g) * std
    return dict(root=r(n, 1, 3, std=0.3), body=r(n, 21, 3), jaw=r(n, 1, 3), leye=r(n, 1, 3), reye=r(n, 1, 3),
                lhand=r(n, 15, 3), rhand=r(n, 15, 3), betas=r(n, 11, std=0.8))


def make_cases(dataset, assets, seed=0):
    """Images of `dataset` in the reference's collate_fn format (batch size 1) with the prescribed predictions of
    a stub model: list of (x [1,3,S,S], y, persons); two images for 3DPW / BEDLAM, three single-person images for EHF.
    Predictions are SMPL-X bodies near the ground truths (noisy parameters), plus one false positive per image; one
    ground truth of the last image has no prediction (a miss), and in BEDLAM two ground truths share the head patch
    (the second is dropped by prepare_gt)."""
    g = torch.Generator().manual_seed({"3dpw": 11, "ehf": 12, "bedlam": 13}[dataset] + 100 * seed)
    S = IMG_SIZE
    K = _camera(S)
    body = SMPLXFullShim(assets["smplx"], num_betas=11)
    cases = []
    n_gt_per_image = {"3dpw": [2, 3], "ehf": [1, 1, 1], "bedlam": [2, 3]}[dataset]
    last = len(n_gt_per_image) - 1
    for img, G in enumerate(n_gt_per_image):
        xs = torch.linspace(-1.6, 1.6, G) if G > 1 else torch.zeros(1)
        transl = torch.stack([xs, torch.randn(G, generator=g) * 0.1, 6.0 + torch.rand(G, generator=g)], dim=1)
        if dataset == "bedlam" and img == 1:
            transl[2] = transl[1] + torch.tensor([0.0005, 0.0, 0.0])  # same head patch as person 1
        p = _smplx_params(g, G)
        y = {"K": K.clone(), "valid_humans": torch.ones(1, G)}
        if dataset == "3dpw":
            y.update(smpl_root_pose=p["root"].reshape(1, G, 1, 3), smpl_body_pose=(torch.randn(1, G, 23, 3, generator=g) * 0.15),
                     smpl_shape=torch.randn(1, G, 10, generator=g) * 0.8, smpl_transl=transl.reshape(1, G, 3),
                     smpl_gender_id=torch.tensor([[1, 2, 2][:G]]))
        elif dataset == "ehf":
            with torch.no_grad():
                v = body(betas=p["betas"], global_orient=p["root"].reshape(G, 3), body_pose=p["body"].reshape(G, 63),
                         left_hand_pose=p["lhand"].reshape(G, 45), right_hand_pose=p["rhand"].reshape(G, 45),
                         jaw_pose=p["jaw"].reshape(G, 3), leye_pose=p["leye"].reshape(G, 3),
                         reye_pose=p["reye"].reshape(G, 3), transl=transl).vertices
            y["smplx_vertices"] = v.reshape(1, -1, 3)
        else:
            y.update(smplx_root_pose=p["root"].reshape(1, G, 1, 3), smplx_body_pose=p["body"].reshape(1, G, 21, 3),
                     smplx_jaw_pose=p["jaw"].reshape(1, G, 1, 3), smplx_leye_pose=p["leye"].reshape(1, G, 1, 3),
                     smplx_reye_pose=p["reye"].reshape(1, G, 1, 3),
                     smplx_left_hand_pose=p["lhand"].reshape(1, G, 15, 3),
                     smplx_right_hand_pose=p["rhand"].reshape(1, G, 15, 3), smplx_shape=p["betas"].reshape(1, G, 11),
                     smplx_transl=transl.reshape(1, G, 3))
        # predictions: all but the last ground truth of the last image (a miss), noisy, plus one far-away false positive
        keep = list(range(G - 1 if img == last else G))
        n = len(keep) + 1
        q = {k: torch.cat([v[keep] + torch.randn(v[keep].shape, generator=g) * 0.03,
                           torch.randn((1,) + v.shape[1:], generator=g) * 0.1]) for k, v in p.items()}
        pt = torch.cat([transl[keep] + torch.randn(len(keep), 3, generator=g) * 0.02, torch.tensor([[4.5, -1.0, 7.0]])])
        with torch.no_grad():
            out = body(betas=q["betas"], global_orient=q["root"].reshape(n, 3), body_pose=q["body"].reshape(n, 63),
                       left_hand_pose=q["lhand"].reshape(n, 45), right_hand_pose=q["rhand"].reshape(n, 45),
                       jaw_pose=q["jaw"].reshape(n, 3), leye_pose=q["leye"].reshape(n, 3),
                       reye_pose=q["reye"].reshape(n, 3), transl=pt)
        j2d = perspective_projection(out.joints, K.expand(n, 3, 3))
        order = torch.randperm(n, generator=g).tolist()
        persons = [dict(v3d=out.vertices[i], j3d=out.joints[i], j2d=j2d[i], transl_pelvis=out.joints[i, 0:1])
                   for i in order]
        cases.append((torch.zeros(1, 3, S, S), y, persons))
    return cases
