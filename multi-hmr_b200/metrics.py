"""Evaluation metrics on the device (SURVEY.md §8f row 3): host-side mirror of what the reference's
`Trainer.evaluate` (train.py:336-482) does with the persons returned by `Model.forward`, over the C-ABI entry points
`mhmr_eval_match_2d` / `mhmr_eval_points_error` / `mhmr_eval_regress` (csrc/metrics.cu) and the ground-truth body
models `mhmr_body_*` (csrc/body.cu).  The matched pairs stay on the device between the kernels; the host reads back
a few small tensors per image.

The three protocols of the reference README ("Evaluating BEDLAM-val / EHF-test / 3DPW-test"):
  BEDLAM  ground truth = SMPL-X parameters (11 betas) -> `BodyModel(kind='smplx')`; PVE / PA-PVE on 10475 vertices
  EHF     ground truth = SMPL-X vertices, joints = J_regressor @ vertices; PVE / PA-PVE
  3DPW    ground truth = SMPL parameters (male / female) -> `BodyModel(kind='smpl')`; predictions moved to the SMPL
          mesh by the SMPL-X -> SMPL transfer matrix; PVE / PA-PVE on 6890 vertices, MPJPE / PA-MPJPE on the 14
          H36M joints of J_regressor_h36m"""
from __future__ import annotations

import math

import torch

from . import _lib
from ._lib import call, stream
from .model import BODY_TABLES, body_model_arrays

# train.py:402-403 (SPIN's constants.py): the 14 LSP joints of the 17 H36M joints
H36M_TO_J17 = [6, 5, 4, 1, 2, 3, 16, 15, 14, 11, 12, 13, 8, 10, 0, 7, 9]
H36M_TO_J14 = H36M_TO_J17[:14]
SMPL_NUM_VERTS = 6890
# Trainer.evaluate's meters in their order (train.py:341-343)
EVAL_METERS = ("pve", "pa_pve", "precision", "recall", "f1_score", "mpjpe", "pa_mpjpe")


class AverageMeter:
    """utils/training.py:196-221."""

    def __init__(self, name):
        self.name, self.sum, self.count, self.val, self.avg = name, 0.0, 0, 0.0, 0.0

    def update(self, val, n=1):
        self.val = float(val)
        self.sum += float(val) * n
        self.count += n
        self.avg = self.sum / self.count


def compute_prf1(count, miss, fp):
    """utils/training.py:9-23 (host arithmetic on three integers)."""
    if count == 0:
        return 0, 0, 0
    tp, fn = count - miss, miss
    if tp == 0:
        return 0.0, 0.0, 0.0
    f1 = round(tp / (tp + 0.5 * (fp + fn)), 2)
    recall = round(tp / (tp + fn), 2)
    precision = round(tp / (tp + fp), 2)
    return 100.0 * precision, 100.0 * recall, 100.0 * f1


def match_2d_greedy(pred_j2d: torch.Tensor, gt_j2d: torch.Tensor, valid_mask: torch.Tensor | None = None,
                    iou_thresh: float = 0.05):
    """utils/training.py:25-147 on the device.  pred_j2d [P,J,2], gt_j2d [G,J,2] (CUDA, fp32).  Returns device tensors
    (pairs [min(P,G),2] int32, n_pairs [1] int32, pred_to_gt [P] int32, gt_to_pred [G] int32)."""
    dev = gt_j2d.device
    assert dev.type == "cuda", "the evaluation kernels need CUDA tensors (no CPU fallback)"
    P, G, J = int(pred_j2d.shape[0]), int(gt_j2d.shape[0]), int(gt_j2d.shape[1])
    pred = pred_j2d.to(dev, torch.float32)[:, :J].contiguous() if P else torch.zeros(0, J, 2, device=dev)
    gt = gt_j2d.to(torch.float32).contiguous()
    vm = valid_mask.to(dev, torch.uint8).contiguous() if valid_mask is not None else None
    pairs = torch.full((max(1, min(P, G)), 2), -1, device=dev, dtype=torch.int32)
    n_pairs = torch.zeros(1, device=dev, dtype=torch.int32)
    p2g = torch.full((max(P, 1),), -1, device=dev, dtype=torch.int32)
    g2p = torch.full((G,), -1, device=dev, dtype=torch.int32)
    with torch.cuda.device(dev):
        call("mhmr_eval_match_2d", pred, gt, vm, P, G, J, iou_thresh, pairs, n_pairs, p2g, g2p, stream(dev))
    return pairs, n_pairs, p2g[:P], g2p


def points_error(pred, gt, pairs, n_pairs, pred_center=None, gt_center=None):
    """Mean point error (mm) and Procrustes-aligned mean point error (mm) of the matched pairs
    (train.py:387-394, :419-427).  pred [P,n,3], gt [G,n,3]; returns two device tensors [pairs.shape[0]]."""
    dev = gt.device
    n = int(gt.shape[1])
    assert pred.shape[1] == n, "prediction and ground truth need the same number of points"
    M = int(pairs.shape[0])
    c = lambda t: None if t is None else t.to(dev, torch.float32).reshape(-1, 3).contiguous()
    pred, gt = pred.to(dev, torch.float32).contiguous(), gt.to(torch.float32).contiguous()
    pc, gc = c(pred_center), c(gt_center)
    err = torch.zeros(M, device=dev)
    pa = torch.zeros(M, device=dev)
    with torch.cuda.device(dev):
        call("mhmr_eval_points_error", pred, pc, gt, gc, pairs, n_pairs, M, n, err, pa, stream(dev))
    return err, pa


class CSR:
    """A [R, N] in compressed-sparse-row form on the device (built once at load time on the host with torch).
    `A` is a dense array / tensor or a torch sparse tensor; explicit zeros are dropped."""

    def __init__(self, A, device="cuda"):
        A = A if isinstance(A, torch.Tensor) else torch.as_tensor(A)
        A = A.detach().to("cpu", torch.float32)
        S = A.coalesce().to_sparse_csr() if A.layout == torch.sparse_coo else A.to_sparse_csr()
        self.shape = (int(S.shape[0]), int(S.shape[1]))
        dev = torch.device(device)
        self.rowptr = S.crow_indices().to(dev, torch.int32).contiguous()
        self.col = S.col_indices().to(dev, torch.int32).contiguous()
        self.val = S.values().to(dev, torch.float32).contiguous()

    def to_dense(self) -> torch.Tensor:
        return torch.sparse_csr_tensor(self.rowptr.long().cpu(), self.col.long().cpu(), self.val.cpu(),
                                       size=self.shape).to_dense()


def regress(A: CSR, X, pairs, n_pairs, side: int, center=None, rows=None, root: int = -1, K=None):
    """out[m] = A[rows] . (X[s] - center[s]) (minus the root row's result when root >= 0), s = pairs[m, side], for the
    matched pairs m < n_pairs still on the device (`mhmr_eval_regress`).  X [*, N, 3]; returns out [M, R_out, 3] and,
    when K [*, 3, 3] is given, the projection out2d [M, R_out, 2]."""
    dev = X.device
    R, N = A.shape
    assert X.shape[1] == N, f"regressor takes {N} points, got {X.shape[1]}"
    M = int(pairs.shape[0])
    X = X.to(torch.float32).contiguous()
    c = None if center is None else center.to(dev, torch.float32).reshape(-1, 3).contiguous()
    if rows is not None:
        rows = torch.as_tensor(rows, dtype=torch.int64).reshape(-1)
        if rows.numel() == 0 or int(rows.min()) < 0 or int(rows.max()) >= R:
            raise ValueError(f"regressor rows must lie in [0, {R})")
    r = None if rows is None else rows.to(dev, torch.int32).contiguous()
    R_out = R if r is None else int(r.numel())
    out = torch.zeros(M, R_out, 3, device=dev)
    Kd = None if K is None else K.to(dev, torch.float32).reshape(-1, 9).contiguous()
    out2d = None if K is None else torch.zeros(M, R_out, 2, device=dev)
    with torch.cuda.device(dev):
        call("mhmr_eval_regress", A.rowptr, A.col, A.val, R, N, r, R_out, root, X, c, pairs, side, n_pairs, M, Kd, out,
             out2d, stream(dev))
    return out, out2d


class BodyModel:
    """The raw `smplx` body model on the device (`mhmr_body_*`), as Trainer.prepare_gt calls it (train.py:41-43,
    :76-109): kind 'smpl' (24 joints, output joints 24 + 21 vertex-picked) or 'smplx' (55 joints, `num_betas`
    default 11, flat_hand_mean, 127 output joints).  `bm` is a body-model dict as made by `synth.make_body_model` /
    `synth.make_smpl_body_model` or read by `api.body_model_from_smplx_npz` / `api.body_model_from_smpl_pkl`."""

    def __init__(self, bm: dict, kind: str, num_betas: int | None = None, max_persons: int = 48, device="cuda"):
        assert kind in ("smpl", "smplx"), kind
        dev = torch.device(device)
        self.kind, self.device, self.max_persons = kind, dev, int(max_persons)
        nb = int(num_betas if num_betas is not None else (11 if kind == "smplx" else 10))
        arrays = {k: torch.as_tensor(v).to(dev, torch.int32 if k in BODY_TABLES else torch.float32).contiguous()
                  for k, v in body_model_arrays(bm, nb, landmarks=kind == "smplx").items()}
        V = int(arrays["v_template"].shape[0])
        self.num_verts, self.num_betas = V, nb
        keys = ("v_template", "shapedirs", "expr_dirs", "posedirs", "J_regressor", "lbs_weights", "parents",
                "extra_joints_idxs", "lmk_tri", "lmk_bary_coords")
        h = torch.zeros(1, dtype=torch.int64)
        with torch.cuda.device(dev):
            call("mhmr_body_create", 1 if kind == "smplx" else 0, V, nb, self.max_persons,
                 *(arrays.get(k) for k in keys), stream(dev), h)
        self._h = h.item()
        self._lib = _lib.load()
        nj_out, nj = torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32)
        call("mhmr_body_info", self._h, None, nj_out, nj, None, None)
        self.num_joints, self.num_pose_joints = nj_out.item(), nj.item()
        # smplx J_regressor (EHF joints = J_regressor @ vertices, train.py:73)
        self.j_regressor = CSR(bm["J_regressor"], dev)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._lib.mhmr_body_destroy(h)
            self._h = None

    def __call__(self, full_pose, betas, transl, K, expression=None):
        """full_pose [P, num_pose_joints, 3] (smplx order), betas [P, num_betas], transl [P, 3], K [P, 3, 3],
        expression [P, 10] (SMPL-X; zeros when None).  Returns v3d [P,V,3], j3d [P,J,3], j2d [P,J,2],
        transl_pelvis [P,3] on the device.  Differentiable in full_pose, betas, transl and expression when grad mode
        is on and one of them requires grad (`mhmr_body_backward`); gradients with respect to K are not provided."""
        P = int(betas.shape[0])
        if P > self.max_persons:
            raise ValueError(f"{P} persons > max_persons {self.max_persons}")
        if torch.is_grad_enabled():
            if isinstance(K, torch.Tensor) and K.requires_grad:
                raise NotImplementedError("BodyModel: gradients with respect to K are not provided")
            if any(isinstance(t, torch.Tensor) and t.requires_grad for t in (full_pose, betas, transl, expression)):
                v3d, j3d, j2d, tp = _BodyFunction.apply(self, K, full_pose, betas, transl, expression)
                return dict(v3d=v3d, j3d=j3d, j2d=j2d, transl_pelvis=tp)
        return self._forward(*self._inputs(full_pose, betas, transl, K, expression))

    def _inputs(self, full_pose, betas, transl, K, expression):
        dev, P = self.device, int(betas.shape[0])
        f = lambda t, n: t.detach().to(dev, torch.float32).reshape(P, n).contiguous()
        fp = f(full_pose, self.num_pose_joints * 3)
        b = f(betas, self.num_betas)
        tr = f(transl, 3)
        Kd = f(K, 9)
        ex = None
        if self.kind == "smplx":
            ex = f(expression, 10) if expression is not None else torch.zeros(P, 10, device=dev)
        return fp, b, tr, Kd, ex

    def _forward(self, fp, b, tr, Kd, ex, want_v2d=False):
        dev, P = self.device, int(b.shape[0])
        V, J = self.num_verts, self.num_joints
        out = dict(v3d=torch.empty(P, V, 3, device=dev), j3d=torch.empty(P, J, 3, device=dev),
                   j2d=torch.empty(P, J, 2, device=dev), transl_pelvis=torch.empty(P, 3, device=dev))
        if want_v2d:
            out["v2d"] = torch.empty(P, V, 2, device=dev)
        with torch.cuda.device(dev):
            call("mhmr_body_forward", self._h, P, fp, b, ex, tr, Kd, out["v3d"], out.get("v2d"), out["j3d"],
                 out["j2d"], out["transl_pelvis"], stream(dev))
        return out

    def _backward(self, fp, b, tr, Kd, ex, g_v3d=None, g_v2d=None, g_j3d=None, g_j2d=None, g_transl_pelvis=None):
        """`mhmr_body_backward` on converted inputs (see `_inputs`) and fp32 upstream gradients (each None = zero).
        Returns d_full_pose [P, NJ*3], d_betas [P, num_betas], d_expression [P, 10] (SMPL-X, else None), d_transl."""
        dev, P = self.device, int(b.shape[0])
        g = lambda t: None if t is None else t.to(dev, torch.float32).contiguous()
        d_fp, d_b, d_tr = torch.empty_like(fp), torch.empty_like(b), torch.empty_like(tr)
        d_ex = torch.empty(P, 10, device=dev) if ex is not None else None
        with torch.cuda.device(dev):
            call("mhmr_body_backward", self._h, P, fp, b, ex, tr, Kd, g(g_v3d), g(g_v2d), g(g_j3d), g(g_j2d),
                 g(g_transl_pelvis), d_fp, d_b, d_ex, d_tr, stream(dev))
        return d_fp, d_b, d_ex, d_tr


def _grad_like(d, t):
    """A computed gradient in the shape, dtype and device of the input `t` it belongs to."""
    return d.reshape(t.shape).to(device=t.device, dtype=t.dtype)


class _BodyFunction(torch.autograd.Function):
    """BodyModel.__call__ with gradients: forward = `mhmr_body_forward`, backward = `mhmr_body_backward`."""

    @staticmethod
    def forward(ctx, body, K, full_pose, betas, transl, expression):
        ctx.set_materialize_grads(False)
        x = body._inputs(full_pose, betas, transl, K, expression)
        out = body._forward(*x)
        ctx.body, ctx.x = body, x
        ctx.orig = (full_pose, betas, transl, expression)
        return out["v3d"], out["j3d"], out["j2d"], out["transl_pelvis"]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_v3d, g_j3d, g_j2d, g_tp):
        d_fp, d_b, d_ex, d_tr = ctx.body._backward(*ctx.x, g_v3d=g_v3d, g_j3d=g_j3d, g_j2d=g_j2d,
                                                   g_transl_pelvis=g_tp)
        full_pose, betas, transl, expression = ctx.orig
        need = ctx.needs_input_grad
        grads = [_grad_like(d_fp, full_pose) if need[2] else None, _grad_like(d_b, betas) if need[3] else None,
                 _grad_like(d_tr, transl) if need[4] else None,
                 _grad_like(d_ex, expression) if need[5] and expression is not None and d_ex is not None else None]
        return (None, None, *grads)


def _center_index(person_center) -> int:
    from .model import KINEMATIC_JOINTS

    return person_center if isinstance(person_center, int) else KINEMATIC_JOINTS.index(person_center)


def _gt_bodies(y: dict, body_models, want_v2d: bool = False):
    """The ground-truth body forward of Trainer.prepare_gt (train.py:61-112) on the valid persons of `y`:
    (idx_h, outputs {'v3d', 'j3d', 'j2d', 'transl_pelvis'} (+ 'v2d' with want_v2d)), or None when `y` holds no persons'
    annotation."""
    valid_h = y["valid_humans"]
    idx_h = torch.where(valid_h)
    nhv = int(valid_h.sum())
    K = y["K"][idx_h[0]]

    def run(bm, *args):
        return bm._forward(*bm._inputs(*args, None), want_v2d=True) if want_v2d else bm(*args)

    if "smplx_vertices" in y:
        verts = y["smplx_vertices"].reshape(1, -1, 3).to(torch.float32).contiguous()
        bm = body_models["smplx"]
        one = torch.tensor([[0, 0]], dtype=torch.int32, device=verts.device)
        n = torch.ones(1, dtype=torch.int32, device=verts.device)
        jts, j2d = regress(bm.j_regressor, verts, one, n, side=1, K=K[:1])
        out = dict(v3d=verts, j3d=jts, j2d=j2d, transl_pelvis=jts[:, 0].contiguous())
        if want_v2d:
            out["v2d"] = _project(verts, K[:1])
    elif "smpl_root_pose" in y:
        sel = lambda k, n: y[k][idx_h[0], idx_h[1]].reshape(nhv, n)
        full_pose = torch.cat([sel("smpl_root_pose", 3), sel("smpl_body_pose", 23 * 3)], dim=1)
        args = (full_pose, sel("smpl_shape", 10), sel("smpl_transl", 3), K)
        out = run(body_models["smpl_male"], *args)
        if int(y["smpl_gender_id"].max()) == 2:
            fem = run(body_models["smpl_female"], *args)
            idx = torch.where(y["smpl_gender_id"] == 2)[1]
            for k in out:
                out[k][idx] = fem[k][idx]
    elif "smplx_root_pose" in y:
        sel = lambda k, n: y[k][idx_h[0], idx_h[1]].reshape(nhv, n)
        # smplx full_pose order: global, body 21, jaw, leye, reye, left hand 15, right hand 15
        full_pose = torch.cat([sel("smplx_root_pose", 3), sel("smplx_body_pose", 21 * 3), sel("smplx_jaw_pose", 3),
                               sel("smplx_leye_pose", 3), sel("smplx_reye_pose", 3),
                               sel("smplx_left_hand_pose", 15 * 3), sel("smplx_right_hand_pose", 15 * 3)], dim=1)
        out = run(body_models["smplx"], full_pose, sel("smplx_shape", 11), sel("smplx_transl", 3), K)
    else:
        return None
    return idx_h, out


def _one_per_patch(idx_h, pk_loc, img_size: int, patch_size: int):
    """One person per patch of the primary keypoint (train.py:137-157): (kept persons in order, their patch
    (x, y) indices [n, 2] as a host list); the patch indices come to the host once."""
    n_patch = img_size // patch_size
    pk_idx = torch.clamp((pk_loc // patch_size).int(), 0, n_patch - 1).cpu().tolist()
    taken, keep = set(), []
    for k in range(len(pk_idx)):
        cell = (int(idx_h[0][k]), pk_idx[k][1], pk_idx[k][0])
        if cell not in taken:
            taken.add(cell)
            keep.append(k)
    return keep, pk_idx


def _project(x, K):
    """utils/camera.py:14-27 perspective_projection: x [P, N, 3], K [P, 3, 3] -> [P, N, 2]."""
    y = x / x[:, :, -1:]
    return torch.einsum("bij,bkj->bki", K, y)[:, :, :2]


def _rotvec_to_rotmat(rv):
    """roma.rotvec_to_rotmat (first order below 1e-6 rad): [..., 3] -> [..., 3, 3]."""
    shape = rv.shape[:-1]
    rv = rv.reshape(-1, 3)
    theta = rv.norm(dim=-1)
    axis = rv / theta.clamp_min(1e-6)[:, None]
    kx, ky, kz = axis.unbind(-1)
    s, omc = torch.sin(theta), 1 - torch.cos(theta)
    R = torch.stack([1 - (ky * ky + kz * kz) * omc, kx * ky * omc - kz * s, kx * kz * omc + ky * s,
                     kx * ky * omc + kz * s, 1 - (kx * kx + kz * kz) * omc, ky * kz * omc - kx * s,
                     kx * kz * omc - ky * s, ky * kz * omc + kx * s, 1 - (kx * kx + ky * ky) * omc], -1)
    x, y_, z = rv.unbind(-1)
    o = torch.ones_like(x)
    first = torch.stack([o, -z, y_, z, o, -x, -y_, x, o], -1)
    R = torch.where((theta < 1e-6)[:, None], first, R)
    return R.reshape(*shape, 3, 3)


def prepare_gt(y: dict, body_models, person_center="head", *, img_size: int, patch_size: int = 14):
    """What Trainer.evaluate reads from Trainer.prepare_gt (train.py:58-182): {'K', 'j2d', 'v3d', 'transl_pelvis', 'j3d'}
    for a batch `y` in the reference's collate_fn format, on the device.  body_models maps 'smpl_male', 'smpl_female'
    and 'smplx' to `BodyModel`s (an `EvalAssets` works).  Input kinds:
      smplx_vertices  EHF: the vertices themselves, joints = smplx J_regressor @ vertices (:70-73)
      smpl_*          3DPW: SMPL male, replaced by SMPL female for persons with smpl_gender_id == 2 (:74-94)
      smplx_*         BEDLAM: SMPL-X neutral, 11 betas, eyes and jaw included, expression zero (:95-110)
    Persons whose `person_center` joint falls on a patch already taken by an earlier person are dropped (:137-180).
    Returns None when `y` holds none of the three (an image without annotated persons)."""
    r = _gt_bodies(y, body_models)
    if r is None:
        return None
    idx_h, out = r
    keep, _ = _one_per_patch(idx_h, out["j2d"][:, _center_index(person_center)], img_size, patch_size)
    dev = out["v3d"].device
    keep = torch.tensor(keep, dtype=torch.long, device=dev)
    gt = {k: v[keep].contiguous() for k, v in out.items()}
    gt["K"] = y["K"]
    return gt


def prepare_train_targets(y: dict, body_models, person_center="head", *, img_size: int, patch_size: int = 14):
    """The training targets of Trainer.prepare_gt (train.py:58-182, its `_target` dict) on the device: 'idx'
    (batch, patch y, patch x, 0) of the kept persons, 'scores' [B, res, res] (1 at their patches), 'K', and per kept
    person 'transl' (the person_center joint), 'transl_pelvis', 'dist', 'dist_postprocessed' (log depth normalised
    by the focal length, fovn 60 at img_size), 'v3d', 'j3d', 'j2d', 'v2d', 'loc' (projected centre joint), 'offset'
    (from the patch centre, in patches), and for SMPL-X parameters (BEDLAM) 'rotvec' / 'rotmat' [P, 53, ...] in the
    model's order root, body 21, left hand 15, right hand 15, jaw, and 'shape'.  Input kinds and the one-person-per-
    patch rule as in `prepare_gt`; None when `y` holds no annotation."""
    r = _gt_bodies(y, body_models, want_v2d=True)
    if r is None:
        return None
    idx_h, out = r
    B = y["valid_humans"].shape[0]
    jts = out["j3d"]
    dev = jts.device
    c = _center_index(person_center)
    K = y["K"][idx_h[0]].to(dev, torch.float32)
    tgt = dict(transl=jts[:, c], transl_pelvis=jts[:, 0], dist=jts[:, 0, 2])
    fn = img_size / (2 * math.tan(math.radians(60) / 2))        # utils/camera.py:50-61, fovn 60
    tgt["dist_postprocessed"] = torch.log(tgt["dist"] + 1e-10) * (fn / K[:, 0, 0])
    tgt.update(v3d=out["v3d"], j3d=jts, j2d=out["j2d"], v2d=out["v2d"])
    pk_loc = out["j2d"][:, c]
    keep, pk_idx = _one_per_patch(idx_h, pk_loc, img_size, patch_size)
    pk = torch.tensor(pk_idx, dtype=torch.float32, device=dev).reshape(-1, 2)
    tgt["loc"] = pk_loc
    tgt["offset"] = (pk_loc - (pk + 0.5) * patch_size) / patch_size
    if "smplx_root_pose" in y:
        sel = lambda k: y[k][idx_h[0], idx_h[1]].reshape(len(idx_h[0]), -1, 3).to(dev, torch.float32)
        tgt["rotvec"] = torch.cat([sel("smplx_root_pose"), sel("smplx_body_pose"), sel("smplx_left_hand_pose"),
                                   sel("smplx_right_hand_pose"), sel("smplx_jaw_pose")], 1)
        tgt["rotmat"] = _rotvec_to_rotmat(tgt["rotvec"])
        tgt["shape"] = y["smplx_shape"][idx_h[0], idx_h[1]].to(dev, torch.float32)
    keep_t = torch.tensor(keep, dtype=torch.long, device=dev)
    n_patch = img_size // patch_size
    scores = torch.zeros(B, n_patch, n_patch, device=dev)
    cells = pk.long()[keep_t] if keep else torch.zeros(0, 2, dtype=torch.long, device=dev)
    b = idx_h[0].to(dev)[keep_t]
    scores[b, cells[:, 1], cells[:, 0]] = 1.0
    targets = {"idx": (b, cells[:, 1], cells[:, 0], torch.zeros_like(b)), "scores": scores, "K": y["K"]}
    for k, v in tgt.items():
        targets[k] = v[keep_t].contiguous()
    return targets


class Evaluator:
    """The accumulation loop of `Trainer.evaluate` (train.py:336-482) for predictions in the reference's person-dict
    format (model.py:329-347) and ground truths {j2d [G,J,2], v3d [G,V,3], transl_pelvis [G,1,3]}.

    smplx2smpl: the SMPL-X -> SMPL transfer matrix [6890, 10475] (`smplx2smpl.pkl['matrix']`), needed when the ground
    truth is an SMPL mesh (3DPW): the centred predictions are moved to it before the errors (train.py:383-384).
    j_regressor_h36m: [17, 6890]; adds the 3DPW meters mpjpe / pa_mpjpe on the 14 H36M joints (train.py:396-429).
    Per-pair values are kept in `values` in the order the meters saw them."""

    def __init__(self, smplx2smpl=None, j_regressor_h36m=None, device="cuda"):
        keys = ["pve", "pa_pve", "precision", "recall", "f1_score"]
        as_csr = lambda A: A if A is None or isinstance(A, CSR) else CSR(A, device)
        self.smplx2smpl, self.j_regressor_h36m = as_csr(smplx2smpl), as_csr(j_regressor_h36m)
        if self.j_regressor_h36m is not None:
            keys += ["mpjpe", "pa_mpjpe"]
        self.meters = {k: AverageMeter(k) for k in keys}
        self.values = {k: [] for k in keys if k not in ("precision", "recall", "f1_score")}
        self.count = self.miss = self.fp = 0

    def _update(self, key, vals):
        for v in vals:
            self.meters[key].update(v)
            self.values[key].append(v)

    def update(self, persons: list, gt: dict):
        G = int(gt["j2d"].shape[0])
        dev = gt["j2d"].device
        if len(persons):
            pj = torch.stack([p["j2d"] for p in persons])
            pv = torch.stack([p["v3d"] for p in persons])
            pp = torch.stack([p["transl_pelvis"].reshape(3) for p in persons])
        else:
            pj, pv, pp = torch.zeros(0, gt["j2d"].shape[1], 2, device=dev), None, None
        pairs, n_pairs, p2g, g2p = match_2d_greedy(pj, gt["j2d"])
        Vg = int(gt["v3d"].shape[1])
        smpl_gt = len(persons) and Vg == SMPL_NUM_VERTS and pv.shape[1] != Vg
        if smpl_gt and self.smplx2smpl is None:
            raise ValueError("the ground truth is an SMPL mesh (6890 vertices): construct the Evaluator with "
                             "smplx2smpl= (smplx2smpl.pkl['matrix']) to move the predictions onto it")
        if self.j_regressor_h36m is not None and len(persons) and Vg != SMPL_NUM_VERTS:
            raise ValueError("MPJPE uses J_regressor_h36m, which takes SMPL meshes (6890 vertices)")
        if len(persons):
            M = int(pairs.shape[0])
            if smpl_gt:
                # centre, then regress (train.py:375-384); pair m of the regressed meshes is row m
                pv_s, _ = regress(self.smplx2smpl, pv, pairs, n_pairs, side=0, center=pp)
                ar = torch.arange(M, dtype=torch.int32, device=dev)
                pairs_s = torch.stack([ar, pairs[:, 1]], dim=1).contiguous()
                pve, pa = points_error(pv_s, gt["v3d"], pairs_s, n_pairs, None, gt["transl_pelvis"])
            else:
                pve, pa = points_error(pv, gt["v3d"], pairs, n_pairs, pp, gt["transl_pelvis"])
            if self.j_regressor_h36m is not None:
                ar = torch.arange(M, dtype=torch.int32, device=dev)
                same = torch.stack([ar, ar], dim=1).contiguous()
                j14 = H36M_TO_J14
                src = pv_s if smpl_gt else pv
                src_pairs, src_c = (same, None) if smpl_gt else (pairs, pp)
                h_hat, _ = regress(self.j_regressor_h36m, src, src_pairs, n_pairs, 0, src_c, rows=j14, root=0)
                h_gt, _ = regress(self.j_regressor_h36m, gt["v3d"], pairs, n_pairs, 1, gt["transl_pelvis"],
                                  rows=j14, root=0)
                mpjpe, pa_mpjpe = points_error(h_hat, h_gt, same, n_pairs)
        n = int(n_pairs.item())  # the one host read-back of the image
        self.count += G
        self.miss += G - n
        self.fp += len(persons) - n
        if n:
            self._update("pve", pve[:n].tolist())
            self._update("pa_pve", pa[:n].tolist())
            if self.j_regressor_h36m is not None:
                self._update("mpjpe", mpjpe[:n].tolist())
                self._update("pa_mpjpe", pa_mpjpe[:n].tolist())
        return pairs[:n]

    def summary(self) -> dict:
        precision, recall, f1 = compute_prf1(self.count, self.miss, self.fp)
        out = {k: m.avg for k, m in self.meters.items() if k not in ("precision", "recall", "f1_score")}
        out.update(precision=precision, recall=recall, f1_score=f1)
        return out


class EvalAssets:
    """The three ground-truth body models and two regressors an evaluation holds (train.py:41-45, :400), on one
    device: body-model dicts for SMPL-X neutral (11 betas), SMPL male and SMPL female; the SMPL-X -> SMPL transfer
    matrix [6890, 10475] and J_regressor_h36m [17, 6890] (dense or torch sparse)."""

    def __init__(self, smplx_bm: dict, smpl_male_bm: dict, smpl_female_bm: dict, smplx2smpl, j_regressor_h36m,
                 device="cuda", max_persons: int = 48):
        self.body_models = {
            "smplx": BodyModel(smplx_bm, "smplx", 11, max_persons, device),
            "smpl_male": BodyModel(smpl_male_bm, "smpl", 10, max_persons, device),
            "smpl_female": BodyModel(smpl_female_bm, "smpl", 10, max_persons, device),
        }
        self.smplx2smpl = CSR(smplx2smpl, device)
        self.j_regressor_h36m = CSR(j_regressor_h36m, device)
        self.device = torch.device(device)

    def __getitem__(self, k):
        return self.body_models[k]

    @classmethod
    def from_dir(cls, models_dir: str = "models", device="cuda", max_persons: int = 48):
        """models/smplx/SMPLX_NEUTRAL.npz, models/smpl/SMPL_{MALE,FEMALE}.pkl, models/smplx/smplx2smpl.pkl and
        models/smpl/J_regressor_h36m.npy -- the reference's layout (utils/constants.py, train.py:400)."""
        import os

        from . import api

        j = lambda *p: os.path.join(models_dir, *p)
        return cls(api.body_model_from_smplx_npz(j("smplx", "SMPLX_NEUTRAL.npz"), num_betas=10),
                   api.body_model_from_smpl_pkl(j("smpl", "SMPL_MALE.pkl")),
                   api.body_model_from_smpl_pkl(j("smpl", "SMPL_FEMALE.pkl")),
                   api.load_smplx2smpl(j("smplx", "smplx2smpl.pkl")),
                   api.load_j_regressor_h36m(j("smpl", "J_regressor_h36m.npy")), device, max_persons)


@torch.no_grad()
def evaluate(model, data, assets: EvalAssets, dataset: str, det_thresh: float = 0.3, nms_kernel_size: int = 3,
             person_center="head") -> dict:
    """The loop of `Trainer.evaluate` (train.py:336-482) over an iterable of (x, y) in the reference's collate_fn
    format (batch size 1, train.py:506): prepare the ground truth, run `model(x, K=..., det_thresh, nms_kernel_size)`,
    match, accumulate.  `dataset` is the reference's `data.dataset.name`: MPJPE / PA-MPJPE only for '3dpw' (:397).
    Returns the reference's final meters {pve, pa_pve, precision, recall, f1_score, mpjpe, pa_mpjpe} (.avg; meters
    that saw nothing stay 0); the Evaluator with its per-pair values is in the `evaluator` key."""
    dev = assets.device
    ev = Evaluator(assets.smplx2smpl, assets.j_regressor_h36m if dataset == "3dpw" else None, dev)
    for x, y in data:
        y = {k: v.to(dev) if isinstance(v, torch.Tensor) else v for k, v in y.items()}
        gt = prepare_gt(y, assets.body_models, person_center, img_size=int(x.shape[-1]))
        if gt is None:
            raise ValueError("an evaluation image without annotated persons (Trainer.evaluate needs them too)")
        persons = model(x.to(dev), is_training=False, K=gt["K"], det_thresh=det_thresh,
                        nms_kernel_size=nms_kernel_size)
        ev.update(persons, gt)
    s = ev.summary()
    out = {k: float(s.get(k, 0.0)) for k in EVAL_METERS}
    out["evaluator"] = ev
    return out
