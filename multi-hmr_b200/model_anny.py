"""Host-side mirror of the reference's Anny variant `Multi_HMR` (multi_hmr_anny/multi_hmr.py) over libmhmr_sm90.so.

Same constructor keywords, same `forward(x, K=None, idx=None, is_training=False, det_thresh, nms_kernel_size)` and
return conventions (flat dict when `is_training=True`; otherwise the person list sorted by depth, or `({}, [])` when
nothing is detected).  Everything before the body model (backbone, detection, field of view, decoder, regressors) and
after it (centre bone, translation, projection) runs in the sm_90a kernels behind `mhmr_forward_anny` /
`mhmr_anny_place`.  The body model itself is the PyTorch module it is given: the `anny` package's full-body model
(`anny.create_fullbody_model`), or any object with the same interface.
"""
from __future__ import annotations

import torch

from ._lib import call, stream
from .model import ARCH_ID, PATCH_SIZE, _EngineModel

ANNY_SHAPE_KEYS = ("age", "gender", "weight", "height", "muscle", "proportions")   # multi_hmr.py:171
HEAD_ANNY = 1


def create_anny_body_model():
    """The body model the reference builds (multi_hmr.py:70, :76): needs the `anny` package."""
    try:
        import anny
    except ImportError as err:
        raise ImportError("the Anny variant needs the `anny` package for its body model (or pass body_model=...)") from err
    bm = anny.create_fullbody_model(remove_unattached_vertices=False, all_phenotypes=True).to(dtype=torch.float32)
    bm.set_skinning_method("lbs")
    return bm


class ModelAnny(_EngineModel):
    """H100-native drop-in for reference `multi_hmr_anny.multi_hmr.Multi_HMR` (inference path)."""

    _IGNORED_PREFIX = "body_model."   # the body model's own buffers
    _POS_EMBED_KEY = "encoder.backbone.pos_embed"
    _SKIPPED_KEYS = ("encoder.backbone.mask_token", "eye")
    _ENTRY = "mhmr_forward_anny"
    _OUTPUTS = "mhmr_anny_outputs"

    def __init__(self, img_size=896, backbone="dinov2_vits14", pretrained_backbone=False, xat_dim=512, xat_depth=8,
                 xat_heads=16, xat_dim_head=32, xat_mlp_dim=4 * 512, xat_dropout=0.0, person_center="head",
                 num_betas=11, default_pose_parameterization="root_relative_world", *args, max_batch=8,
                 max_persons=None, body_model=None, device=None, refine_central=True, **kwargs):
        assert kwargs.get("simple_depth_encoding") == 1                               # multi_hmr.py:41
        if isinstance(img_size, (list, tuple)):
            img_size = img_size[0]
        if backbone not in ARCH_ID:
            raise ValueError(f"unknown backbone {backbone!r}")
        assert img_size % PATCH_SIZE == 0, "Invalid img size"                           # multi_hmr.py:47
        if xat_dim_head != 32:
            raise NotImplementedError("the HPH kernels are built for xat_dim_head = 32")
        super().__init__(backbone, img_size, max_batch, max_persons, refine_central, device)
        self.xat_dim, self.xat_depth, self.xat_heads, self.xat_mlp_dim = xat_dim, xat_depth, xat_heads, xat_mlp_dim
        self.num_betas, self.person_center = num_betas, person_center
        self.body_model = (body_model if body_model is not None else create_anny_body_model()).to(self.device)
        self.person_center_idx = list(self.body_model.bone_labels).index(person_center)
        self.n_joints = len(self.body_model.bone_labels)
        self._shape_cols = [(k, l) for l, k in enumerate(self.body_model.phenotype_labels) if k in ANNY_SHAPE_KEYS]
        if any(l >= num_betas for _, l in self._shape_cols):
            raise ValueError("the body model's phenotype labels do not fit in num_betas shape outputs")

    def _head_config(self):
        return dict(xat_depth=self.xat_depth, xat_num_heads=self.xat_heads, num_betas=self.num_betas,
                    person_center_idx=self.person_center_idx, head=HEAD_ANNY, xat_dim=self.xat_dim,
                    xat_mlp_dim=self.xat_mlp_dim, num_joints=self.n_joints)

    # ------------------------------------------------------------------ forward
    def forward_raw(self, x, K=None, idx=None, det_thresh=0.3, nms_kernel_size=3, want_z=False):
        """Enqueues the forward up to the body model's inputs; returns (max_persons-sized device tensors, P)."""
        self.finalize()
        with torch.cuda.device(self.device):
            return self._forward_raw(x, K, idx, det_thresh, nms_kernel_size, want_z)

    def _forward_raw(self, x, K, idx, det_thresh, nms_kernel_size, want_z):
        dev = self.device
        x, fused = self._prepare_image(x)
        B = x.shape[0]
        if K is not None:
            K = K.to(dev, dtype=torch.float32, non_blocking=True).contiguous()
            assert K.shape == (B, 3, 3), "K must be [B,3,3]"
        Pm, J, nb, r = self.max_persons, self.n_joints, self.num_betas, self.res
        f = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)
        t = {"scores_map": f(B, r, r), "logits": f(B, r, r), "count": torch.zeros(1, device=dev, dtype=torch.int32),
             "det_idx": torch.zeros(3, Pm, device=dev, dtype=torch.int32), "K_regressed": f(B, 3, 3), "fov": f(B),
             "K_det": f(Pm, 3, 3), "offset": f(Pm, 2), "loc": f(Pm, 2), "dist": f(Pm), "dist_pp": f(Pm),
             "shape": f(Pm, nb), "rotmat": f(Pm, J, 3, 3), "rotmat_homo": f(Pm, J, 4, 4), "rotvec": f(Pm, J, 3),
             "transl": f(Pm, 3), "z": f(B, r * r, self.embed_dim) if want_z else None}
        fidx = None
        if idx is not None:
            fidx = self._forced_idx(idx[:3], B)
            if (fidx[0][1:] < fidx[0][:-1]).any():
                raise ValueError("idx must list the persons of each image contiguously, in image order")
        return t, self._run(x, fused, K, det_thresh, nms_kernel_size, fidx, t)

    def place(self, out_bm, t, P, want_v2d):
        """Body-model output -> camera space (mhmr_anny_place): v3d, j3d, j2d, v2d, transl_pelvis."""
        dev = self.device
        v3d = out_bm["vertices"].to(dev, dtype=torch.float32).contiguous().clone()
        bones = out_bm["bone_poses"].to(dev, dtype=torch.float32).contiguous()
        V, J = v3d.shape[1], bones.shape[1]
        assert J == self.n_joints, "the body model returned a different number of bones"
        f = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)
        res = {"v3d": v3d, "j3d": f(P, J, 3), "j2d": f(P, J, 2), "v2d": f(P, V, 2) if want_v2d else None,
               "transl_pelvis": f(P, 3)}
        with torch.cuda.device(dev):
            call("mhmr_anny_place", self._handle, P, V, bones, t["transl"], t["K_det"], v3d, res["j3d"], res["v2d"],
                 res["j2d"], res["transl_pelvis"], stream(dev))
        return res

    def forward(self, x, K=None, idx=None, is_training=False, det_thresh=0.3, nms_kernel_size=3, *args, **kwargs):
        """multi_hmr.py:98-246."""
        if not is_training and idx is None and nms_kernel_size > 1 and nms_kernel_size % 2 == 0:
            raise ValueError(f"nms_kernel_size={nms_kernel_size}: an even kernel changes the score map's shape in "
                             "the reference (multi_hmr.py:118-120)")
        t, P = self.forward_raw(x, K, idx=idx, det_thresh=det_thresh, nms_kernel_size=nms_kernel_size,
                                want_z=is_training)
        if P == 0 and not is_training:
            return {}, []                                                               # multi_hmr.py:123-124
        shape = t["shape"][:P]
        pheno = {k: shape[:, l] for k, l in self._shape_cols}
        out_bm = self.body_model(pose_parameters=t["rotmat_homo"][:P], phenotype_kwargs=pheno)
        pl = self.place(out_bm, t, P, want_v2d=is_training)
        B = t["fov"].shape[0]
        K_used = K.to(self.device, dtype=torch.float32) if K is not None else t["K_regressed"]
        if is_training:
            r = self.res
            return {
                "scores": t["scores_map"], "scores_logits": t["logits"], "K": K_used, "K_regressed": t["K_regressed"],
                "fov_regressed": t["fov"][:, None], "loc": t["loc"][:P], "offset": t["offset"][:P],
                "dist": t["dist"][:P, None], "dist_postprocessed": t["dist_pp"][:P, None], "shape": shape,
                "rotvec": t["rotvec"][:P], "rotmat": t["rotmat"][:P], "v3d": pl["v3d"], "j3d": pl["j3d"],
                "j2d": pl["j2d"], "v2d": pl["v2d"], "transl": t["transl"][:P],
                "transl_pelvis": pl["transl_pelvis"][:, None], "feat": t["z"].reshape(B, r, r, -1),
                "blendshape_coeffs": out_bm["blendshape_coeffs"],
            }
        b_idx = t["det_idx"][0, :P].long()
        persons = []
        for i in range(P):                                                              # multi_hmr.py:215-235
            persons.append({
                "K": t["K_det"][i], "K_regressed": t["K_regressed"][b_idx[i]], "loc": t["loc"][i],
                "transl": t["transl"][i], "transl_pelvis": pl["transl_pelvis"][i][None], "rotvec": t["rotvec"][i],
                "rotmat": t["rotmat"][i], "shape": shape[i], "v3d": pl["v3d"][i], "j3d": pl["j3d"][i],
                "j2d": pl["j2d"][i], "fov": t["fov"][:, None],
            })
        # closest first, stable (multi_hmr.py:238)
        z = t["transl"][:P, 2].tolist()
        order = sorted(range(P), key=lambda i: z[i])
        return [persons[i] for i in order]

    __call__ = forward
