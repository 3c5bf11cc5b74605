"""Host-side mirror of the reference's `Model` (reference model.py:30-349) over libmhmr_sm90.so.

Same constructor keywords, same `forward(x, idx, det_thresh, nms_kernel_size, K, is_training)` signature,
same return conventions (list of per-person dicts in inference, flat dict when `is_training=True`), same
`load_state_dict(sd, strict=False)` key names — but every tensor operation of the forward runs in the
hand-written sm_90a kernels behind the C-ABI (`mhmr_forward`).  PyTorch is used for device memory,
streams and (once, at load) the bicubic pos-embed interpolation.  There is no CPU fallback: a CUDA device
and the built extension are required, otherwise construction / forward raise.
"""
from __future__ import annotations

import ctypes
import math
from types import SimpleNamespace

import torch
import torch.nn.functional as F

from . import _lib
from ._lib import c_int, c_int64, c_void_p, check, ptr

ARCH_ID = {"dinov2_vits14": 0, "dinov2_vitb14": 1, "dinov2_vitl14": 2}
EMBED_DIM = {"dinov2_vits14": 384, "dinov2_vitb14": 768, "dinov2_vitl14": 1024}
PATCH_SIZE = 14
NUM_VERTS = 10475
# index of the 55 kinematic SMPL-X joints in smplx.joint_names.JOINT_NAMES (utils/humans.py:25-26); only
# kinematic joints can be a person centre (blocks/smpl_layer.py:41-45 looks the name up in JOINT_NAMES).
KINEMATIC_JOINTS = ["pelvis", "left_hip", "right_hip", "spine1", "left_knee", "right_knee", "spine2",
                    "left_ankle", "right_ankle", "spine3", "left_foot", "right_foot", "neck", "left_collar",
                    "right_collar", "head", "left_shoulder", "right_shoulder", "left_elbow", "right_elbow",
                    "left_wrist", "right_wrist", "jaw", "left_eye_smplhf", "right_eye_smplhf",
                    "left_index1", "left_index2", "left_index3", "left_middle1", "left_middle2", "left_middle3",
                    "left_pinky1", "left_pinky2", "left_pinky3", "left_ring1", "left_ring2", "left_ring3",
                    "left_thumb1", "left_thumb2", "left_thumb3",
                    "right_index1", "right_index2", "right_index3", "right_middle1", "right_middle2",
                    "right_middle3", "right_pinky1", "right_pinky2", "right_pinky3", "right_ring1", "right_ring2",
                    "right_ring3", "right_thumb1", "right_thumb2", "right_thumb3"]
assert len(KINEMATIC_JOINTS) == 55
# the 72 non-kinematic names of JOINT_NAMES[:127] (vertex-picked joints and face landmarks): valid in the
# reference (utils/humans.py:25-26), not supported as a person centre here
DEFAULT_PERSONS_PER_IMAGE = 16
# the integer tables among body_model_arrays' entries; the others are fp32
BODY_TABLES = ("parents", "extra_joints_idxs", "lmk_tri")


def body_model_arrays(bm: dict, num_betas: int, landmarks: bool = True) -> dict:
    """The arrays a body-model loader takes (the engine's `smplx.*` weights and tables, `mhmr_body_create`) from a
    body-model dict (`synth.make_body_model`, `api.body_model_from_smplx_npz`, ...): shapedirs with `num_betas`
    columns, the 11th (kid) component taken from `shapedirs_extra`; with `landmarks` (SMPL-X) also the expression
    directions and the landmark triangles faces[lmk_faces_idx] with their barycentric coordinates."""
    sd = torch.as_tensor(bm["shapedirs"])
    if sd.shape[-1] < num_betas:
        sd = torch.cat([sd, torch.as_tensor(bm["shapedirs_extra"])[..., : num_betas - sd.shape[-1]]], dim=-1)
    out = {k: bm[k] for k in ("v_template", "posedirs", "J_regressor", "lbs_weights", "parents", "extra_joints_idxs")}
    out["shapedirs"] = sd[..., :num_betas]
    if landmarks:
        faces = torch.as_tensor(bm["faces"]).long()
        out.update(expr_dirs=bm["expr_dirs"], lmk_tri=faces[torch.as_tensor(bm["lmk_faces_idx"]).long()],
                   lmk_bary_coords=bm["lmk_bary_coords"])
    return out


class _Config(ctypes.Structure):
    _fields_ = [(n, c_int) for n in ("arch", "img_size", "max_batch", "max_persons", "xat_depth",
                                     "xat_num_heads", "num_betas", "person_center_idx", "num_verts",
                                     "refine_central", "head", "xat_dim", "xat_mlp_dim", "num_joints")]


_OUT_FIELDS = ("scores_map", "count", "det_idx", "det_score", "offset", "loc", "dist_pp", "dist", "rotmat",
               "rotvec", "shape", "expression", "transl", "transl_pelvis", "v3d", "v2d", "j3d", "j2d", "z")


class _Outputs(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in _OUT_FIELDS]


def interpolate_pos_embed(pos_embed: torch.Tensor, grid: int) -> torch.Tensor:
    """[1, 1+M*M, D] -> [1, 1+grid*grid, D]: the bicubic interpolation DINOv2 applies on every forward
    (`DinoVisionTransformer.interpolate_pos_encoding`, scale_factor with the 0.1 offset, antialias off).
    It only depends on the image size, so it is folded once at load time."""
    n = pos_embed.shape[1] - 1
    if n == grid * grid:
        return pos_embed.float()
    m = int(math.sqrt(n))
    assert m * m == n, "pos_embed is not a square grid"
    pos = pos_embed.float()
    d = pos.shape[-1]
    s = float(grid + 0.1) / m
    patch = F.interpolate(pos[:, 1:].reshape(1, m, m, d).permute(0, 3, 1, 2), mode="bicubic", antialias=False,
                          scale_factor=(s, s))
    assert tuple(patch.shape[-2:]) == (grid, grid)
    return torch.cat((pos[:, :1], patch.permute(0, 2, 3, 1).reshape(1, -1, d)), dim=1)


class _EngineModel:
    """What the SMPL-X and Anny models share: one engine behind the C-ABI, the weight upload, the forward call."""

    _IGNORED_PREFIX = ""   # state-dict keys load_state_dict drops
    _POS_EMBED_KEY = ""    # the backbone's pos_embed, interpolated to the working grid at upload
    _SKIPPED_KEYS = ()     # state-dict keys the engine does not read
    _ENTRY = ""            # forward entry of the C-ABI; "_u8" appended for uint8 images
    _OUT_STRUCT = None     # ctypes struct of that entry's output pointers, one field per output tensor
    PROFILE_CATEGORIES = ("misc", "layernorm", "gemm_qkv", "attention", "gemm_proj", "gemm_fc1", "gemm_fc2",
                          "gemm_other", "head", "smplx", "refine")

    def __init__(self, backbone, img_size, max_batch, max_persons, refine_central, device):
        if not torch.cuda.is_available():
            raise RuntimeError(f"multihmr_b200.{type(self).__name__} needs a CUDA device (sm_90a); there is no CPU "
                               "fallback")
        self.device = torch.device(device if device is not None else "cuda:0")
        self.backbone_name, self.img_size, self.patch_size = backbone, int(img_size), PATCH_SIZE
        self.embed_dim = EMBED_DIM[backbone]
        # capacity of the per-person buffers for the WHOLE batch; the reference has no limit, so the default
        # scales with the batch (crowded scenes: 16 persons per image on average)
        self.max_batch = int(max_batch)
        self.max_persons = int(max_persons) if max_persons is not None else DEFAULT_PERSONS_PER_IMAGE * self.max_batch
        self.refine_central = bool(refine_central)
        self.res = self.img_size // PATCH_SIZE
        self._lib = _lib.load()
        self._handle = None
        self._state = {}
        self._finalized = False
        self.training = False

    # ------------------------------------------------------------------ nn.Module-like surface
    def to(self, *a, **k):
        return self

    def cuda(self, *a, **k):
        return self

    def eval(self):
        return self

    def state_dict(self):
        return dict(self._state)

    def load_state_dict(self, state_dict, strict=False):
        """Accepts the reference's state-dict keys; keys under `_IGNORED_PREFIX` are ignored."""
        if self._finalized:
            raise RuntimeError("weights are frozen after the first forward")
        unexpected = []
        for k, v in state_dict.items():
            if k.startswith(self._IGNORED_PREFIX):
                continue
            if not torch.is_tensor(v):
                unexpected.append(k)
                continue
            self._state[k] = v.detach()
        if strict and unexpected:
            raise RuntimeError(f"unexpected keys: {unexpected}")
        return SimpleNamespace(missing_keys=[], unexpected_keys=unexpected)

    # ------------------------------------------------------------------ load-time packing
    def _head_config(self) -> dict:
        """The `_Config` fields of the head (all but arch, sizes, capacities and refine_central)."""
        raise NotImplementedError

    def _upload_extras(self):
        """Uploads what the engine needs beyond the state dict."""

    def _set_weight(self, key, t):
        t = t.detach().to(torch.float32).contiguous()
        check(self._lib.mhmr_set_weight(self._handle, key.encode(), ptr(t), c_int64(t.numel())), f"set_weight({key})")

    def finalize(self):
        if self._finalized:
            return self
        with torch.cuda.device(self.device):
            cfg = _Config(arch=ARCH_ID[self.backbone_name], img_size=self.img_size, max_batch=self.max_batch,
                          max_persons=self.max_persons, refine_central=1 if self.refine_central else 0,
                          **self._head_config())
            h = c_void_p()
            check(self._lib.mhmr_create(ctypes.byref(cfg), ctypes.byref(h)), "mhmr_create")
            self._handle = h
            for k, v in self._state.items():
                if k == self._POS_EMBED_KEY:
                    v = interpolate_pos_embed(v.cpu(), self.res)
                if k in self._SKIPPED_KEYS:
                    continue
                self._set_weight(k, v)
            self._upload_extras()
            check(self._lib.mhmr_finalize(self._handle), "mhmr_finalize")
        self._finalized = True
        return self

    def __del__(self):
        try:
            if self._handle is not None:
                self._lib.mhmr_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    # ------------------------------------------------------------------ forward
    def _prepare_image(self, x):
        """-> (image on the device, fused): uint8 [B,S,S,3] RGB goes to the fused loader (normalize_rgb + patch rows in
        one kernel), anything else is the normalised [B,3,S,S] image as fp32."""
        fused = x.dtype == torch.uint8
        if fused:
            x = x.to(self.device, non_blocking=True).contiguous()
            assert x.dim() == 4 and x.shape[3] == 3 and x.shape[1] == x.shape[2] == self.img_size, "bad image shape"
        else:
            x = x.to(self.device, dtype=torch.float32, non_blocking=True).contiguous()
            assert x.dim() == 4 and x.shape[1] == 3 and x.shape[2] == x.shape[3] == self.img_size, "bad image shape"
        return x, fused

    def _forced_idx(self, rows, B):
        """Index rows (batch, y, x[, 4th]) of the forced persons -> [4, P] int64 host tensor, zeros as the missing 4th
        row.  The reference indexes tensors with idx and raises IndexError when it is out of range (model.py:246-255);
        the kernels trust the indices, so they are validated here."""
        rows = [i.to(torch.int64).cpu() for i in rows]
        h_idx = torch.stack(rows if len(rows) == 4 else rows + [torch.zeros_like(rows[0])])
        P = int(h_idx.shape[1])
        if P > 0:
            if h_idx[0].min() < 0 or h_idx[0].max() >= B or h_idx[1:3].min() < 0 or h_idx[1:3].max() >= self.res:
                raise IndexError(f"idx out of range for batch {B} and a {self.res}x{self.res} token grid")
            if P > self.max_persons:
                raise _lib.MhmrError(f"{P} forced persons > max_persons {self.max_persons}")
        return h_idx

    def _run(self, x, fused, K, det_thresh, nms_kernel_size, fidx, t):
        """Enqueues the forward into the output tensors `t` (None: not wanted) on the current stream and returns the
        number of persons."""
        if isinstance(det_thresh, list):
            det_thresh = det_thresh[0]                                               # model.py:614-615
        o = self._OUT_STRUCT(*[ptr(t[n]).value if t[n] is not None else None for n, _ in self._OUT_STRUCT._fields_])
        fP = 0
        if fidx is not None:
            fP = int(fidx.shape[1])
            fidx = fidx.to(self.device).contiguous()
        stream = c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        args = (ptr(K), c_int(x.shape[0]), ctypes.c_float(float(det_thresh)), c_int(int(nms_kernel_size)), ptr(fidx),
                c_int(fP), ctypes.byref(o), stream)
        if fused:
            from .preprocess import device_table
            entry = self._ENTRY + "_u8"
            check(getattr(self._lib, entry)(self._handle, ptr(x), ptr(device_table(self.device)), *args), entry)
        else:
            check(getattr(self._lib, self._ENTRY)(self._handle, ptr(x), *args), self._ENTRY)
        n = c_int(0)
        check(self._lib.mhmr_sync_count(self._handle, stream, ctypes.byref(n)), "mhmr_sync_count")
        self.last_outputs = t
        return int(n.value)

    def last_launch_count(self) -> int:
        return int(self._lib.mhmr_last_launch_count(self._handle))

    def set_profiling(self, enable: bool):
        self.finalize()
        check(self._lib.mhmr_set_profiling(self._handle, c_int(1 if enable else 0)), "mhmr_set_profiling")

    def get_profile(self) -> dict:
        """{category: (device ms summed over launches, launches)} since profiling was enabled / last read."""
        n = len(self.PROFILE_CATEGORIES)
        ms, cnt = (ctypes.c_float * n)(), (ctypes.c_int * n)()
        check(self._lib.mhmr_get_profile(self._handle, ms, cnt), "mhmr_get_profile")
        return {c: (float(ms[i]), int(cnt[i])) for i, c in enumerate(self.PROFILE_CATEGORIES)}


class Model(_EngineModel):
    """H100-native drop-in for reference `model.Model` (inference path)."""

    # the reference's checkpoints exclude the body model's buffers (train.py:195-201)
    _IGNORED_PREFIX = "smpl_layer."
    _POS_EMBED_KEY = "backbone.encoder.pos_embed"
    _SKIPPED_KEYS = ("backbone.encoder.mask_token", "x_attention_head.init_betas_kid", "x_attention_head.init_expression")
    _ENTRY = "mhmr_forward"
    _OUT_STRUCT = _Outputs

    def __init__(self, backbone="dinov2_vitb14", pretrained_backbone=False, img_size=896,
                 camera_embedding="geometric", camera_embedding_num_bands=16,
                 camera_embedding_max_resolution=64, nearness=True, xat_depth=2, xat_num_heads=8,
                 dict_smpl_layer=None, person_center="head", clip_dist=True, num_betas=10, *args,
                 max_batch=8, max_persons=None, body_model=None, device=None, refine_central=True, **kwargs):
        if backbone not in ARCH_ID:
            raise ValueError(f"unknown backbone {backbone!r}")
        assert img_size % PATCH_SIZE == 0, "Invalid img size"                      # model.py:65
        if camera_embedding != "geometric":
            raise NotImplementedError("Only geometric camera embedding is implemented")  # model.py:72-75
        if camera_embedding_num_bands != 16 or camera_embedding_max_resolution != 64:
            raise NotImplementedError("camera embedding is built for 16 bands / max_resolution 64")
        if not nearness:
            raise NotImplementedError("only nearness=True (log-depth) checkpoints are supported")
        assert num_betas in (10, 11)                                                 # model.py:384
        if person_center not in KINEMATIC_JOINTS:
            raise NotImplementedError(f"person_center {person_center!r}: only the 55 kinematic SMPL-X joints are "
                                      "supported as person centre (vertex-picked joints / landmarks are not)")
        super().__init__(backbone, img_size, max_batch, max_persons, refine_central, device)
        self.nearness = nearness
        self.clip_dist = (clip_dist,)
        self.xat_depth, self.xat_num_heads, self.num_betas = xat_depth, xat_num_heads, num_betas
        self.person_center = person_center
        self.fovn = 60
        self.num_verts = NUM_VERTS
        self.smpl_layer = {}
        if body_model is not None:
            self.set_body_model(body_model)

    def set_body_model(self, bm: dict):
        """Body-model buffers as `smplx.create(..., 'smplx', gender='neutral', use_pca=False,
        flat_hand_mean=True)` registers them (blocks/smpl_layer.py:38): see synth.make_body_model."""
        self._bm = bm
        self.num_verts = int(bm["v_template"].shape[0])
        faces = bm["faces"].cpu().numpy()
        layer = SimpleNamespace(bm_x=SimpleNamespace(faces=faces))
        self.smpl_layer = {"neutral_10": layer, "neutral_11": layer}  # demo.py:310 reads .bm_x.faces

    # ------------------------------------------------------------------ load-time packing
    def _set_table(self, key, t):
        t = t.detach().to(torch.int32).contiguous().cpu()
        check(self._lib.mhmr_set_table_i32(self._handle, key.encode(), ptr(t), c_int64(t.numel())), f"set_table({key})")

    def finalize(self):
        if not self._finalized and not hasattr(self, "_bm"):
            raise RuntimeError("no body model: call set_body_model() (SMPL-X buffers) before the first forward")
        return super().finalize()

    def _head_config(self):
        return dict(xat_depth=self.xat_depth, xat_num_heads=self.xat_num_heads, num_betas=self.num_betas,
                    person_center_idx=KINEMATIC_JOINTS.index(self.person_center), num_verts=self.num_verts)

    def _upload_extras(self):
        self._set_weight("camera.freq_bands", torch.linspace(1.0, 32.0, 16))       # blocks/camera_embed.py:46
        for k, v in body_model_arrays(self._bm, self.num_betas).items():
            (self._set_table if k in BODY_TABLES else self._set_weight)("smplx." + k, v)

    # ------------------------------------------------------------------ forward
    def _alloc_outputs(self, B, want_v2d, want_z):
        Pm, V, nb, dev = self.max_persons, self.num_verts, self.num_betas, self.device
        f = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)
        t = {
            "scores_map": f(B, self.res, self.res), "count": torch.zeros(1, device=dev, dtype=torch.int32),
            "det_idx": torch.zeros(3, Pm, device=dev, dtype=torch.int32), "det_score": f(Pm), "offset": f(Pm, 2),
            "loc": f(Pm, 2), "dist_pp": f(Pm), "dist": f(Pm), "rotmat": f(Pm, 53, 3, 3), "rotvec": f(Pm, 53, 3),
            "shape": f(Pm, nb), "expression": f(Pm, 10), "transl": f(Pm, 3), "transl_pelvis": f(Pm, 3),
            "v3d": f(Pm, V, 3), "v2d": f(Pm, V, 2) if want_v2d else None, "j3d": f(Pm, 127, 3), "j2d": f(Pm, 127, 2),
            "z": f(B, self.res * self.res, self.embed_dim) if want_z else None,
        }
        return t

    def forward_raw(self, x, K, idx=None, det_thresh=0.3, nms_kernel_size=3, want_v2d=False, want_z=False):
        """Enqueues one forward and returns (outputs dict of max_persons-sized device tensors, P)."""
        self.finalize()
        with torch.cuda.device(self.device):
            return self._forward_raw(x, K, idx, det_thresh, nms_kernel_size, want_v2d, want_z)

    def _forward_raw(self, x, K, idx, det_thresh, nms_kernel_size, want_v2d, want_z):
        x, fused = self._prepare_image(x)
        K = K.to(self.device, dtype=torch.float32, non_blocking=True).contiguous()
        B = x.shape[0]
        assert K.shape == (B, 3, 3), "K must be [B,3,3]"
        t = self._alloc_outputs(B, want_v2d, want_z)
        fidx, unsort = None, None
        if idx is not None:
            fidx = self._forced_idx(idx[:4] if len(idx) >= 4 else idx[:3], B)
            if (fidx[0][1:] < fidx[0][:-1]).any():
                # persons of one image must be contiguous for the engine: run in image order, restore after
                order = torch.argsort(fidx[0], stable=True)
                fidx = fidx[:, order]
                unsort = torch.argsort(order).to(self.device)
        P = self._run(x, fused, K, det_thresh, nms_kernel_size, fidx, t)
        if unsort is not None and P > 0:
            per_person = ("det_score", "offset", "loc", "dist_pp", "dist", "rotmat", "rotvec", "shape", "expression",
                          "transl", "transl_pelvis", "v3d", "v2d", "j3d", "j2d")
            for k in per_person:
                if t[k] is not None:
                    t[k][:P] = t[k][:P].index_select(0, unsort)
            t["det_idx"][:, :P] = t["det_idx"][:, :P].index_select(1, unsort)
        return t, P

    def forward(self, x, idx=None, det_thresh=0.3, nms_kernel_size=3, K=None, is_training=False, *args, **kwargs):
        """reference model.py:205-349."""
        assert K is not None, "camera intrinsics K are required"
        if is_training:
            assert idx is not None                                                   # model.py:151
        t, P = self.forward_raw(x, K, idx=idx if is_training else None, det_thresh=det_thresh,
                                nms_kernel_size=nms_kernel_size, want_v2d=is_training)
        if P == 0 and not is_training:
            return []                                                                # model.py:241-243
        if is_training:
            return {
                "dist_postprocessed": t["dist_pp"][:P, None], "scores": t["scores_map"][..., None],
                "offset": t["offset"][:P], "dist": t["dist"][:P, None], "expression": t["expression"][:P],
                "rotmat": t["rotmat"][:P], "shape": t["shape"][:P], "rotvec": t["rotvec"][:P], "loc": t["loc"][:P],
                "v3d": t["v3d"][:P], "j3d": t["j3d"][:P], "j2d": t["j2d"][:P], "v2d": t["v2d"][:P],
                "transl": t["transl"][:P], "transl_pelvis": t["transl_pelvis"][:P, None],
            }
        persons = []
        for i in range(P):                                                           # model.py:329-347
            persons.append({
                "scores": t["det_score"][i], "loc": t["loc"][i], "transl": t["transl"][i],
                "transl_pelvis": t["transl_pelvis"][i][None], "rotvec": t["rotvec"][i],
                "expression": t["expression"][i], "shape": t["shape"][i], "v3d": t["v3d"][i], "j3d": t["j3d"][i],
                "j2d": t["j2d"][i],
            })
        return persons

    __call__ = forward

    # ------------------------------------------------------------------ stage-level entries (parity / ncu)
    def backbone(self, x):
        """`Dinov2Backbone.forward` (blocks/dinov2.py:16-26): [B,3,S,S] -> [B,N,D]."""
        self.finalize()
        x = x.to(self.device, dtype=torch.float32).contiguous()
        B = x.shape[0]
        z = torch.empty(B, self.res * self.res, self.embed_dim, device=self.device)
        with torch.cuda.device(self.device):
            stream = c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            check(self._lib.mhmr_vit_forward(self._handle, ptr(x), c_int(B), ptr(z), stream), "mhmr_vit_forward")
        return z

    def smplx(self, rotvec, shape, loc, dist, K, expression, want_v2d=True):
        """`SMPL_Layer.forward` (blocks/smpl_layer.py:47-155) for P persons.  Differentiable in rotvec, shape, loc,
        dist and expression when grad mode is on and one of them requires grad (`mhmr_smplx_backward`); gradients
        with respect to K are not provided."""
        self.finalize()
        P = rotvec.shape[0]
        assert list(rotvec.shape[1:]) == [53, 3] and P <= self.max_persons                       # :67
        if torch.is_grad_enabled():
            if isinstance(K, torch.Tensor) and K.requires_grad:
                raise NotImplementedError("Model.smplx: gradients with respect to K are not provided")
            if any(isinstance(t, torch.Tensor) and t.requires_grad for t in (rotvec, shape, loc, dist, expression)):
                v3d, v2d, j3d, j2d, transl, tp = _SmplxFunction.apply(self, K, rotvec, shape, loc, dist, expression)
                return {"v3d": v3d, "v2d": v2d if want_v2d else None, "j3d": j3d, "j2d": j2d, "transl": transl,
                        "transl_pelvis": tp[:, None]}
        return self._smplx_forward(*self._smplx_inputs(rotvec, shape, loc, dist, K, expression), want_v2d)

    def _smplx_inputs(self, rotvec, shape, loc, dist, K, expression):
        c = lambda a: a.detach().to(self.device, dtype=torch.float32).contiguous()
        return tuple(map(c, (rotvec, shape, loc, dist, K, expression)))

    def _smplx_backward(self, x, g_v3d=None, g_v2d=None, g_j3d=None, g_j2d=None, g_transl=None,
                        g_transl_pelvis=None):
        """`mhmr_smplx_backward` on converted inputs x = (rotvec, shape, loc, dist, K, expression) and fp32 upstream
        gradients (each None = zero).  Returns d_rotvec [P,53,3], d_shape, d_loc [P,2], d_dist [P], d_expression."""
        self.finalize()
        rotvec, shape, loc, dist, K, expression = x
        P, dev = rotvec.shape[0], self.device
        g = lambda t: None if t is None else t.to(dev, torch.float32).contiguous()
        d = [torch.empty_like(t) for t in (rotvec, shape, loc, dist, expression)]
        with torch.cuda.device(dev):
            stream = c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            check(self._lib.mhmr_smplx_backward(self._handle, c_int(P), ptr(rotvec), ptr(shape), ptr(expression),
                                                ptr(loc), ptr(dist), ptr(K), ptr(g(g_v3d)), ptr(g(g_v2d)),
                                                ptr(g(g_j3d)), ptr(g(g_j2d)), ptr(g(g_transl)),
                                                ptr(g(g_transl_pelvis)), ptr(d[0]), ptr(d[1]), ptr(d[4]), ptr(d[2]),
                                                ptr(d[3]), stream), "mhmr_smplx_backward")
        return tuple(d)

    def _smplx_forward(self, rotvec, shape, loc, dist, K, expression, want_v2d=True):
        self.finalize()
        P, dev, V = rotvec.shape[0], self.device, self.num_verts
        f = lambda *s: torch.empty(*s, device=dev)
        out = {"v3d": f(P, V, 3), "v2d": f(P, V, 2) if want_v2d else None, "j3d": f(P, 127, 3), "j2d": f(P, 127, 2),
               "transl": f(P, 3), "transl_pelvis": f(P, 3)}
        with torch.cuda.device(dev):
            stream = c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            check(self._lib.mhmr_smplx_forward(self._handle, c_int(P), ptr(rotvec), ptr(shape), ptr(expression),
                                               ptr(loc), ptr(dist), ptr(K), ptr(out["v3d"]), ptr(out["v2d"]),
                                               ptr(out["j3d"]), ptr(out["j2d"]), ptr(out["transl"]),
                                               ptr(out["transl_pelvis"]), stream), "mhmr_smplx_forward")
        out["transl_pelvis"] = out["transl_pelvis"][:, None]
        return out


class _SmplxFunction(torch.autograd.Function):
    """Model.smplx with gradients: forward = `mhmr_smplx_forward`, backward = `mhmr_smplx_backward`."""

    @staticmethod
    def forward(ctx, model, K, rotvec, shape, loc, dist, expression):
        ctx.set_materialize_grads(False)
        x = model._smplx_inputs(rotvec, shape, loc, dist, K, expression)
        out = model._smplx_forward(*x, want_v2d=True)
        ctx.model, ctx.x, ctx.orig = model, x, (rotvec, shape, loc, dist, expression)
        return out["v3d"], out["v2d"], out["j3d"], out["j2d"], out["transl"], out["transl_pelvis"][:, 0]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_v3d, g_v2d, g_j3d, g_j2d, g_transl, g_tp):
        d_rot, d_shape, d_loc, d_dist, d_expr = ctx.model._smplx_backward(
            ctx.x, g_v3d=g_v3d, g_v2d=g_v2d, g_j3d=g_j3d, g_j2d=g_j2d, g_transl=g_transl, g_transl_pelvis=g_tp)
        need = ctx.needs_input_grad[2:]
        like = lambda d, t, n: d.reshape(t.shape).to(device=t.device, dtype=t.dtype) if n else None
        return (None, None, *(like(d, t, n) for d, t, n in zip((d_rot, d_shape, d_loc, d_dist, d_expr), ctx.orig, need)))
