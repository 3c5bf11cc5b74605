"""Seeded synthetic assets with the exact names/shapes the reference loads (there is no network for the
published checkpoints, `SMPLX_NEUTRAL.npz` or `smpl_mean_params.npz`):

  make_state_dict  : `model_state_dict` keys of a Multi-HMR checkpoint (SURVEY.md Appendix B;
                     reference demo.py:87-103, train.py:195-207)
  make_mean_params : contents of models/smpl_mean_params.npz used at model.py:440-477
  make_body_model  : SMPL-X-shaped body model (V=10475, 55 joints, 486 pose-corrective features,
                     51 static landmarks, 21 vertex-picked joints) as consumed by smplx.create at
                     blocks/smpl_layer.py:38
  make_smpl_body_model, make_smplx2smpl, make_j_regressor_h36m : the evaluation assets of train.py:41-45, :400
                     (SMPL-shaped body model, SMPL-X -> SMPL transfer matrix, H36M joint regressor)

Everything is generated on the CPU from torch.Generator seeds so the GPU box, the build container and
the golden-fixture script see bit-identical inputs.
"""
from __future__ import annotations

import math

import numpy as np

import torch

BACKBONES = {
    "dinov2_vits14": dict(embed_dim=384, depth=12, num_heads=6),
    "dinov2_vitb14": dict(embed_dim=768, depth=12, num_heads=12),
    "dinov2_vitl14": dict(embed_dim=1024, depth=24, num_heads=16),
}
PATCH = 14
NUM_VERTS = 10475
NUM_FACES = 20908
NUM_JOINTS = 55
SMPLX_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15,
                 20, 25, 26, 20, 28, 29, 20, 31, 32, 20, 34, 35, 20, 37, 38,
                 21, 40, 41, 21, 43, 44, 21, 46, 47, 21, 49, 50, 21, 52, 53]
HPH_DIM = 1024
CAMERA_EMBED_DIM = 99


def _gen(seed: int) -> torch.Generator:
    return torch.Generator(device="cpu").manual_seed(seed)


def _randn(g, *shape, std=1.0):
    return torch.randn(*shape, generator=g) * std


def _makers(sd, g):
    def lin(name, out_f, in_f, std=0.02, bias=True, bias_std=0.02):
        sd[name + ".weight"] = _randn(g, out_f, in_f, std=std)
        if bias:
            sd[name + ".bias"] = _randn(g, out_f, std=bias_std)

    def ln(name, dim):
        sd[name + ".weight"] = 1.0 + _randn(g, dim, std=0.1)
        sd[name + ".bias"] = _randn(g, dim, std=0.05)

    return lin, ln


def _backbone_weights(sd, g, backbone, e):
    """DINOv2 hub-model weights under the prefix `e` (the random stream is consumed in a fixed order)."""
    cfg = BACKBONES[backbone]
    D, depth = cfg["embed_dim"], cfg["depth"]
    lin, ln = _makers(sd, g)
    sd[e + "cls_token"] = _randn(g, 1, 1, D, std=0.02)
    sd[e + "pos_embed"] = _randn(g, 1, 1 + 37 * 37, D, std=0.02)
    sd[e + "mask_token"] = torch.zeros(1, D)
    sd[e + "patch_embed.proj.weight"] = _randn(g, D, 3, PATCH, PATCH, std=0.02)
    sd[e + "patch_embed.proj.bias"] = _randn(g, D, std=0.02)
    for i in range(depth):
        b = f"{e}blocks.{i}."
        ln(b + "norm1", D)
        lin(b + "attn.qkv", 3 * D, D)
        lin(b + "attn.proj", D, D)
        sd[b + "ls1.gamma"] = 0.05 + 0.95 * torch.rand(D, generator=g)
        ln(b + "norm2", D)
        lin(b + "mlp.fc1", 4 * D, D)
        lin(b + "mlp.fc2", D, 4 * D)
        sd[b + "ls2.gamma"] = 0.05 + 0.95 * torch.rand(D, generator=g)
    ln(e + "norm", D)


def make_state_dict(backbone: str = "dinov2_vitl14", img_size: int = 896, num_betas: int = 10,
                    xat_depth: int = 2, xat_num_heads: int = 8, seed: int = 0,
                    det_bias: float = -4.0) -> dict:
    """Random-init weights with trained-like scales.  `det_bias` shifts the detection logit so that only a
    few cells per image pass the 0.3 threshold."""
    cfg = BACKBONES[backbone]
    D = cfg["embed_dim"]
    C = D + CAMERA_EMBED_DIM
    res = img_size // PATCH
    g = _gen(seed)
    sd = {}
    lin, ln = _makers(sd, g)
    _backbone_weights(sd, g, backbone, "backbone.encoder.")

    lin("mlp_classif.0", D, D)
    lin("mlp_classif.2", 1, D, std=0.07)
    sd["mlp_classif.2.bias"] = torch.full((1,), float(det_bias))
    lin("mlp_offset.0", D, D)
    lin("mlp_offset.2", 2, D, std=0.02)

    h = "x_attention_head."
    for nm in ("cross_queries_x", "cross_queries_y", "cross_values_x", "cross_values_y"):
        sd[h + nm] = _randn(g, res, C, std=0.2)
    mean = make_mean_params(seed)
    init_pose = torch.eye(3).reshape(1, 3, 3).repeat(53, 1, 1)[:, :, :2].flatten(1).reshape(1, -1)
    init_pose[:, : 24 * 6] = mean["pose"].float()
    sd[h + "init_body_pose"] = init_pose
    init_betas = mean["shape"].float().unsqueeze(0)
    sd[h + "init_betas_kid"] = torch.cat([init_betas, torch.zeros(1, 1)], 1)
    if num_betas == 11:
        init_betas = torch.cat([init_betas, torch.zeros(1, 1)], 1)
    sd[h + "init_betas"] = init_betas
    sd[h + "init_cam"] = mean["cam"].float().unsqueeze(0)
    sd[h + "init_expression"] = torch.zeros(1, 10)

    t = h + "transformer."
    token_dim = 318 + num_betas + 3 + C
    sd[t + "pos_embedding"] = _randn(g, 1, 1, HPH_DIM)
    lin(t + "to_token_embedding", HPH_DIM, token_dim)
    inner = xat_num_heads * 32
    for l in range(xat_depth):
        p = f"{t}transformer.layers.{l}."
        ln(p + "0.norm", HPH_DIM)
        lin(p + "0.fn.to_qkv", 3 * inner, HPH_DIM, bias=False)
        lin(p + "0.fn.to_out.0", HPH_DIM, inner)
        ln(p + "1.norm", HPH_DIM)
        lin(p + "1.fn.to_kv", 2 * inner, C, bias=False, std=0.03)
        lin(p + "1.fn.to_q", inner, HPH_DIM, bias=False, std=0.03)
        lin(p + "1.fn.to_out.0", HPH_DIM, inner)
        ln(p + "2.norm", HPH_DIM)
        lin(p + "2.fn.net.0", HPH_DIM, HPH_DIM)
        lin(p + "2.fn.net.3", HPH_DIM, HPH_DIM)
    # Trained-like conditioning of the 6D pose head: joints 24..52 start from the degenerate init
    # [1,0,0,1,0,0] (model.py:444-450: two identical columns after utils/humans.py:20), so a trained decoder
    # must add ~[0,0,0,-1,1,0] to produce a valid rotation.  Random weights without that offset make the
    # Gram-Schmidt step arbitrarily ill-conditioned (SURVEY.md §7 "hard parts"), which would measure the
    # conditioning of the fixture rather than the kernels.
    lin(h + "decpose", 318, HPH_DIM, std=0.005)
    pose_bias = sd[h + "decpose.bias"].view(53, 6)
    pose_bias[24:] += torch.tensor([0.0, 0.0, 0.0, -1.0, 1.0, 0.0])
    lin(h + "decshape", num_betas, HPH_DIM, std=0.01)
    lin(h + "deccam", 3, HPH_DIM, std=0.005)
    lin(h + "decexpression", 10, HPH_DIM, std=0.01)
    return sd


def add_outlier_channels(sd: dict, backbone: str, seed: int = 0, magnitude: float = 60.0) -> dict:
    """DINOv2-like 'massive activations' on top of make_state_dict (in place; the random stream of make_state_dict
    is untouched, so the other fixtures do not change): a few residual channels carry values of O(100) — on a few
    tokens from the position embedding on, and on every token after two MLP blocks whose fc2 rows / LayerScale for
    those channels are large.  Trained ViTs have such channels; N(0, 0.02) weights alone do not, and fp16
    tensor-core operands (Xn16 / QKV16 / H16) are stressed differently by them."""
    cfg = BACKBONES[backbone]
    D, depth = cfg["embed_dim"], cfg["depth"]
    g = _gen(seed + 909)
    ch = torch.randperm(D, generator=g)[:4]
    e = "backbone.encoder."
    pos = sd[e + "pos_embed"].clone()
    cells = 1 + torch.randperm(37 * 37, generator=g)[:40]          # ~3 % of the pretraining grid
    for c in ch[:2]:
        pos[0, cells, c] += magnitude * (0.5 + torch.rand(cells.numel(), generator=g))
    sd[e + "pos_embed"] = pos
    for l in (depth // 3, depth // 2):
        b = f"{e}blocks.{l}."
        w = sd[b + "mlp.fc2.weight"].clone()
        w[ch[2:]] *= 25.0
        sd[b + "mlp.fc2.weight"] = w
        gma = sd[b + "ls2.gamma"].clone()
        gma[ch[2:]] = 1.0
        sd[b + "ls2.gamma"] = gma
    return sd


def make_mean_params(seed: int = 0) -> dict:
    """pose[144] (24 joints x 6D, in the (a1, a2) order rot6d_to_rotmat reads, utils/humans.py:20),
    shape[10], cam[3]."""
    g = _gen(seed + 101)
    rv = _randn(g, 24, 3, std=0.3)
    ang = rv.norm(dim=1, keepdim=True).clamp_min(1e-8)
    ax = rv / ang
    Kx = torch.zeros(24, 3, 3)
    Kx[:, 0, 1], Kx[:, 0, 2] = -ax[:, 2], ax[:, 1]
    Kx[:, 1, 0], Kx[:, 1, 2] = ax[:, 2], -ax[:, 0]
    Kx[:, 2, 0], Kx[:, 2, 1] = -ax[:, 1], ax[:, 0]
    R = torch.eye(3)[None] + torch.sin(ang)[:, :, None] * Kx + (1 - torch.cos(ang))[:, :, None] * (Kx @ Kx)
    pose6 = torch.cat([R[:, :, 0], R[:, :, 1]], dim=1).reshape(-1)  # [a1(3), a2(3)] per joint
    return {"pose": pose6, "shape": _randn(g, 10, std=0.5), "cam": torch.tensor([0.9, 0.0, 0.0])}


def make_body_model(seed: int = 0, num_verts: int = NUM_VERTS, num_faces: int = NUM_FACES) -> dict:
    g = _gen(seed + 202)
    V = num_verts
    bm = {}
    bm["v_template"] = _randn(g, V, 3) * torch.tensor([0.25, 0.45, 0.12])
    bm["shapedirs"] = _randn(g, V, 3, 10, std=0.01)
    bm["shapedirs_extra"] = _randn(g, V, 3, 1, std=0.01)  # 11th (kid) component of the neutral_11 layer
    bm["expr_dirs"] = _randn(g, V, 3, 10, std=0.005)
    bm["posedirs"] = _randn(g, (NUM_JOINTS - 1) * 9, V * 3, std=1e-3)
    Jr = torch.zeros(NUM_JOINTS, V)
    for j in range(NUM_JOINTS):
        ids = torch.randint(0, V, (32,), generator=g)
        w = torch.rand(32, generator=g)
        Jr[j].index_add_(0, ids, w / w.sum())
    bm["J_regressor"] = Jr
    W = torch.zeros(V, NUM_JOINTS)
    ids = torch.randint(0, NUM_JOINTS, (V, 4), generator=g)
    w = torch.rand(V, 4, generator=g) + 0.05
    W.scatter_add_(1, ids, w / w.sum(dim=1, keepdim=True))
    bm["lbs_weights"] = W
    bm["parents"] = torch.tensor(SMPLX_PARENTS, dtype=torch.int64)
    bm["faces"] = torch.randint(0, V, (num_faces, 3), generator=g)
    bm["lmk_faces_idx"] = torch.randint(0, num_faces, (51,), generator=g)
    bary = torch.rand(51, 3, generator=g) + 0.1
    bm["lmk_bary_coords"] = bary / bary.sum(dim=1, keepdim=True)
    bm["extra_joints_idxs"] = torch.randint(0, V, (21,), generator=g)
    return bm


SMPL_NUM_VERTS = 6890
SMPL_NUM_FACES = 13776
SMPL_NUM_JOINTS = 24
SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]


def make_smpl_body_model(seed: int = 0, gender: str = "male") -> dict:
    """SMPL-shaped body model (V = 6890, the standard 24-joint parent table, 207 pose-corrective features, 10 betas,
    21 vertex-picked joints at the smplx.vertex_ids['smplh'] ids) in the dict layout of `api.body_model_from_smpl_pkl`.
    Male and female differ through the seed."""
    from .api import SMPL_EXTRA_JOINTS_IDXS

    g = _gen(seed + 606 + (0 if gender == "male" else 17))
    V, NJ = SMPL_NUM_VERTS, SMPL_NUM_JOINTS
    bm = {"v_template": _randn(g, V, 3) * torch.tensor([0.25, 0.45, 0.12]),
          "shapedirs": _randn(g, V, 3, 10, std=0.01),
          "posedirs": _randn(g, (NJ - 1) * 9, V * 3, std=1e-3)}
    Jr = torch.zeros(NJ, V)
    for j in range(NJ):
        ids = torch.randint(0, V, (32,), generator=g)
        w = torch.rand(32, generator=g)
        Jr[j].index_add_(0, ids, w / w.sum())
    bm["J_regressor"] = Jr
    W = torch.zeros(V, NJ)
    ids = torch.randint(0, NJ, (V, 4), generator=g)
    w = torch.rand(V, 4, generator=g) + 0.05
    W.scatter_add_(1, ids, w / w.sum(dim=1, keepdim=True))
    bm["lbs_weights"] = W
    bm["parents"] = torch.tensor(SMPL_PARENTS, dtype=torch.int64)
    bm["faces"] = torch.randint(0, V, (SMPL_NUM_FACES, 3), generator=g)
    bm["extra_joints_idxs"] = torch.tensor(SMPL_EXTRA_JOINTS_IDXS, dtype=torch.int64)
    bm["num_verts"] = V
    return bm


def make_smplx2smpl(seed: int = 0) -> torch.Tensor:
    """SMPL-X -> SMPL transfer matrix [6890, 10475] with barycentric rows (3 distinct SMPL-X vertices, positive weights
    summing to 1), as a torch sparse COO tensor (the dense fp32 matrix is 290 MB)."""
    g = _gen(seed + 707)
    R = SMPL_NUM_VERTS
    pick = torch.randint(0, NUM_VERTS, (R, 3), generator=g)
    pick[:, 1] = (pick[:, 0] + 1 + torch.randint(0, 50, (R,), generator=g)) % NUM_VERTS
    pick[:, 2] = (pick[:, 1] + 1 + torch.randint(0, 50, (R,), generator=g)) % NUM_VERTS
    w = torch.rand(R, 3, generator=g) + 0.05
    w = w / w.sum(dim=1, keepdim=True)
    rows = torch.arange(R).repeat_interleave(3)
    return torch.sparse_coo_tensor(torch.stack([rows, pick.reshape(-1)]), w.reshape(-1),
                                   (R, NUM_VERTS), check_invariants=True).coalesce()


def make_j_regressor_h36m(seed: int = 0) -> torch.Tensor:
    """H36M joint regressor [17, 6890]: non-negative rows summing to 1 over 48 random SMPL vertices each."""
    g = _gen(seed + 808)
    Jr = torch.zeros(17, SMPL_NUM_VERTS)
    for j in range(17):
        ids = torch.randint(0, SMPL_NUM_VERTS, (48,), generator=g)
        w = torch.rand(48, generator=g)
        Jr[j].index_add_(0, ids, w / w.sum())
    return Jr


def make_images(batch: int, img_size: int, seed: int = 0) -> torch.Tensor:
    """fp32 NCHW in the range normalize_rgb produces (utils/image.py:8-24)."""
    g = _gen(seed + 303)
    return torch.randn(batch, 3, img_size, img_size, generator=g).clamp_(-2.1, 2.6)


def make_images_u8(batch: int, img_size: int, seed: int = 0) -> torch.Tensor:
    """uint8 [B,S,S,3] RGB (HWC), what PIL + ImageOps.pad yield in demo.py:33-47 before normalize_rgb."""
    g = _gen(seed + 313)
    return torch.randint(0, 256, (batch, img_size, img_size, 3), generator=g, dtype=torch.uint8)


def make_cameras(batch: int, img_size: int, fov_deg=60.0, jitter: bool = False, seed: int = 0,
                 asymmetric: bool = False) -> torch.Tensor:
    """K [B,3,3] as demo.py:get_camera_parameters (demo.py:53-68); optional per-image fov jitter;
    `asymmetric` adds fx != fy and an off-centre principal point with cx != cy (exercises the (row, col)
    ordering of model.py:164-178, SURVEY.md Appendix D)."""
    g = _gen(seed + 404)
    K = torch.eye(3).repeat(batch, 1, 1)
    for b in range(batch):
        fov = fov_deg + (float(torch.rand(1, generator=g)) * 20 - 10 if jitter else 0.0)
        f = img_size / (2 * math.tan(math.radians(fov) / 2))
        K[b, 0, 0] = K[b, 1, 1] = f
        K[b, 0, 2] = K[b, 1, 2] = img_size // 2
        if asymmetric:
            K[b, 1, 1] = f * (0.9 + 0.05 * b)
            K[b, 0, 2] = img_size * (0.40 + 0.03 * b)
            K[b, 1, 2] = img_size * (0.57 - 0.02 * b)
    return K


def make_forced_idx(batch: int, res: int, persons_per_image, seed: int = 0):
    """Distinct (b, y, x) cells in torch.where order, as the `idx=` argument of Model.forward
    (model.py:150-151, train.py:171-176): tuple (b, y, x, c=0) of int64 tensors."""
    g = _gen(seed + 505)
    if isinstance(persons_per_image, int):
        persons_per_image = [persons_per_image] * batch
    bs, ys, xs = [], [], []
    for b, n in enumerate(persons_per_image):
        cells = torch.randperm(res * res, generator=g)[:n].sort().values
        bs += [b] * n
        ys += (cells // res).tolist()
        xs += (cells % res).tolist()
    t = lambda v: torch.tensor(v, dtype=torch.int64)
    return (t(bs), t(ys), t(xs), torch.zeros(len(bs), dtype=torch.int64))


# ------------------------------------------------------------------------------------------------------------------
# Anny variant (reference multi_hmr_anny/): state dict of `Multi_HMR` and an Anny-like body model
# ------------------------------------------------------------------------------------------------------------------
ANNY_NUM_JOINTS = 163
ANNY_NUM_BETAS = 11
ANNY_PHENOTYPES = ["gender", "age", "muscle", "weight", "height", "proportions", "cupsize", "firmness",
                   "african", "asian", "caucasian"]
ANNY_HEAD_BONE = 9


def sincos_pos_embed_2d(dim: int, grid: int) -> torch.Tensor:
    """[grid*grid, dim] fixed 2-D sine-cosine table (MAE / CroCo convention): the first half of the channels encodes
    the row index, the second half the column index; each half is [sin(pos w) | cos(pos w)] with
    w_i = 10000^(-i / (dim/4)).  Row n = y * grid + x.  Computed in float64, stored as float32."""
    q = dim // 4
    omega = 1.0 / 10000 ** (torch.arange(q, dtype=torch.float64) / q)
    ys, xs = torch.meshgrid(torch.arange(grid, dtype=torch.float64), torch.arange(grid, dtype=torch.float64),
                            indexing="ij")

    def enc(pos):
        a = pos.reshape(-1, 1) * omega[None]
        return torch.cat([torch.sin(a), torch.cos(a)], 1)

    return torch.cat([enc(ys), enc(xs)], 1).float()


def make_anny_state_dict(backbone: str = "dinov2_vitl14", img_size: int = 672, xat_dim: int = 512,
                         xat_depth: int = 8, xat_heads: int = 16, xat_mlp_dim: int = 2048, seed: int = 0,
                         det_bias: float = -4.0, fov_deg: float = 60.0, dist_m: float = 3.5) -> dict:
    """`Multi_HMR.state_dict()` keys of an Anny checkpoint (encoder.backbone.*, encoder.mlp_det / mlp_fov_unique,
    dec_to_token, decoder.transformer.layers.*, mlp_offset / pose / shape / dist, useful_rotmat, init_body_pose,
    dec_pos_emb, encoder.fov_max, eye).  The output biases put the regressed field of view near `fov_deg` and the
    distances near `dist_m`; `det_bias` shifts the detection logit as in make_state_dict."""
    cfg = BACKBONES[backbone]
    D = cfg["embed_dim"]
    res = img_size // PATCH
    J = ANNY_NUM_JOINTS
    g = _gen(seed + 1000)
    sd = {}
    lin, ln = _makers(sd, g)
    _backbone_weights(sd, g, backbone, "encoder.backbone.")
    lin("encoder.mlp_det.0", D, D)
    lin("encoder.mlp_det.2", 1, D, std=0.07)
    sd["encoder.mlp_det.2.bias"] = torch.full((1,), float(det_bias))
    lin("encoder.mlp_fov_unique.0", D, D)
    lin("encoder.mlp_fov_unique.2", 1, D, std=0.02)
    s = fov_deg / 180.0
    sd["encoder.mlp_fov_unique.2.bias"] = torch.full((1,), math.log(s / (1.0 - s)))
    sd["encoder.fov_max"] = torch.tensor([math.pi])
    sd["dec_pos_emb"] = sincos_pos_embed_2d(xat_dim, res)
    lin("dec_to_token", xat_dim, D)
    inner = xat_heads * 32
    for l in range(xat_depth):
        p = f"decoder.transformer.layers.{l}."
        ln(p + "0.norm", xat_dim)
        lin(p + "0.fn.to_qkv", 3 * inner, xat_dim, bias=False, std=0.03)
        lin(p + "0.fn.to_out.0", xat_dim, inner)
        ln(p + "1.norm", xat_dim)
        lin(p + "1.fn.to_kv", 2 * inner, xat_dim, bias=False, std=0.03)
        lin(p + "1.fn.to_q", inner, xat_dim, bias=False, std=0.03)
        lin(p + "1.fn.to_out.0", xat_dim, inner)
        ln(p + "2.norm", xat_dim)
        lin(p + "2.fn.net.0", xat_mlp_dim, xat_dim)
        lin(p + "2.fn.net.3", xat_dim, xat_mlp_dim)
    lin("mlp_offset.0", xat_dim, xat_dim)
    lin("mlp_offset.2", 2, xat_dim, std=0.02)
    lin("mlp_pose.0", xat_dim, xat_dim + 6 * J)
    lin("mlp_pose.2", 6 * J, xat_dim, std=0.005)
    lin("mlp_shape.0", xat_dim, xat_dim)
    lin("mlp_shape.2", ANNY_NUM_BETAS, xat_dim, std=0.05)
    lin("mlp_dist.0", xat_dim, xat_dim)
    lin("mlp_dist.2", 1, xat_dim, std=0.01)
    focal = (img_size / 2) / math.tan(math.radians(fov_deg) / 2)
    sd["mlp_dist.2.bias"] = torch.full((1,), math.log(focal / dist_m))
    sd["useful_rotmat"] = (torch.rand(1, J, generator=g) < 0.6).float()
    # 6-D initial rotations in the layout rot6d.reshape(3, 2) reads (columns = the two basis vectors): a
    # seeded root rotation, identities elsewhere
    R0 = _rotation(_randn(g, 3, std=0.8))
    init = torch.eye(3).reshape(1, 3, 3).repeat(J, 1, 1)
    init[0] = R0
    sd["init_body_pose"] = init[:, :, :2].flatten(1).reshape(1, -1)
    sd["eye"] = torch.eye(3).unsqueeze(0)
    return sd


def _rotation(rv: torch.Tensor) -> torch.Tensor:
    ang = rv.norm().clamp_min(1e-8)
    ax = rv / ang
    Kx = torch.tensor([[0.0, -ax[2], ax[1]], [ax[2], 0.0, -ax[0]], [-ax[1], ax[0], 0.0]])
    return torch.eye(3) + torch.sin(ang) * Kx + (1 - torch.cos(ang)) * (Kx @ Kx)


def _ellipsoid(n_lat: int, n_lon: int):
    """Unit UV sphere: vertices [2 + (n_lat-1) n_lon, 3] and faces wound so that cross(v1-v0, v2-v0) points out."""
    verts = [[0.0, -1.0, 0.0]]
    for i in range(1, n_lat):
        th = np.pi * i / n_lat
        for j in range(n_lon):
            ph = 2 * np.pi * j / n_lon
            verts.append([np.sin(th) * np.cos(ph), -np.cos(th), np.sin(th) * np.sin(ph)])
    verts.append([0.0, 1.0, 0.0])
    ring = lambda i, j: 1 + (i - 1) * n_lon + (j % n_lon)
    faces = []
    for j in range(n_lon):
        faces.append([0, ring(1, j), ring(1, j + 1)])
        faces.append([len(verts) - 1, ring(n_lat - 1, j + 1), ring(n_lat - 1, j)])
        for i in range(1, n_lat - 1):
            faces.append([ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)])
            faces.append([ring(i, j), ring(i + 1, j + 1), ring(i, j + 1)])
    v, f = np.asarray(verts), np.asarray(faces)
    p = v[f]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    flip = (n * p.mean(1)).sum(-1) < 0
    f[flip] = f[flip][:, [0, 2, 1]]
    return v, f


# (centre, radii) of the parts of a blob person 1.7 m tall, y down (OpenCV camera convention)
_BLOB_PARTS = [((0.0, -0.75, 0.0), (0.11, 0.13, 0.11)), ((0.0, -0.35, 0.0), (0.19, 0.28, 0.12)),
               ((-0.27, -0.35, 0.0), (0.06, 0.3, 0.06)), ((0.27, -0.35, 0.0), (0.06, 0.3, 0.06)),
               ((-0.1, 0.35, 0.0), (0.08, 0.42, 0.08)), ((0.1, 0.35, 0.0), (0.08, 0.42, 0.08))]


def make_blob_people(positions, seed: int = 0, n_lat: int = 8, n_lon: int = 12):
    """Structured test meshes for the renderer: one person = six tessellated ellipsoids (head, torso, arms, legs)
    with one shared topology.  positions: [P,3] pelvis positions in camera coordinates (metres).  Each person gets a
    seeded scale, yaw and part jitter.  Returns (verts fp32 [P,V,3], faces int64 [F,3])."""
    g = np.random.default_rng(seed)
    uv, uf = _ellipsoid(n_lat, n_lon)
    faces = np.concatenate([uf + k * len(uv) for k in range(len(_BLOB_PARTS))])
    out = []
    for pos in np.asarray(positions, np.float64).reshape(-1, 3):
        s = g.uniform(0.85, 1.1)
        yaw = g.uniform(-0.6, 0.6)
        Ry = np.array([[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]])
        parts = []
        for c, r in _BLOB_PARTS:
            rr = np.asarray(r) * g.uniform(0.9, 1.15, 3)
            cc = np.asarray(c) + g.normal(0, 0.01, 3)
            parts.append((uv * rr + cc) * s)
        out.append(np.concatenate(parts) @ Ry.T + pos)
    return np.asarray(out, np.float32), faces.astype(np.int64)


class AnnyLikeBodyModel(torch.nn.Module):
    """A deterministic stand-in for the `anny` package's full-body model with the interface Multi_HMR uses
    (multi_hmr_anny/multi_hmr.py:70-77, :169-182): `bone_labels` (163, with 'head'), `phenotype_labels`, `faces`,
    `set_skinning_method`, and `forward(pose_parameters=[P,163,4,4], phenotype_kwargs={name: [P]})` returning
    `vertices` [P,V,3], `bone_poses` [P,163,4,4] and `blendshape_coeffs` [P,6].  Its arithmetic is a plain
    phenotype blendshape + forward kinematics + linear blend skinning on seeded data; it is NOT the Anny model."""

    SHAPE_KEYS = ("age", "gender", "weight", "height", "muscle", "proportions")

    def __init__(self, num_verts: int = 14000, seed: int = 0):
        super().__init__()
        g = _gen(seed + 2000)
        J, V = ANNY_NUM_JOINTS, num_verts
        parents = [-1] + [int(torch.randint(0, j, (1,), generator=g)) for j in range(1, J)]
        self.register_buffer("parents", torch.tensor(parents, dtype=torch.int64))
        self.register_buffer("joints_rest", _randn(g, J, 3) * torch.tensor([0.2, 0.5, 0.1]))
        self.register_buffer("joint_dirs", _randn(g, len(self.SHAPE_KEYS), J, 3, std=0.02))
        self.register_buffer("v_template", _randn(g, V, 3) * torch.tensor([0.25, 0.6, 0.12]))
        self.register_buffer("shape_dirs", _randn(g, len(self.SHAPE_KEYS), V, 3, std=0.03))
        ids = torch.randint(0, J, (V, 4), generator=g)
        w = torch.rand(V, 4, generator=g) + 0.05
        W = torch.zeros(V, J)
        W.scatter_add_(1, ids, w / w.sum(1, keepdim=True))
        self.register_buffer("weights", W)
        self.faces = torch.randint(0, V, (2 * V, 3), generator=g)
        self.bone_labels = [f"bone_{j:03d}" for j in range(J)]
        self.bone_labels[ANNY_HEAD_BONE] = "head"
        self.phenotype_labels = list(ANNY_PHENOTYPES)
        self.skinning_method = "lbs"

    def set_skinning_method(self, name):
        assert name == "lbs"
        self.skinning_method = name

    def forward(self, pose_parameters, phenotype_kwargs):
        P = pose_parameters.shape[0]
        c = torch.stack([phenotype_kwargs[k] for k in self.SHAPE_KEYS], 1) - 0.5          # [P, 6]
        Jr = self.joints_rest[None] + torch.einsum("pk,kjc->pjc", c, self.joint_dirs)     # [P, J, 3]
        vs = self.v_template[None] + torch.einsum("pk,kvc->pvc", c, self.shape_dirs)      # [P, V, 3]
        G = [None] * ANNY_NUM_JOINTS
        for j in range(ANNY_NUM_JOINTS):
            T = pose_parameters[:, j].clone()
            p = int(self.parents[j])
            T[:, :3, 3] = Jr[:, j] - (Jr[:, p] if p >= 0 else 0.0)
            G[j] = T if p < 0 else G[p] @ T
        G = torch.stack(G, 1)                                                             # [P, J, 4, 4]
        A = G.clone()
        A[:, :, :3, 3] = G[:, :, :3, 3] - torch.einsum("pjab,pjb->pja", G[:, :, :3, :3], Jr)
        Tv = torch.einsum("vj,pjab->pvab", self.weights, A)                               # [P, V, 4, 4]
        verts = torch.einsum("pvab,pvb->pva", Tv[..., :3, :3], vs) + Tv[..., :3, 3]
        return {"vertices": verts, "bone_poses": G, "blendshape_coeffs": c.reshape(P, -1)}
