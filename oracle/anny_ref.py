"""Oracle of the Anny variant (reference multi_hmr_anny/): TEST INFRASTRUCTURE ONLY, plain fp32 torch.

  install_anny_shim : an `anny` module for sys.modules whose `create_fullbody_model` returns the deterministic
                      synthetic body model of multihmr_b200.synth (the `anny` package is not installed here, so
                      its arithmetic is not restated: any deterministic body model pins the head around it)
  anny_forward      : restatement of `Multi_HMR.forward` (multi_hmr_anny/multi_hmr.py:98-246) with the encoder of
                      encoder.py:33-67 and the HPH of hph.py, pinned against the unmodified reference by
                      oracle/make_golden.py and usable where the reference checkout is absent.
"""
import math
import types

import torch
import torch.nn.functional as F

from oracle import dinov2_ref, roma_ref


def install_anny_shim(sys_modules, body_model_factory):
    anny = types.ModuleType("anny")
    anny.create_fullbody_model = lambda **kw: body_model_factory()
    sys_modules["anny"] = anny
    return anny


class AnnyConfig:
    def __init__(self, backbone="dinov2_vits14", img_size=224, xat_depth=8, xat_heads=16, person_center="head"):
        self.backbone, self.img_size, self.xat_depth, self.xat_heads = backbone, img_size, xat_depth, xat_heads
        self.person_center = person_center


def _mlp(x, sd, pre):
    """Linear -> ReLU -> Linear (the nn.Sequential heads of encoder.py:26,29 and multi_hmr.py:59-66)."""
    return F.linear(F.relu(F.linear(x, sd[pre + ".0.weight"], sd[pre + ".0.bias"])), sd[pre + ".2.weight"],
                    sd[pre + ".2.bias"])


def _attention(q, k, v, heads):
    """softmax(q k^T / sqrt(32)) v per head; q [n, h*32], k, v [m, h*32]."""
    n, m = q.shape[0], k.shape[0]
    q, k, v = (t.reshape(t.shape[0], heads, -1).transpose(0, 1) for t in (q, k, v))
    a = torch.softmax(q @ k.transpose(-1, -2) * (q.shape[-1] ** -0.5), dim=-1)
    return (a @ v).transpose(0, 1).reshape(n, -1)


def hph(x, ctx, sd, depth, heads):
    """hph.py TransformerCrossAttn for the n persons of ONE image (x [n, dim]) against that image's N context tokens
    (ctx [N, dim]).  The reference pads the queries of a batch to the largest count: padded keys of self-attention get
    zero weight (mask of :64) and the cross-attention mask (:104-105) shifts every logit of a padded query by the same
    constant, so restricting to the real persons is exact."""
    D = x.shape[1]
    for l in range(depth):
        p = f"decoder.transformer.layers.{l}."
        y = F.layer_norm(x, (D,), sd[p + "0.norm.weight"], sd[p + "0.norm.bias"], 1e-5)
        q, k, v = F.linear(y, sd[p + "0.fn.to_qkv.weight"]).chunk(3, dim=-1)
        x = F.linear(_attention(q, k, v, heads), sd[p + "0.fn.to_out.0.weight"], sd[p + "0.fn.to_out.0.bias"]) + x
        y = F.layer_norm(x, (D,), sd[p + "1.norm.weight"], sd[p + "1.norm.bias"], 1e-5)
        k, v = F.linear(ctx, sd[p + "1.fn.to_kv.weight"]).chunk(2, dim=-1)
        q = F.linear(y, sd[p + "1.fn.to_q.weight"])
        x = F.linear(_attention(q, k, v, heads), sd[p + "1.fn.to_out.0.weight"], sd[p + "1.fn.to_out.0.bias"]) + x
        y = F.layer_norm(x, (D,), sd[p + "2.norm.weight"], sd[p + "2.norm.bias"], 1e-5)
        y = F.linear(F.gelu(F.linear(y, sd[p + "2.fn.net.0.weight"], sd[p + "2.fn.net.0.bias"])),
                     sd[p + "2.fn.net.3.weight"], sd[p + "2.fn.net.3.bias"])
        x = y + x
    return x


def intermediate_layers_with_cls(x_img, sd, name, prefix=""):
    """`get_intermediate_layers(x, return_class_token=True)[0]` of the DINOv2 hub model (encoder.py:45): the
    final-normed patch tokens [B, N, D] and the final-normed cls token [B, D], from the blocks of oracle.dinov2_ref."""
    x = dinov2_ref.prepare_tokens(x_img, sd, prefix)
    for i in range(dinov2_ref.ARCHS[name]["depth"]):
        x = dinov2_ref.vit_block(x, sd, f"{prefix}blocks.{i}.", dinov2_ref.ARCHS[name]["num_heads"])
    x = F.layer_norm(x, (x.shape[-1],), sd[prefix + "norm.weight"], sd[prefix + "norm.bias"], dinov2_ref.LN_EPS)
    return x[:, 1:], x[:, 0]


class HubModelShimWithCls(dinov2_ref.HubModelShim):
    """dinov2_ref.HubModelShim whose get_intermediate_layers also accepts `return_class_token=True`, as the Anny
    encoder calls it (encoder.py:45); the default call returns what the base shim returns."""

    def get_intermediate_layers(self, x, return_class_token=False):
        if not return_class_token:
            return super().get_intermediate_layers(x)
        return (intermediate_layers_with_cls(x, dict(self.state_dict()), self.name_),)


def encoder(x, sd, cfg):
    """encoder.py:33-67: features [B,h,w,D], detection logits [B,h,w], fov [B,1], K_regressed [B,3,3]."""
    z, cls = intermediate_layers_with_cls(x, sd, cfg.backbone, "encoder.backbone.")
    B, N, D = z.shape
    w = int(math.sqrt(N))
    S = x.shape[-1]
    fov = sd["encoder.fov_max"] * torch.sigmoid(_mlp(cls, sd, "encoder.mlp_fov_unique"))
    focal = (S / 2) / torch.tan(fov / 2)
    K = torch.eye(3, device=x.device).reshape(1, 3, 3).repeat(B, 1, 1)
    K[:, 0, 0] = K[:, 1, 1] = focal[:, 0]
    K[:, 0, 2] = K[:, 1, 2] = S / 2.0
    feat = z.reshape(B, w, w, D)
    logits = _mlp(feat, sd, "encoder.mlp_det")[..., 0]
    return feat, logits, fov, K


def nms_pad(k):
    """max_pool2d padding of multi_hmr.py:118; the reference then fails for even k (shape mismatch)."""
    if k % 2 == 0:
        raise ValueError(f"nms_kernel_size={k}: an even kernel changes the score map's shape in the reference")
    return (k - 1) // 2


def anny_forward(sd, body_model, cfg, x, K=None, idx=None, is_training=False, det_thresh=0.3, nms_kernel_size=3):
    """Multi_HMR.forward (multi_hmr.py:98-246) with the same return conventions."""
    feat, logits, fov, K_reg = encoder(x, sd, cfg)
    K = K_reg if K is None else K
    scores = torch.sigmoid(logits)
    if not is_training:
        if nms_kernel_size > 1:
            pooled = F.max_pool2d(scores[:, None], nms_kernel_size, 1, nms_pad(nms_kernel_size))[:, 0]
            scores = scores * (pooled == scores).float()
        idx = torch.where(scores >= det_thresh) if idx is None else idx
        if len(idx[0]) == 0:
            return {}, []
    B, w, _, _ = feat.shape
    dim = sd["dec_to_token.weight"].shape[0]
    dec = F.linear(feat, sd["dec_to_token.weight"], sd["dec_to_token.bias"]) + sd["dec_pos_emb"].reshape(1, w, w, dim)
    ys = []
    for b in torch.unique(idx[0], sorted=True).tolist():
        sel = idx[0] == b
        q = dec[b, idx[1][sel], idx[2][sel]]
        ys.append(hph(q, dec[b].reshape(-1, dim), sd, cfg.xat_depth, cfg.xat_heads))
    y = torch.cat(ys, 0)

    offset = _mlp(y, sd, "mlp_offset")
    loc = (torch.stack([idx[2], idx[1]], dim=1) + 0.5 + offset) * 14
    Kp = K[idx[0]]
    dist_pp = _mlp(y, sd, "mlp_dist")
    dist = Kp[:, 0, 0].unsqueeze(1) / torch.clamp(torch.exp(dist_pp), 1e-5)
    transl = torch.einsum("pij,pj->pi", torch.inverse(Kp), torch.cat([loc, torch.ones_like(loc[:, :1])], 1)) * dist
    init = sd["init_body_pose"]
    J = init.shape[1] // 6
    shape = torch.sigmoid(_mlp(y, sd, "mlp_shape"))
    rot6d = _mlp(torch.cat([y, init.repeat(y.shape[0], 1)], 1), sd, "mlp_pose") + init
    rotmat = roma_ref.special_gramschmidt(rot6d.reshape(-1, 3, 2)).view(-1, J, 3, 3)
    u = sd["useful_rotmat"].reshape(1, -1, 1, 1)
    rotmat = u * rotmat + (1 - u) * torch.eye(3, device=rotmat.device).reshape(1, 1, 3, 3)
    rotvec = roma_ref.rotmat_to_rotvec(rotmat)
    pheno = {k: shape[:, l] for l, k in enumerate(body_model.phenotype_labels)
             if k in ("age", "gender", "weight", "height", "muscle", "proportions")}
    homo = torch.zeros(rotmat.shape[0], J, 4, 4, device=rotmat.device)
    homo[..., :3, :3] = rotmat
    homo[..., 3, 3] = 1.0
    out_bm = body_model(pose_parameters=homo, phenotype_kwargs=pheno)
    j3d = out_bm["bone_poses"][:, :, :3, -1]
    center = j3d[:, [body_model.bone_labels.index(cfg.person_center)]]
    v3d = out_bm["vertices"] - center + transl.unsqueeze(1)
    j3d = j3d - center + transl.unsqueeze(1)

    def project(p):
        q = p / p[:, :, -1:]
        return torch.einsum("bij,bkj->bki", Kp, q)[:, :, :2]

    out = {"scores": scores, "scores_logits": logits, "K": K, "K_regressed": K_reg, "fov_regressed": fov,
           "loc": loc, "offset": offset, "dist": dist, "dist_postprocessed": dist_pp, "shape": shape,
           "rotvec": rotvec, "rotmat": rotmat, "v3d": v3d, "j3d": j3d, "j2d": project(j3d), "v2d": project(v3d),
           "transl": transl, "transl_pelvis": j3d[:, [0]], "feat": feat,
           "blendshape_coeffs": out_bm["blendshape_coeffs"]}
    if is_training:
        return out
    persons = []
    for i in range(idx[0].shape[0]):
        persons.append({"K": Kp[i], "K_regressed": K_reg[idx[0]][i], "loc": loc[i], "transl": transl[i],
                        "transl_pelvis": out["transl_pelvis"][i], "rotvec": rotvec[i], "rotmat": rotmat[i],
                        "shape": shape[i], "v3d": v3d[i], "j3d": j3d[i], "j2d": out["j2d"][i], "fov": fov})
    return sorted(persons, key=lambda p: p["transl"][2].item())
