"""Per-rounding-point error budget of the engine's precision contract, on the CPU (oracle `emulate` hook).

Emulates where the engine rounds to fp16 (tensor-core operands / fp16 workspaces) inside the fp32 oracle and
reports the output error vs the golden fixture (= the unmodified reference) with each rounding class switched
off / split in two fp16 terms.  TEST/DIAGNOSTIC TOOL, never on the product path.

    python tools/precision_study.py [case] [--classes ...]
    python tools/precision_study.py --refine [case] [--reuse-o]
    python tools/precision_study.py --fp8 [case ...]        FP8 (e4m3, block-scaled) MLP operands, see fp8_study
"""
import argparse
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import ln_fold_study  # noqa: E402
import parity_util as pu  # noqa: E402
from oracle import multihmr_ref, smplx_ref  # noqa: E402


def r16(t):
    return t.to(torch.float16).to(torch.float32)


def split16(t):
    """two-term fp16 representation (hi + lo): ~22 bits"""
    hi = r16(t)
    return hi + r16(t - hi)


class Emu:
    """rounding points:  <gemm>.in / <gemm>.w / <gemm>.out for gemm in {patch,qkv,proj,fc1,fc2,cls0,kv};
    attn.p (P to fp16), attn.o == proj.in (O16).  mode per point: 'r' round, 'n' none, 's' split (2-term)."""

    def __init__(self, sd, modes=None, default="r", layer_modes=None):
        self.names = {}
        for k, v in sd.items():
            if not k.endswith(".weight"):
                continue
            for tag, cls in (("attn.qkv", "qkv"), ("attn.proj", "proj"), ("mlp.fc1", "fc1"), ("mlp.fc2", "fc2"),
                             ("mlp_classif.0", "cls0"), ("mlp_classif.2", "cls2"), ("to_kv", "kv")):
                if tag in k:
                    layer = -1
                    if "blocks." in k:
                        layer = int(k.split("blocks.")[1].split(".")[0])
                    self.names[id(v)] = (cls, layer)
        self.modes = modes or {}
        self.default = default
        self.layer_modes = layer_modes or {}   # {(point, layer): mode}

    def mode(self, point, layer=-1):
        if (point, layer) in self.layer_modes:
            return self.layer_modes[(point, layer)]
        return self.modes.get(point, self.default)

    def apply(self, t, point, layer=-1):
        m = self.mode(point, layer)
        if m == "r":
            return r16(t)
        if m == "s":
            return split16(t)
        return t

    def __call__(self, x, w, b):
        cls, layer = self.names.get(id(w), (None, -1))
        if cls is None:
            return F.linear(x, w, b)
        if cls == "cls2":
            return F.linear(self.apply(x, "cls2.in"), w, b)
        y = F.linear(self.apply(x, cls + ".in", layer), self.apply(w, cls + ".w", layer), b)
        if cls == "fc1":
            return y  # GELU follows; the rounding of H16 is fc2.in
        if cls in ("qkv",):
            y = self.apply(y, "qkv.out", layer)
        return y

    def attention(self, q, k, v):
        # S fp32, online softmax == plain softmax up to fp32 rounding; P rounded to fp16 un-normalised
        s = torch.matmul(q, k.transpose(-1, -2)) * (q.shape[-1] ** -0.5)
        m = s.amax(dim=-1, keepdim=True)
        p = torch.exp(s - m)
        l = p.sum(dim=-1, keepdim=True)
        o = torch.matmul(self.apply(p, "attn.p"), v) / l
        return o  # rounding to O16 is proj.in

    def conv(self, x_img, w, b, patch):
        return F.conv2d(self.apply(x_img, "patch.in"), self.apply(w, "patch.w"), b, stride=patch)


POINTS = ["patch.in", "patch.w", "qkv.in", "qkv.w", "qkv.out", "attn.p", "proj.in", "proj.w", "fc1.in", "fc1.w",
          "fc2.in", "fc2.w", "cls0.in", "cls0.w", "kv.in", "kv.w"]


def run(name, emu_factory):
    case, sd, bm, x, K, idx = pu.build_inputs(name)
    gold = pu.load_golden(name)
    cfg = multihmr_ref.RefConfig(backbone=case["backbone"], img_size=case["img_size"])
    body = smplx_ref.SMPLXShim(bm, 10)
    res = {}
    with torch.no_grad():
        ref = multihmr_ref.model_forward(sd, body, cfg, x, K, idx=idx, is_training=True, taps=(tr := {}))
        for label, emu in emu_factory(sd):
            taps = {}
            out = multihmr_ref.model_forward(sd, body, cfg, x, K, idx=idx, is_training=True, emulate=emu, taps=taps)
            e = {}
            for k in ("v3d", "rotmat", "shape", "dist", "scores", "expression", "transl"):
                d = (out[k] - gold[k]).abs()
                e[k] = (d.max().item(), d.pow(2).mean().sqrt().item())
            dz = (taps["z"] - tr["z"])
            e["z"] = (dz.abs().max().item(), dz.pow(2).mean().sqrt().item())
            res[label] = e
            print(f"{label:28s} v3d max {e['v3d'][0]:.3e} rms {e['v3d'][1]:.3e} | rotmat max {e['rotmat'][0]:.3e} rms "
                  f"{e['rotmat'][1]:.3e} | z rms {e['z'][1]:.3e} | shape {e['shape'][0]:.2e} dist {e['dist'][0]:.2e} "
                  f"scores {e['scores'][0]:.2e}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("case", nargs="?", default="s_280_L_forced")
    ap.add_argument("--study", default="ablate")
    a = ap.parse_args()
    torch.set_num_threads(min(32, os.cpu_count()))

    def factory(sd):
        yield "all-rounded (engine r01)", Emu(sd)
        yield "none (fp32)", Emu(sd, default="n")
        if a.study == "ablate":
            for p in POINTS:
                yield f"without {p}", Emu(sd, modes={p: "n"})
        elif a.study == "groups":
            g = {
                "weights": [p for p in POINTS if p.endswith(".w")],
                "acts": [p for p in POINTS if not p.endswith(".w")],
                "attn-branch": ["qkv.in", "qkv.w", "qkv.out", "attn.p", "proj.in", "proj.w"],
                "mlp-branch": ["fc1.in", "fc1.w", "fc2.in", "fc2.w"],
                "head": ["cls0.in", "cls0.w", "kv.in", "kv.w"],
                "resid-writers(proj,fc2)": ["proj.in", "proj.w", "fc2.in", "fc2.w"],
                "ln-consumers(qkv,fc1)": ["qkv.in", "qkv.w", "fc1.in", "fc1.w"],
            }
            for label, pts in g.items():
                yield f"without {label}", Emu(sd, modes={p: "n" for p in pts})
        elif a.study == "layers":
            depth = 24 if "L" in a.case.split("_")[2] else 12
            for lo in range(0, depth, 4):
                lm = {(p, l): "n" for p in POINTS for l in range(lo, lo + 4)}
                yield f"without layers {lo}-{lo + 3}", Emu(sd, layer_modes=lm)

    run(a.case, factory)




# ---------------------------------------------------------------------------------------------------
# "refine" study: bulk pass with fp16 operands for every token + an fp32 second pass of the residual
# streams of the detected (central) tokens only, attending over the K/V of the bulk pass.
class RefineEmu(Emu):
    """pass 'record': behaves like Emu and records (k, v) per attention call; pass 'replay': fp32 linears,
    attention of the fp32 queries over the recorded K/V."""

    def __init__(self, sd, reuse_o=False, **kw):
        super().__init__(sd, **kw)
        self.kv = []
        self.o = []
        self.reuse_o = reuse_o   # replay the bulk pass's fp16 attention OUTPUT instead of re-attending
        self.replay = False
        self.i = 0

    def __call__(self, x, w, b):
        if self.replay:
            return F.linear(x, w, b)
        return super().__call__(x, w, b)

    def attention(self, q, k, v):
        if not self.replay:
            self.kv.append((k, v))
            o = super().attention(q, k, v)
            self.o.append(r16(o))
            return o
        k, v = self.kv[self.i]
        self.i += 1
        if self.reuse_o:
            return self.o[self.i - 1]
        s = torch.matmul(q, k.transpose(-1, -2)) * (q.shape[-1] ** -0.5)
        return torch.matmul(s.softmax(dim=-1), v)

    def conv(self, x_img, w, b, patch):
        if self.replay:
            return F.conv2d(x_img, w, b, stride=patch)
        return super().conv(x_img, w, b, patch)


def refine_study(name, reuse_o=False):
    from oracle import dinov2_ref
    case, sd, bm, x, K, idx = pu.build_inputs(name)
    gold = pu.load_golden(name)
    cfg = multihmr_ref.RefConfig(backbone=case["backbone"], img_size=case["img_size"])
    body = smplx_ref.SMPLXShim(bm, 10)
    with torch.no_grad():
        emu = RefineEmu(sd, reuse_o=reuse_o)
        zA = dinov2_ref.get_intermediate_layers(x, sd, cfg.backbone, "backbone.encoder.", emu)
        emu.replay = True
        zB = dinov2_ref.get_intermediate_layers(x, sd, cfg.backbone, "backbone.encoder.", emu)
        zR = dinov2_ref.get_intermediate_layers(x, sd, cfg.backbone, "backbone.encoder.")
        print("z rms err: bulk %.3e  refined rows %.3e" % ((zA - zR).pow(2).mean().sqrt(), (zB - zR).pow(2).mean().sqrt()))
        for label, zc_src in (("bulk only", zA), ("central rows refined", zB)):
            # tail of multihmr_ref.model_forward with z_central taken from zc_src
            emu2 = Emu(sd)
            B, N, D = zA.shape
            h = w = int(math.sqrt(N))
            scores, scores_det, idx_ = multihmr_ref.detection(zA, sd, 3, 0.3, idx, True, emu2)
            b_idx, y_idx, x_idx = idx[0], idx[1], idx[2]
            z_central = zc_src[b_idx, y_idx * w + x_idx]
            offset = multihmr_ref.regression_mlp(z_central, sd, "mlp_offset")
            K_det = K[b_idx]
            z_K = multihmr_ref.embed_camera(K, h, w, cfg)
            z_central = torch.cat([z_central, z_K[b_idx, y_idx, x_idx]], 1)
            z_all = torch.cat([zA, z_K.reshape(B, N, -1)], 2)
            loc = (torch.stack([x_idx, y_idx]).permute(1, 0) + 0.5 + offset) * 14
            rotmat, shape, expression, cam = multihmr_ref.hph_forward(z_central, z_all, idx, sd, cfg, F.linear, emu2)
            rotvec = multihmr_ref.roma_ref.rotmat_to_rotvec(rotmat)
            dist_pp = cam[:, 0][:, None]
            focal = K_det[:, [0], [0]]
            dist = dist_pp * (focal / multihmr_ref.focal_from_fov(cfg.fovn, x.shape[-1]))
            dist = torch.clamp(torch.exp(dist) - 1e-10, 0, 50)
            out = {"rotmat": rotmat, "shape": shape, "dist": dist, "scores": scores, "expression": expression, "loc": loc}
            out.update(multihmr_ref.smpl_layer_forward(body, rotvec, shape, loc, dist, K_det, expression, 15))
            print(label, {k: "%.3e" % (out[k] - gold[k]).abs().max().item() for k in
                          ("v3d", "rotmat", "shape", "dist", "scores", "expression", "transl", "loc", "j3d")})


# ---------------------------------------------------------------------------------------------------
# "fp8" study: the engine's folded bulk pass (tools/ln_fold_study.py) with the operands of fc1 and fc2 in e4m3 with
# power-of-two block scales, with and without the fp32 refinement of the detected rows (which reuses O16).
E4M3_MAX = 448.0
BLOCK = 128


def pow2_scale(amax):
    """s = 2^ceil(log2(amax / 448)) (exact: frexp), 1 for an all-zero block; amax / s <= 448 always."""
    m, e = torch.frexp(amax / E4M3_MAX)
    e = torch.where(m == 0.5, e - 1, e)
    return torch.where(amax > 0, torch.ldexp(torch.ones_like(amax), e), torch.ones_like(amax))


def e4m3(t):
    return t.to(torch.float8_e4m3fn).to(torch.float32)


def q8_act(t):
    """activations: one scale per (row, 128-column block); returns the dequantised operand"""
    sh = t.shape
    b = t.reshape(*sh[:-1], sh[-1] // BLOCK, BLOCK)
    s = pow2_scale(b.abs().amax(-1, keepdim=True))
    return (e4m3(b / s) * s).reshape(sh)


def q8_w(w):
    """weights [N, K]: one scale per (128 output rows x 128 K) block (N padded to a multiple of 128)"""
    N, K = w.shape
    Np = -(-N // BLOCK) * BLOCK
    wp = F.pad(w, (0, 0, 0, Np - N)).reshape(Np // BLOCK, BLOCK, K // BLOCK, BLOCK)
    s = pow2_scale(wp.abs().amax(dim=(1, 3), keepdim=True))
    return (e4m3(wp / s) * s).reshape(Np, K)[:N]


FP8_KEYS = ("scores", "rotvec", "shape", "dist", "loc", "v3d")


# which MLP GEMMs take e4m3 operands: (fc1 A, fc1 W, fc2 A, fc2 W), None = the fp16 engine
FP8_VARIANTS = {"fp16": None, "fp8 fc1+fc2": (q8_act, q8_w) * 2, "fp8 fc1 only": (q8_act, q8_w, r16, r16),
                "fp8 fc2 only": (r16, r16, q8_act, q8_w)}


def _bulk_and_refined(x, sd, backbone, pre, mlp8):
    """(bulk features with cls row, refined features with cls row): the refined pass is the fp32 stream of every
    token fed with the bulk pass's O16, so any row of it is what the engine's refinement computes for that row."""
    zb, outs, _ = ln_fold_study.forward(x, sd, backbone, pre, "fold", mlp8=mlp8, keep_cls=True)
    zr, _, _ = ln_fold_study.forward(x, sd, backbone, pre, "refine", o_in=outs, keep_cls=True)
    return zb, zr


def _err(out, gold, keys=FP8_KEYS):
    # the detection goldens hold the reference's person dicts (no dist)
    return {k: (out[k].reshape(gold[k].shape) - gold[k].float()).abs().max().item() for k in keys if k in gold}


def _smplx_tail(case, sd, bm, x, K, idx, zb, zr):
    """multihmr_ref.model_forward after the backbone, the engine's way: detection, context and to_kv on the bulk
    features (fp16 head operands, Emu), the persons' queries from zr (bulk or refined rows)."""
    cfg = multihmr_ref.RefConfig(backbone=case["backbone"], img_size=case["img_size"])
    body = smplx_ref.SMPLXShim(bm, 10)
    emu = Emu(sd)
    zA, zR = zb[:, 1:], zr[:, 1:]
    B, N, D = zA.shape
    h = w = int(math.sqrt(N))
    forced = idx is not None
    scores, scores_det, idx = multihmr_ref.detection(zA, sd, 3, 0.3, idx, forced, emu)
    b_idx, y_idx, x_idx = idx[0], idx[1], idx[2]
    z_central = zR[b_idx, y_idx * w + x_idx]
    offset = multihmr_ref.regression_mlp(z_central, sd, "mlp_offset")
    K_det = K[b_idx]
    z_K = multihmr_ref.embed_camera(K, h, w, cfg)
    z_central = torch.cat([z_central, z_K[b_idx, y_idx, x_idx]], 1)
    z_all = torch.cat([zA, z_K.reshape(B, N, -1)], 2)
    loc = (torch.stack([x_idx, y_idx]).permute(1, 0) + 0.5 + offset) * 14
    rotmat, shape, expression, cam = multihmr_ref.hph_forward(z_central, z_all, idx, sd, cfg, F.linear, emu)
    rotvec = multihmr_ref.roma_ref.rotmat_to_rotvec(rotmat)
    dist = cam[:, 0][:, None] * (K_det[:, [0], [0]] / multihmr_ref.focal_from_fov(cfg.fovn, x.shape[-1]))
    dist = torch.clamp(torch.exp(dist) - 1e-10, 0, 50)
    out = {"rotvec": rotvec, "shape": shape, "dist": dist, "loc": loc, "scores": scores if forced else scores_det}
    out.update(multihmr_ref.smpl_layer_forward(body, rotvec, shape, loc, dist, K_det, expression, 15))
    return out, torch.stack([b_idx, y_idx, x_idx], 1)


def _anny_tail(case, sd, bm, x, K, idx, zb, zr):
    """oracle.anny_ref.anny_forward with the engine's sources: detection logits and decoder context from the bulk
    features, the camera (cls row) and the persons' queries from zr.  Head in fp32."""
    from unittest import mock

    import anny_util
    from oracle import anny_ref
    pre_hph = anny_ref.hph
    w = int(math.sqrt(zb.shape[1] - 1))
    dim = sd["dec_to_token.weight"].shape[0]
    dec_r = F.linear(zr[:, 1:], sd["dec_to_token.weight"], sd["dec_to_token.bias"]) + sd["dec_pos_emb"].reshape(1, w * w, dim)
    queries = iter([dec_r[b, idx[1][idx[0] == b] * w + idx[2][idx[0] == b]]
                    for b in torch.unique(idx[0], sorted=True).tolist()])

    def hph(q, ctx, sd_, depth, heads):
        return pre_hph(next(queries), ctx, sd_, depth, heads)

    with mock.patch.object(anny_ref, "intermediate_layers_with_cls", lambda *a, **k: (zb[:, 1:], zr[:, 0])), \
            mock.patch.object(anny_ref, "hph", hph):
        out = anny_util.oracle(case, sd, bm, x, K, idx)
    return out, torch.stack([idx[0], idx[1], idx[2]], 1)


def fp8_study(name):
    """max |d| per output vs the golden for the fp16 and the FP8-MLP bulk pass, each without and with refinement;
    returns {(variant, refined): (persons, same detections, {output: max |d|})}"""
    anny = name.startswith("anny")
    if anny:
        import anny_util
        case, sd, bm, x, K, idx = anny_util.build_inputs(name)
        gold, pre, tail = anny_util.load_golden(name), "encoder.backbone.", _anny_tail
    else:
        case, sd, bm, x, K, idx = pu.build_inputs(name)
        gold, pre, tail = pu.load_golden(name), "backbone.encoder.", _smplx_tail
    res = {}
    with torch.no_grad():
        for variant, mlp8 in FP8_VARIANTS.items():
            zb, zr = _bulk_and_refined(x, sd, case["backbone"], pre, mlp8)
            for refined in (False, True):
                out, det = tail(case, sd, bm, x, K, idx, zb, zr if refined else zb)
                label = f"{variant:12s} {'refined' if refined else 'bulk   '}"
                n_gold = gold["v3d"].shape[0]
                # natural detections: the same count, each within half a patch of the golden's location
                same = det.shape[0] == n_gold and ("idx" in gold or
                                                   (out["loc"] - gold["loc"]).abs().max().item() < 7.0)
                e = _err(out, gold) if det.shape[0] == n_gold else {}
                res[(variant, refined)] = (det.shape[0], same, e)
                print(f"{name:18s} {label}  persons {det.shape[0]}/{n_gold} {'same' if same else 'DIFFERENT'}  " +
                      " ".join(f"{k} {v:.2e}" for k, v in e.items()), flush=True)
    return res


if __name__ == "__main__":
    if "--fp8" in sys.argv:
        torch.set_num_threads(min(32, os.cpu_count()))
        for n in [a for a in sys.argv[1:] if not a.startswith("--")] or ["s_224_S_forced", "s_224_S_detect",
                                                                         "s_224_S_outliers", "s_280_L_forced",
                                                                         "anny_280_L_forced"]:
            fp8_study(n)
    elif "--refine" in sys.argv:
        torch.set_num_threads(min(32, os.cpu_count()))
        names = [a for a in sys.argv[1:] if not a.startswith("--")] or ["s_280_L_forced"]
        refine_study(names[0], reuse_o="--reuse-o" in sys.argv)
    else:
        main()
