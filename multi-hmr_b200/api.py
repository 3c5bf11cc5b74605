"""The inference glue the reference keeps in demo.py:27-126, with identical signatures, so that callers
(`demo.py:334`, `app.py:132`, `train.py:356`) can switch to this package for the `Model.forward` path:

    open_image, get_camera_parameters, load_model, forward_model

plus `open_images`, the batched form of `open_image`, and `create_jpeg`, the dataset conversion of
datasets/bedlam.py:449-479.  JPEG and PNG decoding (of the files the device takes), the
letterbox (resize + pad) and the forward are H100-native; other files are decoded on the host (PIL), as in the
reference.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from .model import Model
from .model_anny import ModelAnny

from .preprocess import IMG_NORM_MEAN, IMG_NORM_STD, device_table, letterbox, normalize_rgb, normalize_rgb_table  # noqa: F401

SMPLX_DIR = "models"                         # utils/constants.py:7
CACHE_DIR_MULTIHMR = "models/multiHMR"       # utils/constants.py:9


def normalize_rgb_device(img_u8: torch.Tensor) -> torch.Tensor:
    """uint8 [B,H,W,3] on a CUDA device -> normalised fp32 [B,3,H,W], bit-identical to `normalize_rgb` on the
    host (hand-written kernel, `mhmr_op_normalize_u8`); 4x less to upload than the fp32 image."""
    from . import ops

    return ops.normalize_u8(img_u8.contiguous(), device_table(img_u8.device))


def _upload_pil(im, device):
    """A decoded RGB photo copied once into pinned memory and uploaded once."""
    host = torch.empty((im.height, im.width, 3), dtype=torch.uint8, pin_memory=True)
    host.numpy()[...] = np.asarray(im)
    return host.to(device, non_blocking=True)


def _letterbox_photos(imgs_pil, img_size, device, fused):
    """Decoded RGB photos -> (batch, full-resolution uint8 [H, W, 3] device photos, boxes): each photo is uploaded once
    (`_upload_pil`) and letterboxed on the device (`_letterbox_device`)."""
    return _letterbox_device([_upload_pil(im, device) for im in imgs_pil], img_size, fused)


def _letterbox_device(photos, img_size, fused):
    """Full-resolution uint8 [H, W, 3] device photos -> (batch, the photos, boxes): the device letterbox
    (`preprocess.letterbox`) makes the uint8 [B, S, S, 3] batch, normalised to fp32 [B, 3, S, S] unless `fused`."""
    u8, boxes = letterbox(photos, img_size)
    if fused:
        return u8, photos, boxes
    if img_size % 2:
        raise ValueError("the device normalisation needs an even img_size")
    B = u8.shape[0]   # viewed as rows of 4 pixels: the same pixels, channel planes of S*S values
    x = normalize_rgb_device(u8.view(B, img_size * img_size // 4, 4, 3)).view(B, 3, img_size, img_size)
    return x, photos, boxes


def open_images(paths, img_size, device=torch.device("cuda"), fused=False):
    """`open_image` for a batch of photo files of any sizes, on the device.  Pillow first opens every file's header
    in order (`Image.open`, which decodes nothing), so a file it refuses (not an image, a decompression bomb, ...)
    raises exactly as before and no device memory is spent on it.  The bytes of the files Pillow opened as RGB or gray
    go up in one pinned upload, and the baseline ones among them are decoded there in one call
    (`preprocess.decode_jpeg`); the PNGs it opened as RGB, gray, palette, RGBA or gray + alpha go up in another, and
    the eligible ones (8-bit, not interlaced) are decoded there in one call (`preprocess.decode_png`).  Both are byte
    for byte `Image.open(p).convert("RGB")`; each call's statuses come back in one host synchronisation.  Any other
    file (progressive or arithmetic-coded JPEG, CMYK, 4:1:1, interlaced or 16-bit PNG, ...) and any file the device
    flagged is decoded on the host with Pillow, in file order, and uploaded once.
    The batch is then letterboxed on the device, byte for byte as `ImageOps.contain` + `ImageOps.pad`.  Returns
    (normalised fp32 [B, 3, S, S], or with `fused=True` the uint8 [B, S, S, 3] batch that `Model.forward` /
    `forward_model` take through the fused loader; the full-resolution uint8 [H, W, 3] device photos, the renderer's
    backgrounds; int32 [B, 4] host tensor of (x0, y0, new_w, new_h), each photo's box in the square)."""
    from PIL import Image

    from .preprocess import decode_jpeg, decode_png

    device = torch.device(device)
    if device.type != "cuda":
        raise ValueError("open_images letterboxes on a CUDA device (open_image is the host path)")
    # Headers in file order; Pillow's decode of file i used to run before file i + 1 was opened, so an open error is
    # raised only after the files before it have been decoded (and have raised, if they fail to decode).
    ims, open_error = [], None
    for p in paths:
        try:
            ims.append(Image.open(p))
        except Exception as err:   # noqa: BLE001  (re-raised below, unchanged)
            open_error = err
            break
    try:
        jpegs, pngs = [], []
        for p, im in zip(paths, ims):
            jpeg = im.mode in ("RGB", "L")
            png = im.format == "PNG" and im.mode in ("RGB", "L", "P", "RGBA", "LA")
            blob = b""
            if jpeg or png:
                with open(p, "rb") as fh:
                    blob = fh.read()
            jpegs.append(blob if jpeg else b"")
            pngs.append(blob if png else b"")
        with torch.cuda.device(device):
            photos, ok = decode_jpeg(jpegs, device)
            if any(pngs):
                png_photos, png_ok = decode_png(pngs, device)
                for i, good in enumerate(png_ok):
                    if good:
                        photos[i], ok[i] = png_photos[i], True
            for i, im in enumerate(ims):
                if not (ok[i] and im.size == (photos[i].shape[1], photos[i].shape[0])):
                    photos[i] = _upload_pil(im.convert("RGB"), device)
            if open_error is not None:
                raise open_error
            return _letterbox_device(photos, img_size, fused)
    finally:
        for im in ims:
            im.close()


def open_image(img_path, img_size, device=torch.device("cuda"), fused=False):
    """Open, resize keeping the aspect ratio, zero-pad to a square, normalise (demo.py:27-51).  On a CUDA
    device the full-resolution photo is uploaded, letterboxed and normalised there (`open_images` of one photo: the
    same bytes as the host path).  `fused=True` returns the uint8 [1,S,S,3] device tensor itself: `Model.forward` /
    `forward_model` then run the fused loader (uint8 -> normalised fp16 patch rows, `mhmr_forward_u8`) and the fp32
    image never exists."""
    from PIL import Image, ImageOps

    img_pil = Image.open(img_path).convert("RGB")
    img_pil_full = img_pil.copy()
    device = torch.device(device)
    if device.type == "cuda" and img_size % 4 == 0:
        with torch.cuda.device(device):
            return _letterbox_photos([img_pil], img_size, device, fused)[0], img_pil_full
    img_pil = ImageOps.contain(img_pil, (img_size, img_size))
    img_pil = ImageOps.pad(img_pil, size=(img_size, img_size))
    x = torch.from_numpy(normalize_rgb(np.asarray(img_pil))).unsqueeze(0).to(device)
    return x, img_pil_full


def create_jpeg(root_dir, target_size=512, device=torch.device("cuda"), batch=16):
    """datasets/bedlam.py:449-479 on the device, writing the same files byte for byte: every `.png` under `root_dir`
    whose name does not start with '.', in `os.walk` order, opened as RGB, resized (BICUBIC) so that its long side is
    `target_size` (the other `int(side * target_size / long_side)`; the width counts as the long side only when it is
    strictly longer) and saved as a default-quality JPEG next to it as `<name>_<target_size>.jpg`, or unresized as
    `<name>.jpg` when `target_size` is None.  Files go through the device `batch` at a time: PNG decode
    (`preprocess.decode_png`; Pillow for the files it does not take), resize, JPEG encode."""
    import sys

    from PIL import Image

    from .preprocess import decode_png, encode_jpeg, resize

    device = torch.device(device)
    log_freq = 1000
    print(f"ROOT_DIR: {root_dir}")
    jobs = [os.path.join(dirpath, fn) for dirpath, _, filenames in os.walk(root_dir)
            for fn in filenames if fn[-4:] == ".png" and fn[0] != "."]
    tot = 0
    for k in range(0, len(jobs), batch):
        paths = jobs[k:k + batch]
        blobs = []
        for path in paths:
            with open(path, "rb") as fh:
                blobs.append(fh.read())
        photos, ok = decode_png(blobs, device)
        for i, path in enumerate(paths):
            if not ok[i]:
                photos[i] = _upload_pil(Image.open(path).convert("RGB"), device)
        if target_size is not None:
            sizes = []
            for p in photos:
                height, width = p.shape[:2]
                if width > height:
                    sizes.append((target_size, int(float(height) * float(target_size / float(width)))))
                else:
                    sizes.append((int(float(width) * float(target_size / float(height))), target_size))
            photos = resize(photos, sizes)
            names = [p[:-4] + f"_{target_size}.jpg" for p in paths]
        else:
            names = [p[:-4] + ".jpg" for p in paths]
        for name, data in zip(names, encode_jpeg(photos)):
            with open(name, "wb") as fh:
                fh.write(data)
            tot += 1
            if tot % log_freq == 0:
                print(f"Converted {tot} images so far")
                sys.stdout.flush()


def get_focalLength_from_fieldOfView(fov=60, img_size=512):
    """utils/camera.py:50-60."""
    return img_size / (2 * np.tan(np.radians(fov) / 2))


def get_camera_parameters(img_size, fov=60, p_x=None, p_y=None, device=torch.device("cuda")):
    """K [1,3,3] from image size, field of view and principal point (demo.py:53-68)."""
    K = torch.eye(3)
    focal = get_focalLength_from_fieldOfView(fov=fov, img_size=img_size)
    K[0, 0], K[1, 1] = focal, focal
    if p_x is not None and p_y is not None:
        K[0, -1], K[1, -1] = p_x * img_size, p_y * img_size
    else:
        K[0, -1], K[1, -1] = img_size // 2, img_size // 2
    return K.unsqueeze(0).to(device)


def body_model_from_smplx_npz(path: str, num_betas: int = 10) -> dict:
    """Reads `SMPLX_NEUTRAL.npz` the way `smplx.create(..., use_pca=False, flat_hand_mean=True)` does
    (blocks/smpl_layer.py:38): shapedirs[..., :num_betas] + 10 expression directions (stored after the 300
    shape components), posedirs reshaped to [486, 3V], kinematic parents from kintree_table[0]."""
    d = np.load(path, allow_pickle=True)
    t = lambda a, dt=torch.float32: torch.as_tensor(np.asarray(a)).to(dt)
    sdirs = t(d["shapedirs"])
    V = sdirs.shape[0]
    n_shape = 300 if sdirs.shape[-1] >= 310 else sdirs.shape[-1] - 10
    parents = t(d["kintree_table"][0].astype(np.int64), torch.int64)
    parents[0] = -1
    required = ("lmk_faces_idx", "lmk_bary_coords")
    for k in required:
        if k not in d:
            raise KeyError(f"{path} lacks {k} (static face landmarks)")
    if "extra_joints_idxs" in d:
        extra = t(d["extra_joints_idxs"], torch.int64)
    else:  # smplx.vertex_ids.vertex_ids['smplx']: nose, eyes, ears, feet, finger tips
        extra = torch.tensor([9120, 9929, 9448, 616, 6, 5770, 5780, 8846, 8463, 8474, 8635,
                              5361, 4933, 5058, 5169, 5286, 8079, 7669, 7794, 7905, 8022], dtype=torch.int64)
    return {
        "v_template": t(d["v_template"]), "shapedirs": sdirs[..., :num_betas],
        "shapedirs_extra": sdirs[..., num_betas:num_betas + 1], "expr_dirs": sdirs[..., n_shape:n_shape + 10],
        "posedirs": t(d["posedirs"]).reshape(-1, 486).T.contiguous(), "J_regressor": t(d["J_regressor"]),
        "parents": parents, "lbs_weights": t(d["weights"]), "faces": t(d["f"].astype(np.int64), torch.int64),
        "lmk_faces_idx": t(d["lmk_faces_idx"].astype(np.int64), torch.int64),
        "lmk_bary_coords": t(d["lmk_bary_coords"]), "extra_joints_idxs": extra, "num_verts": V,
    }


# smplx.vertex_ids.vertex_ids['smplh'] in the order of smplx.vertex_joint_selector.VertexJointSelector: face (nose,
# reye, leye, rear, lear), feet (LBigToe, LSmallToe, LHeel, RBigToe, RSmallToe, RHeel), then the finger tips of the
# left and the right hand (thumb, index, middle, ring, pinky).  [3P-memory]: recalled from the smplx package, which is
# not installed here; re-verify against smplx/vertex_ids.py before relying on SMPL joints 24..44.
SMPL_EXTRA_JOINTS_IDXS = [332, 6260, 2800, 4071, 583, 3216, 3226, 3387, 6617, 6624, 6787,
                          2746, 2319, 2445, 2556, 2673, 6191, 5782, 5905, 6016, 6133]

# Classes a body-model pickle may name: numpy / scipy containers, and chumpy's array wrapper, which is replaced by the
# ndarray it holds (chumpy is not a dependency).  Anything else is refused.
_PICKLE_NUMPY = {("numpy", "ndarray"), ("numpy", "dtype"), ("numpy.core.multiarray", "_reconstruct"),
                 ("numpy._core.multiarray", "_reconstruct"), ("numpy.core.multiarray", "scalar"),
                 ("numpy._core.multiarray", "scalar"), ("copyreg", "_reconstructor"), ("copy_reg", "_reconstructor"),
                 ("builtins", "object"), ("__builtin__", "object"), ("_codecs", "encode"),
                 ("builtins", "set"), ("__builtin__", "set"), ("builtins", "frozenset"), ("__builtin__", "frozenset")}
_PICKLE_SCIPY = {"csc_matrix", "csr_matrix"}


class _ChumpyArray:
    """Stand-in for a pickled chumpy object: keeps its state; `_unchumpy` swaps it for the ndarray it wraps."""

    def __init__(self, *args, **kwargs):
        pass

    def __setstate__(self, state):
        self.__dict__.update(state if isinstance(state, dict) else {})


class _BodyModelUnpickler:
    @staticmethod
    def make(fh):
        import pickle

        class U(pickle.Unpickler):
            def find_class(self, module, name):
                if (module, name) in _PICKLE_NUMPY:
                    return super().find_class(module, name)
                if module.split(".")[0] == "scipy" and module.startswith("scipy.sparse") and name in _PICKLE_SCIPY:
                    return super().find_class(module, name)
                if module.split(".")[0] == "chumpy":
                    return _ChumpyArray
                raise pickle.UnpicklingError(f"refusing to unpickle {module}.{name}")

        return U(fh, encoding="latin1")


def _unchumpy(obj):
    if isinstance(obj, _ChumpyArray):
        if "x" not in obj.__dict__:
            raise ValueError("chumpy object without a stored value ('x')")
        return np.asarray(_unchumpy(obj.__dict__["x"]))
    if isinstance(obj, dict):
        return {k: _unchumpy(v) for k, v in obj.items()}
    return obj


def load_body_model_pickle(path: str) -> dict:
    """A body-model pickle (SMPL_*.pkl, smplx2smpl.pkl) through a restricted unpickler: numpy and scipy.sparse
    containers only, chumpy arrays mapped to their ndarray (the layout SMPL's python-2 pickles use: chumpy.ch.Ch with
    its value in 'x' -- [3P-memory], re-verify against chumpy/ch.py)."""
    with open(path, "rb") as fh:
        return _unchumpy(_BodyModelUnpickler.make(fh).load())


def body_model_from_smpl_pkl(path: str, num_betas: int = 10) -> dict:
    """Reads `SMPL_{MALE,FEMALE}.pkl` the way `smplx.create(SMPLX_DIR, 'smpl', gender=...)` does (train.py:42-43):
    shapedirs[..., :num_betas], posedirs [V,3,207] -> [207, 3V], J_regressor densified, kinematic parents from
    kintree_table[0], the 21 vertex-picked joints of smplx.vertex_ids['smplh']."""
    d = load_body_model_pickle(path)
    t = lambda a, dt=torch.float32: torch.as_tensor(np.asarray(a)).to(dt)
    jr = d["J_regressor"]
    jr = jr.toarray() if hasattr(jr, "toarray") else np.asarray(jr)
    pd = np.asarray(d["posedirs"])
    parents = t(np.asarray(d["kintree_table"])[0].astype(np.int64), torch.int64)
    parents[0] = -1
    return {
        "v_template": t(d["v_template"]), "shapedirs": t(d["shapedirs"])[..., :num_betas],
        "posedirs": t(pd.reshape(-1, pd.shape[-1]).T.copy()), "J_regressor": t(jr), "parents": parents,
        "lbs_weights": t(d["weights"]), "faces": t(np.asarray(d["f"]).astype(np.int64), torch.int64),
        "extra_joints_idxs": torch.tensor(SMPL_EXTRA_JOINTS_IDXS, dtype=torch.int64),
        "num_verts": int(np.asarray(d["v_template"]).shape[0]),
    }


def load_smplx2smpl(path: str) -> np.ndarray:
    """`smplx2smpl.pkl['matrix']` [6890, 10475] as fp32 (train.py:44-45)."""
    m = load_body_model_pickle(path)["matrix"]
    return np.asarray(m.toarray() if hasattr(m, "toarray") else m, dtype=np.float32)


def load_j_regressor_h36m(path: str) -> np.ndarray:
    """`J_regressor_h36m.npy` [17, 6890] (train.py:400)."""
    return np.load(path).astype(np.float32)


def load_model(model_name, device=torch.device("cuda"), max_batch=8, max_persons=None, body_model=None):
    """Open a checkpoint, build the engine from its saved arguments, load the weights (demo.py:70-106).
    No download is attempted (this build has no network): a missing file is an error.  A checkpoint whose name
    contains 'anny' builds the Anny variant (demo.py:95-96) with `body_model`, or with the `anny` package's
    full-body model when none is given."""
    ckpt_path = os.path.join(CACHE_DIR_MULTIHMR, model_name + ".pt")
    if not os.path.isfile(ckpt_path):
        raise FileNotFoundError(f"{ckpt_path} not found (place the reference checkpoint there)")
    ckpt = torch.load(ckpt_path, map_location="cpu", weights_only=False)
    if "anny" in ckpt_path:
        model = ModelAnny(max_batch=max_batch, max_persons=max_persons, body_model=body_model, device=device,
                          **vars(ckpt["args"]))
        model.load_state_dict(ckpt["model_state_dict"], strict=False)
        return model.finalize()
    kwargs = dict(vars(ckpt["args"]))
    kwargs["type"] = ckpt["args"].train_return_type
    kwargs["img_size"] = ckpt["args"].img_size[0]
    smplx_npz = os.path.join(SMPLX_DIR, "smplx", "SMPLX_NEUTRAL.npz")
    bm = body_model_from_smplx_npz(smplx_npz, kwargs.get("num_betas", 10))
    model = Model(max_batch=max_batch, max_persons=max_persons, body_model=bm, device=device, **kwargs)
    model.load_state_dict(ckpt["model_state_dict"], strict=False)
    return model.finalize()


class HostBatchLoader:
    """Double-buffered upload of (image batch, intrinsics) from pinned host memory on a copy stream: a serving loop
    submits batch i+1 while batch i is inside `Model.forward`, so the host->device copy (19 MB of uint8 for 8 images
    at 896x896) overlaps the previous forward instead of preceding its own.  `get()` makes the current stream wait
    for the copy and hands the device tensors to `forward_model`."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device)
        self._pending = None

    def submit(self, images: torch.Tensor, K: torch.Tensor):
        with torch.cuda.stream(self.stream):
            x = images.to(self.device, non_blocking=True)
            k = K.to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self._pending = (x, k, ev)

    @property
    def pending(self) -> bool:
        return self._pending is not None

    def get(self):
        x, k, ev = self._pending
        self._pending = None
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(ev)
        x.record_stream(cur)
        k.record_stream(cur)
        return x, k


def overlay_human_meshes(humans, faces, K, model, img_pil, unique_color=False, alpha=0.8, _color=None):
    """demo.py:128-158: the persons of `forward_model` drawn over the photo with `render.render_meshes`, on the
    device (the vertices stay there).  Colours default to this package's `render.PALETTE` (the first one for
    every person with `unique_color`).  Returns (uint8 array [H,W,3], colours)."""
    from .render import PALETTE, render_meshes

    if _color is None:
        _color = [PALETTE[0] for _ in range(len(humans))] if unique_color else list(PALETTE)
    K0 = torch.as_tensor(K)[0].detach().cpu().double().numpy()
    focal, princpt = np.asarray([K0[0, 0], K0[1, 1]]), np.asarray([K0[0, -1], K0[1, -1]])
    arr = np.asarray(img_pil)
    if len(humans) > 0:
        name = "verts_smplx" if "verts_smplx" in humans[0] else "v3d"
        arr = render_meshes(arr, [h[name] for h in humans], [faces] * len(humans),
                            {"focal": focal, "princpt": princpt}, alpha=alpha, color=_color)
    return arr, _color


def create_rotating_video(humans, faces, K, model, img_pil_visu, unique_color=False, alpha=0.8, fn=None, n_frames=20,
                          angle_range=60):
    """demo.py:188-241: the frames of the rotating video of one image's persons, as a list of uint8 [H,W,3] arrays
    (None without persons): the overlay on the photo, then orbits about the first person's centroid (y by
    +angle_range, y by -angle_range, x by +angle_range) over white, each sweep forth and back, the overlay between.
    All distinct frames come from one render call on the device.  Writing the video is the caller's: `fn` must
    be None."""
    from .render import PALETTE, _humans_dict, _person_colors, renderer_for

    if fn is not None:
        raise NotImplementedError("create_rotating_video returns the frames; encode them to a video file yourself")
    if len(humans) == 0:
        return None
    _color = [PALETTE[0] for _ in range(len(humans))] if unique_color else list(PALETTE)
    photo = np.asarray(img_pil_visu)
    if photo.dtype != np.uint8:
        raise ValueError("img_pil_visu must be an 8-bit RGB image")
    dev = torch.device("cuda")
    t = _humans_dict(humans, dev, "verts_smplx" if "verts_smplx" in humans[0] else "v3d")  # demo.py:195
    r = renderer_for(faces, t["v3d"].shape[1], dev)
    cols = torch.tensor(np.asarray(_person_colors(_color, len(humans)), np.float64)[:, :3], dtype=torch.float32)
    out = r.render_views(t, torch.from_numpy(np.ascontiguousarray(photo[..., :3]))[None].to(dev),
                         torch.as_tensor(K)[:1], orbit=(n_frames, angle_range), alpha=alpha, colors=cols)
    seq = torch.cat([out["overlay"], out["orbit"][0]]).cpu().numpy()
    return [seq[i] for i in out["frame_order"]]


def forward_model(model, input_image, camera_parameters, det_thresh=0.3, nms_kernel_size=1):
    """One forward on an image batch and its intrinsics (demo.py:108-126).  The reference wraps the call in
    no_grad + fp16 autocast; here precision is fixed by the kernels (fp16 tensor-core operands, fp32
    accumulation / residual stream / softmax / head)."""
    return model(input_image, is_training=False, nms_kernel_size=int(nms_kernel_size), det_thresh=det_thresh,
                 K=camera_parameters)
