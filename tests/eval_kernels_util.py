"""fp64 references, case builders and error bounds of the evaluation kernels (csrc/metrics.cu): the greedy 2-D
matching (`mhmr_eval_match_2d`), PVE / PA-PVE (`mhmr_eval_points_error`) and the sparse pair regression
(`mhmr_eval_regress`).  Shared by tests/test_eval_kernels_cpu.py (the premises) and tests/test_eval_kernels_gpu.py.

Matching.  The oracle is `oracle.eval_ref.match_2d_greedy` (pinned to the reference's own function by the goldens),
fed float64 copies of the exact fp32 inputs.  The builders make the greedy order well defined:
  * person k's joints are B + s_k U (+ garbage on joints the valid mask drops), with B and U integer [J, 2] shared by
    every person.  The difference of a pair is (s_p - s_g) U on the valid joints, so its spectral norm is
    |s_p - s_g| ||U||_2.  Predictions take s_p = A_p >= 0 and ground truths s_g = -1 - B_g, where A_p and B_g put the
    bits of two random 6-bit labels on disjoint bit positions: every |s_p - s_g| = 1 + A_p + B_g is a distinct integer
    <= 4096, so consecutive errors differ by >= 2.4e-4 relative, in fp32 (the reference's arithmetic) and in fp64;
  * designed exact ties duplicate persons, which gives identical bits in both precisions;
  * joint coordinates are integers (boxes at least 1 px in each direction, as the reference asserts), and every
    IoU is >= 1e-3 away from the threshold, except in the threshold-edge cases, whose dyadic thresholds (0.25, 0.5)
    make the IoU exact in fp32.

Points.  The kernel centres in fp32 (`X - c`, one fp32 subtraction, bitwise what numpy fp32 does) and does everything
else in double.  The oracle centres the same way, then runs in fp64 with `oracle.roma_ref.rigid_points_registration`.
Bounds (mm):
  * PVE: fp32 difference, sum of squares (FMA contraction allowed) and sqrtf per point, then the double mean and one
    fp32 rounding: 1000 * 6u * mean|d_i| + 1/2 ulp32(out);
  * PA: after centring all work is double: 1/2 ulp32(out) + 1e-8 out + 1000 * 2^-40 * max|coord|, plus the scale
    error of rank-deficient sets (n = 3, coplanar, collinear).  There the kernel takes sigma_k = sqrt(w_k) of a zero
    eigenvalue of M^T M known to ~16 eps sigma1^2, i.e. sigma_k ~ 4 sqrt(eps) sigma1 = 4e-8 sigma1: s moves by that
    over sxx, and each aligned point by that times |xhat_i|.  The term vanishes on full-rank sets.  It is needed: the
    numpy port of the kernel's algorithm reaches 0.8 of the bound without it on a 3-point set
    (tests/test_eval_kernels_cpu.py), and the device's PA of an exact 3-point fit is ~5e-6 mm, about 2000 times the
    bound without it.  The absolute floor covers exact fits of full rank.
  Excluded: with d = det(U) det(V) = -1 and sigma2 = sigma3 the optimal rotation is a continuum, so the mean-norm PA is
  not defined.  Builders keep sigma2 - sigma3 >= 1e-3 sigma1 whenever d = -1; every other degeneracy here (coplanar,
  collinear, isotropic, sigma1 ~ sigma2, exact fits, far from the origin) has a unique PA and is in scope.

Regression.  y = A[rows] (X - c) - A[root] (X - c) in fp64.  Each lane of the kernel does ceil(nnz / 32) fmaf, then 5
shuffle levels and the centring: (ceil(nnz / 32) + 6) u sum |w| |x - c| per row, the root row's bound added, plus the
subtraction.  The projection bound propagates that through y / y_z and K.

Planted mistakes (variants of the oracles, which the tests show fall outside the bounds):
  matching    spectral norm -> Frobenius; IoU without the +1 pixel; ties broken by the last index; false positives
              counted per prediction instead of per popped pair
  points      no reflection fix; scale from sigma1 + sigma2 + sigma3 (no d); s = 1; R transposed; PVE centred on the
              mean instead of the given centre
  regression  regressing before centring; root not subtracted; projection with the K of the pair's other side"""
import math

import numpy as np
import torch

from oracle import eval_ref, roma_ref

U = 2.0 ** -24
F32, F64 = np.float32, np.float64

# ------------------------------------------------------------------------------------------------------ matching
PG_SWEEP = (0, 1, 2, 31, 32, 33, 47, 48)
J_SWEEP = (2, 14, 17, 31, 32, 33, 44, 127)
MIN_SEP = 1e-4
IOU_MARGIN = 1e-3
OFFSET = 5000  # image coordinates of the shared joint layout B
MATCH_MISTAKES = ("frobenius", "no_plus1", "tie_last", "fp_per_prediction")
# (P, G, J, masked): every P x G of the sweeps (G >= 1, the entry's minimum), J and the mask taking turns
MATCH_CASES = [(P, G, J_SWEEP[i % len(J_SWEEP)], bool(i % 2)) for i, (P, G) in
               enumerate((P, G) for P in PG_SWEEP for G in PG_SWEEP if G > 0)]


def _bit_labels(n, positions, rng):
    labels = rng.permutation(64)[:n]
    return np.array([sum(((int(i) >> b) & 1) << int(positions[b]) for b in range(6)) for i in labels], np.int64)


def _pick_threshold(iou, prefer=0.05):
    """`prefer` if every IoU is >= IOU_MARGIN away from it, else the nearest fp32 threshold in [0.02, 0.6] that is."""
    iou = np.asarray(iou, F64).ravel()
    cands = sorted(set([prefer] + np.round(np.linspace(0.02, 0.6, 581), 4).tolist()), key=lambda t: abs(t - prefer))
    for t in cands:
        t32 = float(F32(t))
        if iou.size == 0 or np.abs(iou - t32).min() >= IOU_MARGIN:
            return t32
    raise RuntimeError("no threshold with the IoU margin")


def iou_matrix(pred, gt, plus1=True):
    P, G = len(pred), len(gt)
    out = np.zeros((P, G))
    for p in range(P):
        for g in range(G):
            out[p, g] = eval_ref.get_bbx_overlap(pred[p].astype(F64), gt[g].astype(F64)) if plus1 else \
                _iou_no_plus1(pred[p].astype(F64), gt[g].astype(F64))
    return out


def _iou_no_plus1(p1, p2):
    mn1, mn2, mx1, mx2 = p1.min(0), p2.min(0), p1.max(0), p2.max(0)
    xl, yt, xr, yb = max(mn1[0], mn2[0]), max(mn1[1], mn2[1]), min(mx1[0], mx2[0]), min(mx1[1], mx2[1])
    inter = max(0, xr - xl) * max(0, yb - yt)
    return inter / float((mx1[0] - mn1[0]) * (mx1[1] - mn1[1]) + (mx2[0] - mn2[0]) * (mx2[1] - mn2[1]) - inter)


def match_case(P, G, J, masked, seed, fixed_thresh=False):
    """(pred fp32 [P,J,2], gt fp32 [G,J,2], vmask bool [G,J] or None, thresh) with the promises of the module
    docstring; with `masked`, every ground truth drops the joints of one whole lane-stride slice (j = l mod 32) plus
    some random others, and the dropped joints carry garbage that would move the errors if they were counted."""
    for attempt in range(200 if fixed_thresh else 50):
        rng = np.random.default_rng(1000 * seed + attempt)
        pos = rng.permutation(12)
        a, b = _bit_labels(P, pos[:6], rng), _bit_labels(G, pos[6:], rng)
        lane_set = []
        if masked:
            lane = int(rng.integers(min(J, 32)))
            lane_set = list(range(lane, J, 32))
        rest = [j for j in range(J) if j not in lane_set]
        S = rng.permutation(rest)[:min(8, len(rest))]
        Um = np.zeros((J, 2), np.int64)
        cyc = np.array([[1, 0], [0, 1], [-1, 0], [0, -1]])
        for i, j in enumerate(S):
            Um[j] = cyc[i % 4]
        B = rng.integers(-3, 4, size=(J, 2)) + OFFSET
        pred = np.stack([B + a[p] * Um for p in range(P)]) if P else np.zeros((0, J, 2), np.int64)
        gt = np.stack([B + (-1 - b[g]) * Um for g in range(G)])
        vmask = None
        if masked:
            vmask = np.ones((G, J), bool)
            free = [j for j in rest if j not in set(S.tolist())]
            for g in range(G):
                drop = lane_set + [j for j in free if rng.random() < 0.3]
                vmask[g, drop] = False
                gt[g, drop] += rng.integers(-40, 41, size=(len(drop), 2))
            for p in range(P):
                pred[p, lane_set] += rng.integers(-40, 41, size=(len(lane_set), 2))
        pred, gt = pred.astype(F32), gt.astype(F32)
        if any(len(q) and ((q.max(1) - q.min(1)) < 1).any() for q in (pred, gt)):
            continue  # a box thinner than 1 px (the reference asserts against it)
        thr = _pick_threshold(iou_matrix(pred, gt))
        if fixed_thresh and thr != float(F32(0.05)):
            continue  # Evaluator's matching runs at the reference's 0.05
        try:
            match_reference(pred, gt, vmask, thr)
        except RuntimeError:  # every candidate consumed: the reference would loop forever, outside the contract
            continue
        return pred, gt, vmask, thr
    raise RuntimeError("no well-posed matching case")


def _rect(x0, y0, x1, y1):
    return [[x0, y0], [x1, y0], [x0, y1], [x1, y1]]


def dedicated_match_cases():
    """{name: (pred, gt, vmask, thresh)}: exact ties, IoU exactly at a dyadic threshold next to a box one pixel
    narrower, the reference's early end on false positives, and a spectral-vs-Frobenius order."""
    cases = {}
    base = np.array(_rect(100, 100, 130, 130), F64)
    cyc = np.array([[1, 0], [0, 1], [-1, 0], [0, -1]], F64)
    # ties: two identical ground truths, predictions 1 and 2 identical -> four equal errors, row-major first wins
    gt = np.stack([base, base])
    pred = np.stack([base + 3 * cyc, base + cyc, base + cyc])
    cases["ties"] = (pred, gt, None, float(F32(0.05)))
    # IoU == threshold (matched) next to a box one pixel narrower (false positive), both orders of discovery: the
    # exact box first, or (its inner joints moved to its far corners) the narrower one popped and counted first
    inner = [[2, 2], [3, 2], [1, 1]] * 3
    g = np.array(_rect(0, 0, 9, 9) + inner, F64)
    for thr, exact, narrow in ((0.5, _rect(0, 0, 9, 4), _rect(0, 0, 9, 3)), (0.25, _rect(0, 0, 4, 4), _rect(0, 0, 3, 4))):
        e, nw = np.array(exact + inner, F64), np.array(narrow + inner, F64)
        cases[f"iou_edge_{thr}"] = (np.stack([e, nw]), g[None], None, thr)
        bx, by = exact[3]
        far = np.array(exact + [[bx, by], [0, by], [bx, 0]] * 3, F64)
        cases[f"iou_edge_{thr}_fp_first"] = (np.stack([far, nw]), g[None], None, thr)
    # early end: prediction 0 lies beside both ground truths (IoU 0) with the smallest errors; its two false
    # positives end the loop (n_op + n_fp == P) although prediction 1 overlaps both
    g0 = np.array([[0, 0], [50, 100]], F64)
    g1 = g0 + [0, 5]
    p0 = g0 + [51, 0]
    p1 = np.array([[0, 100], [50, 0]], F64)
    cases["early_fp_end"] = (np.stack([p0, p1]), np.stack([g0, g1]), None, float(F32(0.05)))
    # spectral vs Frobenius: A is isotropic (spectral 2.83, Frobenius 4), B rank one (both 3.16)
    sq = np.array(_rect(0, 0, 30, 30), F64)
    A = sq + 2 * cyc
    Bp = sq + np.array([[2, 0], [2, 0], [1, 0], [1, 0]], F64)
    cases["spectral_vs_frobenius"] = (np.stack([A, Bp]), sq[None], None, float(F32(0.05)))
    return {k: (p.astype(F32), g.astype(F32), m, t) for k, (p, g, m, t) in cases.items()}


def match_reference(pred, gt, vmask, thresh):
    """eval_ref.match_2d_greedy on float64 copies: (pairs [n,2] in discovery order, pred_to_gt [P], gt_to_pred [G])."""
    P, G = len(pred), len(gt)
    vm = np.ones(gt.shape[:2], bool) if vmask is None else np.asarray(vmask, bool)
    best, _, _ = eval_ref.match_2d_greedy(pred.astype(F64), gt.astype(F64), vm, iou_thresh=thresh)
    return _assignments(best, P, G)


def _assignments(best, P, G):
    best = np.asarray(best, np.int64).reshape(-1, 2)
    p2g, g2p = np.full(P, -1, np.int64), np.full(G, -1, np.int64)
    for p, g in best:
        p2g[p], g2p[g] = g, p
    return best, p2g, g2p


def match_variant(pred, gt, vmask, thresh, mistake):
    """The greedy loop of eval_ref.match_2d_greedy with one planted mistake (MATCH_MISTAKES)."""
    P, G = len(pred), len(gt)
    pred, gt = pred.astype(F64), gt.astype(F64)
    vm = np.ones(gt.shape[:2], bool) if vmask is None else np.asarray(vmask, bool)
    err = np.full(P * G, np.inf)
    for p in range(P):
        for g in range(G):
            d = pred[p][vm[g]] - gt[g][vm[g]]
            err[p * G + g] = np.linalg.norm(d) if mistake == "frobenius" else np.linalg.norm(d, 2)
    iou = iou_matrix(pred, gt, plus1=mistake != "no_plus1").ravel()
    ga, oa = np.zeros(G, bool), np.zeros(P, bool)
    best, n_fp, fp_preds = [], 0, set()
    while ga.sum() < G and oa.sum() + n_fp < P:
        found = fpos = False
        while not found:
            if np.all(np.isinf(err)):
                return _assignments(best, P, G)
            i = (len(err) - 1 - int(np.argmin(err[::-1]))) if mistake == "tie_last" else int(np.argmin(err))
            p, g = divmod(i, G)
            err[i] = np.inf
            if not oa[p] and not ga[g] and iou[i] >= thresh:
                found = True
            elif iou[i] < thresh:
                found = fpos = True
                fp_preds.add(p)
                n_fp = len(fp_preds) if mistake == "fp_per_prediction" else n_fp + 1
        if not fpos:
            best.append((p, g))
            oa[p] = ga[g] = True
    return _assignments(best, P, G)


def pair_errors(pred, gt, vmask, dtype):
    """[P, G] np.linalg.norm(D, 2) in `dtype` (float32: the reference's arithmetic)."""
    P, G = len(pred), len(gt)
    vm = np.ones(gt.shape[:2], bool) if vmask is None else np.asarray(vmask, bool)
    e = np.zeros((P, G), F64)
    for p in range(P):
        for g in range(G):
            e[p, g] = np.linalg.norm(pred[p][vm[g]].astype(dtype) - gt[g][vm[g]].astype(dtype), 2)
    return e


# ------------------------------------------------------------------------------------------------------ points
N_SWEEP = (3, 4, 14, 17, 255, 256, 257, 6890, 10475)
GEOMETRIES = ("random", "coplanar", "collinear", "isotropic", "tpose", "mirror_x", "mirror_y", "mirror_z", "exact",
              "far", "mm")
POINT_MISTAKES = ("no_reflection", "scale_no_d", "s_one", "R_transposed", "pve_mean_centre")
FAR = np.array([50.0, -20.0, 35.0])


def applicable(geom, n):
    """Geometries whose definition needs four points (a full-rank spread) are not built at n = 3."""
    return n >= 4 or geom not in ("isotropic", "tpose", "mirror_x", "mirror_y", "mirror_z")


def _rot(rng):
    Q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    return Q if np.linalg.det(Q) > 0 else -Q


def _whiten(x, scales):
    x = x - x.mean(0)
    w, V = np.linalg.eigh(x.T @ x / len(x))
    return (x @ V / np.sqrt(w)) * np.asarray(scales)


def points_geometry(geom, n, seed):
    """Local pred x and ground-truth y [n, 3] (fp64, metres, near the origin), y ~ s R x (+ reflection) + t + noise.
    The cases place them in fp32 around their centres (or, for 'far', 50 m away and uncentred)."""
    rng = np.random.default_rng(seed)
    R, s, t = _rot(rng), rng.uniform(0.8, 1.2), rng.normal(size=3) * 0.05
    noise = 0.01
    x = rng.normal(size=(n, 3)) * [0.25, 0.5, 0.12]
    if geom == "coplanar":
        x[:, 2] = 0.0
    elif geom == "collinear":
        # exactly collinear in fp32 (dyadic steps along an integer direction, dyadic centres): a set that is collinear
        # only up to fp32 rounding has a PA decided by its 1e-8 m off-line components, ill-posed at fp32 precision
        x = np.outer(np.round(rng.normal(size=n) * 128) / 512, [1.0, 2.0, -2.0])
    elif geom == "isotropic":
        x, noise = _whiten(x, [0.3, 0.3, 0.3]), 1e-5
    elif geom == "tpose":
        x, noise = _whiten(x, [0.6, 0.6 * (1 + 1e-4), 0.08]) @ _rot(rng).T, 1e-4
    elif geom.startswith("mirror"):
        x = _whiten(x, [0.5, 0.3, 0.15]) @ _rot(rng).T
        k = "xyz".index(geom[-1])
        F = np.eye(3)
        F[k, k] = -1
        R = R @ F
    elif geom == "exact":
        x = np.round(x * 256) / 256
        perm = np.array([[0, 1, 0], [0, 0, 1], [1, 0, 0]], F64)  # a rotation, exact in fp32
        return x, 2.0 * x @ perm.T + np.round(rng.normal(size=3) * 256) / 256
    elif geom == "mm":
        x, t, noise = x * 1e-3, t * 1e-3, 1e-5
    y = s * x @ R.T + t + rng.normal(size=x.shape) * noise
    return x, y


def center_for(geom, rng):
    """A centre that keeps the geometry's promise in fp32 ('exact': dyadic) or None ('far': uncentred)."""
    if geom == "far":
        return None
    c = rng.normal(size=3) * 0.3 + [0.0, 0.2, 5.0]
    return np.round(c * 256) / 256 if geom in ("exact", "collinear") else c


def centred32(X, c):
    """What the kernel computes first: X - c as one fp32 subtraction per coordinate."""
    return X.astype(F32) if c is None else (X.astype(F32) - np.asarray(c, F32)).astype(F32)


def _ulp32(v):
    return float(np.spacing(F32(abs(v))))


def _umeyama(xc, yc):
    xm, ym = xc.mean(0), yc.mean(0)
    M = (yc - ym).T @ (xc - xm)
    Uu, D, Vt = np.linalg.svd(M)
    return xm, ym, M, Uu, D, Vt, ((xc - xm) ** 2).sum()


def points_reference(X, cx, Y, cy, mistake=None):
    """(pve, pa, tol_pve, tol_pa) in mm for one pair: fp32 inputs X, Y [n, 3], centres [3] or None."""
    xc, yc = centred32(X, cx).astype(F64), centred32(Y, cy).astype(F64)
    d = np.linalg.norm(yc - xc, axis=1)
    pve = d.mean() * 1000.0
    if mistake == "pve_mean_centre":
        xm_, ym_ = X.astype(F64) - X.astype(F64).mean(0), Y.astype(F64) - Y.astype(F64).mean(0)
        pve = np.linalg.norm(ym_ - xm_, axis=1).mean() * 1000.0
    if mistake in (None, "pve_mean_centre"):
        Rt, tt, st = roma_ref.rigid_points_registration(torch.from_numpy(xc), torch.from_numpy(yc), compute_scaling=True)
        R, t, s = Rt.numpy(), tt.numpy(), float(st)
    else:
        xm, ym, M, Uu, D, Vt, sxx = _umeyama(xc, yc)
        dd = np.sign(np.linalg.det(Uu) * np.linalg.det(Vt))
        S = np.diag([1.0, 1.0, 1.0 if mistake == "no_reflection" else dd])
        R = Uu @ S @ Vt
        s = (D @ np.diag(S)) / sxx
        if mistake == "scale_no_d":
            s = D.sum() / sxx
        elif mistake == "s_one":
            s = 1.0
        elif mistake == "R_transposed":
            R = R.T
        t = ym - s * R @ xm
    pa = np.linalg.norm(yc - (s * xc @ R.T + t), axis=1).mean() * 1000.0
    tol_pve = 1000.0 * 6 * U * d.mean() + 0.5 * _ulp32(pve)
    cmax = max(np.abs(xc).max(), np.abs(yc).max())
    tol_base = 0.5 * _ulp32(pa) + 1e-8 * pa + 1000.0 * 2.0 ** -40 * cmax
    # sigma_k = sqrt(w_k) of the Jacobi eigenvalues of M^T M: an absolute eigenvalue error of ~k eps sigma1^2 moves a
    # zero sigma_k by sqrt(k eps) sigma1 (n = 3, coplanar, collinear), a large one by k eps sigma1^2 / sigma_k.  That
    # moves s = sum(d_k sigma_k) / sxx by ds, and each aligned point by at most ds |xhat_i|
    xm = xc.mean(0)
    _, _, _, _, D, _, sxx = _umeyama(xc, yc)
    eps = 16 * 2.0 ** -53
    ds = sum(min(math.sqrt(eps) * D[0], eps * D[0] ** 2 / max(D[k], 1e-300)) for k in (1, 2)) / sxx
    dpa = 1000.0 * np.linalg.norm(xc - xm, axis=1).mean()
    tol_pa = tol_base + ds * dpa
    return pve, pa, tol_pve, tol_pa, tol_base


def cov_facts(X, cx, Y, cy):
    """(d, sigma [3]) of the centred cross-covariance M = sum yhat xhat^T of one pair (fp64 SVD)."""
    xc, yc = centred32(X, cx).astype(F64), centred32(Y, cy).astype(F64)
    _, _, _, Uu, D, Vt, _ = _umeyama(xc, yc)
    return float(np.sign(np.linalg.det(Uu) * np.linalg.det(Vt))), D


# numpy port of csrc/metrics.cu eig_sym3 / procrustes_from_cov (this repository's algorithm), line by line in fp64
def eig_sym3(A):
    with np.errstate(over="ignore"):  # theta^2 may overflow to inf, as in double on the device: t = 0
        return _eig_sym3(A)


def _eig_sym3(A):
    A = np.array(A, F64)
    V = np.eye(3)
    for _ in range(30):
        if abs(A[0, 1]) + abs(A[0, 2]) + abs(A[1, 2]) < 1e-300:
            break
        for p in range(2):
            for q in range(p + 1, 3):
                if abs(A[p, q]) < 1e-300:
                    continue
                theta = (A[q, q] - A[p, p]) / (2.0 * A[p, q])
                t = (1.0 if theta >= 0 else -1.0) / (abs(theta) + math.sqrt(theta * theta + 1.0))
                c = 1.0 / math.sqrt(t * t + 1.0)
                s = t * c
                akp, akq = A[:, p].copy(), A[:, q].copy()
                A[:, p], A[:, q] = c * akp - s * akq, s * akp + c * akq
                apk, aqk = A[p, :].copy(), A[q, :].copy()
                A[p, :], A[q, :] = c * apk - s * aqk, s * apk + c * aqk
                vkp, vkq = V[:, p].copy(), V[:, q].copy()
                V[:, p], V[:, q] = c * vkp - s * vkq, s * vkp + c * vkq
    w = np.diag(A).copy()
    for i in range(2):
        for j in range(i + 1, 3):
            if w[j] > w[i]:
                w[[i, j]] = w[[j, i]]
                V[:, [i, j]] = V[:, [j, i]]
    return V, w


def procrustes_from_cov(M, sxx, xm, ym):
    V, w = eig_sym3(M.T @ M)
    sig = np.sqrt(np.maximum(w, 0.0))
    Uu = np.zeros((3, 3))
    for k in range(2):
        u = M @ V[:, k]
        nrm = math.sqrt(u @ u)
        Uu[:, k] = u / nrm if nrm > 0 else np.eye(3)[:, k]
    d01 = Uu[:, 0] @ Uu[:, 1]
    Uu[:, 1] -= d01 * Uu[:, 0]
    n1 = math.sqrt(Uu[:, 1] @ Uu[:, 1])
    Uu[:, 1] = Uu[:, 1] / n1 if n1 > 0 else Uu[:, 1]
    Uu[:, 2] = np.cross(Uu[:, 0], Uu[:, 1])
    su = -1.0 if Uu[:, 2] @ (M @ V[:, 2]) < 0 else 1.0
    d = su * np.linalg.det(V)
    R = np.outer(Uu[:, 0], V[:, 0]) + np.outer(Uu[:, 1], V[:, 1]) + d * su * np.outer(Uu[:, 2], V[:, 2])
    s = (sig[0] + sig[1] + d * sig[2]) / sxx
    return R, ym - s * R @ xm, s


def points_port(X, cx, Y, cy):
    """PA (mm) of the numpy port of the kernel's algorithm."""
    xc, yc = centred32(X, cx).astype(F64), centred32(Y, cy).astype(F64)
    xm, ym = xc.mean(0), yc.mean(0)
    M = (yc - ym).T @ (xc - xm)
    R, t, s = procrustes_from_cov(M, ((xc - xm) ** 2).sum(), xm, ym)
    return np.linalg.norm(yc - (s * xc @ R.T + t), axis=1).mean() * 1000.0


def points_batch(geom, npt, n_pairs, seed, centres):
    """A batch of n_pairs pairs of `geom`: predictions in shuffled slots, the last pair reusing the first pair's
    ground truth (with a slightly perturbed prediction), one prediction no pair uses.  centres = (pred side given,
    ground-truth side given).  Returns pred, pc, gt, gc, pairs (fp32 numpy; centres None when absent)."""
    rng = np.random.default_rng(seed)
    n_gt = max(1, n_pairs - 1)
    P = n_pairs + 1
    pred, gt = np.zeros((P, npt, 3), F32), np.zeros((n_gt + 1, npt, 3), F32)
    pc, gc = np.zeros((P, 3), F32), np.zeros((n_gt + 1, 3), F32)
    pslot, gslot = rng.permutation(P), rng.permutation(n_gt + 1)
    pairs = []
    for m in range(n_pairs):
        k = m if m < n_gt else 0
        X, cx, Y, cy = placed_pair(geom, npt, seed=seed * 100 + k)
        if m >= n_gt:
            X = (X + rng.normal(size=X.shape) * 1e-3 * (1e-3 if geom == "mm" else 1)).astype(F32)
        p, g = pslot[m], gslot[k]
        pred[p], gt[g] = X, Y
        if cx is not None:
            pc[p], gc[g] = cx, cy
        pairs.append((p, g))
    use_pc, use_gc = centres if geom != "far" else (False, False)
    return pred, pc if use_pc else None, gt, gc if use_gc else None, np.array(pairs, np.int32).reshape(-1, 2)


def points_refs(pred, pc, gt, gc, pairs, mistake=None):
    """[n_pairs, 5] (pve, pa, tol_pve, tol_pa, PA tolerance without the rank-deficiency term) of a batch."""
    out = [points_reference(pred[p], None if pc is None else pc[p], gt[g], None if gc is None else gc[g], mistake)
           for p, g in pairs]
    return np.array(out, F64).reshape(-1, 5)


# the cases of the sensitivity test of tests/test_eval_kernels_gpu.py (the CPU test shows the premise on them)
SENSITIVITY_POINTS = [(geom, npt, 90 + i) for i, geom in enumerate(GEOMETRIES) for npt in (14, 257)]


def placed_pair(geom, n, seed):
    """(X fp32, cx, Y fp32, cy) of one pair: the geometry placed around its centres (centres as fp32 or None)."""
    rng = np.random.default_rng(seed + 77)
    x, y = points_geometry(geom, n, seed)
    cx, cy = center_for(geom, rng), center_for(geom, rng)
    if geom == "far":
        return (x + FAR).astype(F32), None, (y + FAR).astype(F32), None
    return (x + cx).astype(F32), cx.astype(F32), (y + cy).astype(F32), cy.astype(F32)


# ------------------------------------------------------------------------------------------------------ regression
NNZ_EDGES = (0, 1, 31, 32, 33, 200)
R_OUT_SWEEP = (1, 7, 8, 9, 14, 17)
REG_MISTAKES = ("before_centring", "no_root", "other_K")
# row lists of the projection and root cases of tests/test_eval_kernels_gpu.py (repeated rows included)
PROJ_ROWS = [0, 4, 4, 8, 2, 1, 7, 3, 5]
ROOT_ROWS = [2, 3, 5, 11]


def make_csr(nnz, N, seed, positive=False):
    """Dense fp32 A [len(nnz), N] with the given non-zeros per row (mixed-sign weights unless `positive`, then rows
    summing to 1) and its CSR (rowptr, col, val) as int32 / fp32 numpy."""
    rng = np.random.default_rng(seed)
    A = np.zeros((len(nnz), N), F32)
    for r, k in enumerate(nnz):
        cols = np.sort(rng.choice(N, size=k, replace=False))
        w = rng.uniform(0.05, 1.0, size=k) if positive else rng.normal(size=k)
        if positive and k:
            w = w / w.sum()
        A[r, cols] = w
    rowptr = np.concatenate([[0], np.cumsum([int((A[r] != 0).sum()) for r in range(len(nnz))])]).astype(np.int32)
    col = np.concatenate([np.nonzero(A[r])[0] for r in range(len(nnz))]).astype(np.int32)
    val = np.concatenate([A[r][A[r] != 0] for r in range(len(nnz))]).astype(F32)
    return A, rowptr, col, val


def regress_reference(A, rowptr, X, c, rows, root, mistake=None):
    """(y [R_out, 3] fp64, tol [R_out, 3]) for one source mesh X [N, 3] fp32, centre c [3] fp32 or None.
    A: fp64-able dense [R, N] (numpy or torch)."""
    A = torch.as_tensor(A).double()
    Xd = torch.as_tensor(X).double()
    cd = torch.zeros(3, dtype=torch.float64) if c is None else torch.as_tensor(np.asarray(c, F64))
    xc = Xd - cd
    y = A @ (Xd if mistake == "before_centring" else xc)
    if mistake == "before_centring":
        y = y - cd
    mag = A.abs() @ xc.abs()
    nnz = torch.as_tensor(np.diff(np.asarray(rowptr)), dtype=torch.float64)
    b = (torch.ceil(nnz / 32) + 6)[:, None] * U * mag
    rows = list(range(A.shape[0])) if rows is None else list(rows)
    out, tol = y[rows], b[rows]
    if root >= 0 and mistake != "no_root":
        out = out - y[root]
        tol = tol + b[root]
    return out, tol + U * out.abs()


def reg_inputs(N, seed):
    """Five source meshes X [5, N, 3] (z ~ 6 m), centres [5, 3] (z ~ 0.5 m, so that X - c stays in front of the
    camera), distinct intrinsics K [5, 3, 3] and four pairs (fp32 / int32 numpy)."""
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(5, N, 3)) * 0.3 + [0.3, -0.2, 6.0]).astype(F32)
    c = (rng.normal(size=(5, 3)) * 0.2 + [0.0, 0.0, 0.5]).astype(F32)
    K = np.stack([[[400 + 10 * i, 0, 200 + i], [0, 380 - 5 * i, 210], [0, 0, 1]] for i in range(5)]).astype(F32)
    pairs = np.array([[3, 1], [0, 4], [2, 2], [4, 1]], np.int32)
    return X, c, K, pairs


def project_reference(y, tol, K):
    """(q [R_out, 2], tol) of (K . (y / y_z))[:2] in fp64 for fp32 y within `tol` of the fp64 y."""
    K = torch.as_tensor(K).double().reshape(3, 3)
    z, tz = y[:, 2:3], tol[:, 2:3]
    q = y / z
    eq = (tol + q.abs() * tz) / (z.abs() - tz) + U * q.abs()
    eq[:, 2] = 0.0  # y_z / y_z is exactly 1
    out = q @ K.t()
    etol = eq @ K.abs().t() + 4 * U * (q.abs() @ K.abs().t())
    return out[:, :2], etol[:, :2]
