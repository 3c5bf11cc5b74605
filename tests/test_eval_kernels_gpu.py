"""The evaluation kernels (csrc/metrics.cu) against the fp64 oracles of eval_kernels_util, through the C-ABI entries
`mhmr_eval_match_2d`, `mhmr_eval_points_error` and `mhmr_eval_regress`, at their person, point, lane, warp and
degenerate-geometry edges.

  * Matching: P x G over {0, 1, 2, 31, 32, 33, 47, 48} x {1, ..., 48}, J not a multiple of the 32 lanes, with and
    without a valid mask (one that drops a whole lane-stride slice included); pairs in discovery order, n_pairs,
    pred_to_gt and gt_to_pred equal the oracle's exactly.  Dedicated cases: exact ties (row-major first wins), IoU
    exactly at a dyadic threshold next to a box one pixel narrower, the reference's early end on false positives.
  * Points error: n around the 256 threads of a CTA and at the mesh sizes, up to 48 pair slots, pairs out of order
    with a repeated ground truth, centres given or absent on each side, every geometry of the util; PVE and PA within
    their bounds; a pair's values do not depend on its slot or its neighbours, and repeated calls are bitwise equal.
  * Regression: rows with 0, 1, 31, 32, 33 and 200 non-zeros and negative weights, R_out around the 8 warps of a CTA
    with repeated rows, root in {-1, 0, R - 1}, both sides, with and without centre and projection, and the
    real-shape SMPL-X -> SMPL and H36M matrices.
Every output lands in a canvas with sentinel guard bands: slots from n_pairs up to max_pairs and anything past P or G
must come back untouched.  n_pairs is written on the device right before each call.  Each planted mistake of the
util falls outside its bound on at least one case here."""
import numpy as np
import pytest
import torch

import eval_kernels_util as ek
from fp64_util import SENTINEL, _report

pytestmark = pytest.mark.gpu
GUARD = 32
ISENT = -777


def _canvas(n, dev, dtype=torch.float32):
    fill = SENTINEL if dtype == torch.float32 else ISENT
    buf = torch.full((2 * GUARD + n,), fill, device=dev, dtype=dtype)
    return buf, buf[GUARD:GUARD + n]


def _untouched(buf, used, what):
    fill = SENTINEL if buf.dtype == torch.float32 else ISENT
    assert (buf[:GUARD] == fill).all(), f"{what}: write before the first slot"
    assert (buf[GUARD + used:] == fill).all(), f"{what}: write past the {used} slots in use"


def _n_pairs(n, dev):
    t = torch.zeros(1, dtype=torch.int32, device=dev)
    t.fill_(n)  # on the device, no host read before the call
    return t


# ------------------------------------------------------------------------------------------------------ matching
def run_match(pred, gt, vmask, thr, dev):
    from multihmr_b200._lib import call, stream

    P, G, J = len(pred), len(gt), gt.shape[1]
    pr = torch.from_numpy(pred).to(dev).contiguous() if P else None
    g = torch.from_numpy(gt).to(dev).contiguous()
    vm = None if vmask is None else torch.from_numpy(vmask.astype(np.uint8)).to(dev).contiguous()
    pairs, pv = _canvas(2 * 48, dev, torch.int32)
    nb, nv = _canvas(1, dev, torch.int32)
    p2g, p2gv = _canvas(48, dev, torch.int32)
    g2p, g2pv = _canvas(48, dev, torch.int32)
    call("mhmr_eval_match_2d", pr, g, vm, P, G, J, thr, pv, nv, p2gv, g2pv, stream())
    torch.cuda.synchronize()
    n = int(nv.item())
    _untouched(nb, 1, "n_pairs")
    _untouched(pairs, 2 * n, "pairs")
    _untouched(p2g, P, "pred_to_gt")
    _untouched(g2p, G, "gt_to_pred")
    return (pv[:2 * n].view(n, 2).cpu().numpy().astype(np.int64), p2gv[:P].cpu().numpy().astype(np.int64),
            g2pv[:G].cpu().numpy().astype(np.int64))


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("P", ek.PG_SWEEP)
def test_match_sweep_vs_oracle(P, cuda_device):
    cases = [(P, G, J, m) for (p, G, J, m) in ek.MATCH_CASES if p == P]
    if P == 48:  # every J, with and without a mask, at the full 48 x 48
        cases += [(48, 48, J, m) for J in ek.J_SWEEP for m in (False, True)]
    n_fp = 0
    for (P_, G, J, masked) in cases:
        pred, gt, vm, thr = ek.match_case(P_, G, J, masked, seed=P_ * 64 + G + 4096 * J)
        got = run_match(pred, gt, vm, thr, cuda_device)
        ref = ek.match_reference(pred, gt, vm, thr)
        assert _same(got, ref), (P_, G, J, masked, got[0].tolist(), ref[0].tolist())
        n_fp += P_ - len(ref[0])
    print(f"matching P={P}: {len(cases)} cases equal to the oracle ({n_fp} false positives in all)")


def test_match_dedicated_cases(cuda_device):
    cases = ek.dedicated_match_cases()
    for name, c in cases.items():
        got = run_match(*c, cuda_device)
        assert _same(got, ek.match_reference(*c)), name
    assert run_match(*cases["ties"], cuda_device)[0].tolist() == [[1, 0], [2, 1]]
    for k in ("iou_edge_0.5", "iou_edge_0.25", "iou_edge_0.5_fp_first", "iou_edge_0.25_fp_first"):
        assert run_match(*cases[k], cuda_device)[0].tolist() == [[0, 0]], k
    assert run_match(*cases["early_fp_end"], cuda_device)[0].size == 0


def test_match_sensitivity(cuda_device):
    cases = ek.dedicated_match_cases()
    sweep = [ek.match_case(P, G, J, m, seed=P * 64 + G + 4096 * J) for (P, G, J, m) in
             [(48, 48, 17, False), (33, 31, 127, True), (2, 2, 14, False)]]
    for mistake in ek.MATCH_MISTAKES:
        hits = [k for k, c in list(cases.items()) + [(f"sweep{i}", c) for i, c in enumerate(sweep)]
                if not _same(run_match(*c, cuda_device), ek.match_variant(*c, mistake))]
        print(f"matching mistake {mistake}: the kernel differs from it on {hits}")
        assert hits, mistake


# ------------------------------------------------------------------------------------------------------ points
def run_points(pred, pc, gt, gc, pairs, n, max_pairs, dev):
    """pred [P, npt, 3], gt [G, npt, 3], centres [*, 3] or None (numpy fp32); pairs [n, 2]."""
    from multihmr_b200._lib import call, stream

    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
    pr, pcd, g, gcd = t(pred), t(pc), t(gt), t(gc)
    slots = np.zeros((max_pairs, 2), np.int32)  # unused slots hold valid indices: only the count may exclude them
    slots[:len(pairs)] = pairs
    pd = torch.from_numpy(slots).to(dev)
    err, ev = _canvas(max_pairs, dev)
    pa, pav = _canvas(max_pairs, dev)
    nd = _n_pairs(n, dev)  # referenced until the kernel has run
    call("mhmr_eval_points_error", pr, pcd, g, gcd, pd, nd, max_pairs, pred.shape[1], ev, pav, stream())
    torch.cuda.synchronize()
    _untouched(err, n, "err_mm")
    _untouched(pa, n, "pa_err_mm")
    return ev[:n].double().cpu().numpy(), pav[:n].double().cpu().numpy()


CENTRES = ((True, True), (False, True), (True, False), (False, False))
MAXP = (1, 7, 48)
RANK_DEFICIENT = ("coplanar", "collinear")


@pytest.mark.parametrize("geom", ek.GEOMETRIES)
def test_points_error_vs_fp64(geom, cuda_device):
    errs, tols, bases = [], [], []
    for i, npt in enumerate(ek.N_SWEEP):
        if not ek.applicable(geom, npt):
            continue
        max_pairs = MAXP[i % 3]
        n_pairs = {1: 1, 7: 5, 48: 45 if npt <= 257 else 9}[max_pairs]
        pred, pc, gt, gc, pairs = ek.points_batch(geom, npt, n_pairs, seed=i + 31 * len(geom), centres=CENTRES[i % 4])
        e, pa = run_points(pred, pc, gt, gc, pairs, n_pairs, max_pairs, cuda_device)
        ref = ek.points_refs(pred, pc, gt, gc, pairs)
        r_pve, r_pa = np.abs(e - ref[:, 0]) / ref[:, 2], np.abs(pa - ref[:, 1]) / ref[:, 3]
        assert (r_pve <= 1).all() and (r_pa <= 1).all(), (geom, npt, r_pve.max(), r_pa.max(), e, ref[:, 0], pa, ref[:, 1])
        errs.append(np.stack([np.abs(e - ref[:, 0]), np.abs(pa - ref[:, 1])], 1))
        tols.append(ref[:, 2:4])
        bases.append(ref[:, 4])
    err, tol = torch.from_numpy(np.concatenate(errs)), torch.from_numpy(np.concatenate(tols))
    _report(f"{geom} PVE", err[:, 0], tol[:, 0])
    _report(f"{geom} PA ", err[:, 1], tol[:, 1])
    # the same errors against the PA bound without the rank-deficiency term (information: where the term matters)
    _report(f"{geom} PA (without the rank-deficiency term)", err[:, 1], torch.from_numpy(np.concatenate(bases)))


def test_points_error_slot_independence_and_repeat(cuda_device):
    for geom, npt in (("random", 257), ("mirror_y", 14), ("collinear", 3)):
        pred, pc, gt, gc, pairs = ek.points_batch(geom, npt, 7, seed=5, centres=(True, True))
        a = run_points(pred, pc, gt, gc, pairs, 7, 48, cuda_device)
        b = run_points(pred, pc, gt, gc, pairs, 7, 48, cuda_device)
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), f"{geom}: repeated call"
        rev = pairs[::-1].copy()
        c = run_points(pred, pc, gt, gc, rev, 7, 7, cuda_device)
        assert all(np.array_equal(x, y[::-1]) for x, y in zip(a, c)), f"{geom}: slots reversed"
        for m in range(7):
            one = run_points(pred, pc, gt, gc, pairs[m:m + 1], 1, 1, cuda_device)
            assert all(np.array_equal(x[m:m + 1], y) for x, y in zip(a, one)), f"{geom}: pair {m} alone"
    # n_pairs = 0: nothing is written, in a single-slot grid and in a wider one
    run_points(pred, pc, gt, gc, pairs[:0], 0, 1, cuda_device)
    run_points(pred, pc, gt, gc, pairs[:0], 0, 7, cuda_device)


def test_points_error_sensitivity(cuda_device):
    worst = {k: 0.0 for k in ek.POINT_MISTAKES}
    for geom, npt, seed in ek.SENSITIVITY_POINTS:
        pred, pc, gt, gc, pairs = ek.points_batch(geom, npt, 3, seed=seed, centres=(True, True))
        e, pa = run_points(pred, pc, gt, gc, pairs, 3, 7, cuda_device)
        ref = ek.points_refs(pred, pc, gt, gc, pairs)
        for mistake in ek.POINT_MISTAKES:
            w = ek.points_refs(pred, pc, gt, gc, pairs, mistake)
            r = max((np.abs(e - w[:, 0]) / ref[:, 2]).max(), (np.abs(pa - w[:, 1]) / ref[:, 3]).max())
            worst[mistake] = max(worst[mistake], r)
    for k, r in worst.items():
        print(f"points mistake {k}: misses its bound by {r:.3g}x")
        assert r > 1.0, k


# ------------------------------------------------------------------------------------------------------ regression
def run_regress(rowptr, col, val, R, N, rows, root, X, c, pairs, side, n, max_pairs, K, dev):
    from multihmr_b200._lib import call, stream

    t = lambda a, dt=np.float32: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    R_out = R if rows is None else len(rows)
    slots = np.zeros((max_pairs, 2), np.int32)
    slots[:len(pairs)] = pairs
    out, ov = _canvas(max_pairs * R_out * 3, dev)
    o2, o2v = _canvas(max_pairs * R_out * 2, dev) if K is not None else (None, None)
    rp, cl = (rowptr, col) if torch.is_tensor(rowptr) else (t(rowptr, np.int32), t(col, np.int32))
    vl = val if torch.is_tensor(val) else t(val)
    Xd = X if torch.is_tensor(X) else t(X)
    # every input stays referenced until the kernel has run (a freed temporary's block goes to the next one)
    rw, cd, pd, nd = t(rows, np.int32), t(c), t(slots, np.int32), _n_pairs(n, dev)
    Kd = None if K is None else t(K.reshape(-1, 9))
    call("mhmr_eval_regress", rp, cl, vl, R, N, rw, R_out, root, Xd, cd, pd, side, nd, max_pairs, Kd, ov, o2v, stream())
    torch.cuda.synchronize()
    _untouched(out, n * R_out * 3, "out")
    y = ov[:n * R_out * 3].view(n, R_out, 3).double().cpu()
    if K is None:
        return y, None
    _untouched(o2, n * R_out * 2, "out2d")
    return y, o2v[:n * R_out * 2].view(n, R_out, 2).double().cpu()


def _check_projection(q, y_ref, tol, K):
    """out2d against the fp64 projection on the rows whose depth is known well (|y_z| > 1000 tol_z; a row of zeros
    has no projection); returns (worst err/tol, rows checked)."""
    ok = y_ref[:, 2].abs() > 1000 * tol[:, 2]
    if not ok.any():
        return 0.0, 0
    qr, qt = ek.project_reference(y_ref[ok], tol[ok], K)
    d = (q[ok] - qr).abs()
    assert (d <= qt).all(), (d / qt).max().item()
    return (d / qt).max().item(), int(ok.sum())


def test_regression_sweep_vs_fp64(cuda_device):
    N = 700
    nnz = list(ek.NNZ_EDGES) * 3  # R = 18 rows
    A, rowptr, col, val = ek.make_csr(nnz, N, seed=11)
    R = len(nnz)
    X, c, K, pairs = ek.reg_inputs(N, 12)
    rng = np.random.default_rng(13)
    worst, worst2, count, count2 = 0.0, 0.0, 0, 0
    for R_out in ek.R_OUT_SWEEP + (None,):
        rows = None if R_out is None else rng.integers(R, size=R_out).tolist()
        if R_out is not None and R_out > 1:
            rows[-1] = rows[0]  # a repeated row
        for root in (-1, 0, R - 1):
            for side in (0, 1):
                for centred in (False, True):
                    for proj in (False, True):
                        cc = c if centred else None
                        y, q = run_regress(rowptr, col, val, R, N, rows, root, X, cc, pairs, side, 3, 6,
                                           K if proj else None, cuda_device)
                        for m in range(3):
                            s = pairs[m, side]
                            ref, tol = ek.regress_reference(A, rowptr, X[s], None if cc is None else cc[s], rows, root)
                            d = (y[m] - ref).abs()
                            assert (d <= tol).all(), (R_out, root, side, centred, m, (d - tol).max().item())
                            worst = max(worst, (d / tol.clamp_min(1e-300)).max().item())  # 0 non-zeros: d = 0
                            count += 1
                            if proj:
                                r2, k2 = _check_projection(q[m], ref, tol, K[s])
                                worst2, count2 = max(worst2, r2), count2 + k2
    print(f"regression sweep: {count} pair outputs, worst err/tol {worst:.3f}; projection of {count2} rows, "
          f"worst err/tol {worst2:.3f}")
    assert count2 > 500


def test_regression_projection_and_sensitivity(cuda_device):
    N = 700
    nnz = [1, 31, 32, 33, 200, 3, 48, 7, 9]
    A, rowptr, col, val = ek.make_csr(nnz, N, seed=21, positive=True)
    R = len(nnz)
    X, c, K, pairs = ek.reg_inputs(N, 22)
    Am, rpm, clm, vlm = ek.make_csr(list(ek.NNZ_EDGES) * 2, N, seed=23)
    wrong = {k: 0.0 for k in ek.REG_MISTAKES}
    worst2 = 0.0
    for side in (0, 1):
        y, q = run_regress(rowptr, col, val, R, N, ek.PROJ_ROWS, -1, X, c, pairs, side, 4, 5, K, cuda_device)
        for m in range(4):
            s, o = pairs[m, side], pairs[m, 1 - side]
            ref, tol = ek.regress_reference(A, rowptr, X[s], c[s], ek.PROJ_ROWS, -1)
            assert ((y[m] - ref).abs() <= tol).all()
            qr, qt = ek.project_reference(ref, tol, K[s])
            worst2 = max(worst2, ((q[m] - qr).abs() / qt).max().item())
            assert ((q[m] - qr).abs() <= qt).all(), (side, m)
            qo, _ = ek.project_reference(ref, tol, K[o])
            wrong["other_K"] = max(wrong["other_K"], ((q[m] - qo).abs() / qt).max().item())
        # mixed-sign rows with a root: centring and root subtraction
        y, _ = run_regress(rpm, clm, vlm, Am.shape[0], N, ek.ROOT_ROWS, 4, X, c, pairs, side, 4, 4, None,
                           cuda_device)
        for m in range(4):
            s = pairs[m, side]
            ref, tol = ek.regress_reference(Am, rpm, X[s], c[s], ek.ROOT_ROWS, 4)
            assert ((y[m] - ref).abs() <= tol).all()
            for mistake in ("before_centring", "no_root"):
                w, _ = ek.regress_reference(Am, rpm, X[s], c[s], ek.ROOT_ROWS, 4, mistake)
                wrong[mistake] = max(wrong[mistake], ((y[m] - w).abs() / tol.clamp_min(1e-300)).max().item())
    print(f"regression projection: worst err/tol {worst2:.3f}")
    for k, r in wrong.items():
        print(f"regression mistake {k}: misses its bound by {r:.3g}x")
        assert r > 1.0, k


def test_regression_real_shapes(cuda_device):
    from multihmr_b200 import metrics
    from oracle import eval_bench_ref

    assets = eval_bench_ref.eval_assets(0)
    rng = np.random.default_rng(31)
    for name, A, rows, root, N in (("smplx2smpl", assets["smplx2smpl"], None, -1, 10475),
                                   ("J_regressor_h36m", assets["j_regressor_h36m"], metrics.H36M_TO_J14, 0, 6890)):
        csr = metrics.CSR(A, cuda_device)
        R = csr.shape[0]
        X = (rng.normal(size=(3, N, 3)) * 0.4 + [0.0, 0.3, 6.0]).astype(np.float32)
        c = X[:, 100].copy()
        pairs = np.array([[2, 0], [0, 1]], np.int32)
        Xd = torch.from_numpy(X).to(cuda_device)
        y, _ = run_regress(csr.rowptr, csr.col, csr.val, R, N, rows, root, Xd, c, pairs, 0, 2, 3, None, cuda_device)
        rowptr = csr.rowptr.cpu().numpy()
        worst = 0.0
        for m in range(2):
            s = pairs[m, 0]
            ref, tol = ek.regress_reference(A, rowptr, X[s], c[s], rows, root)
            assert ((y[m] - ref).abs() <= tol).all(), name
            worst = max(worst, ((y[m] - ref).abs() / tol.clamp_min(1e-300)).max().item())
        print(f"regression {name} [{R}, {N}]: worst err/tol {worst:.3f}")


# ------------------------------------------------------------------------------------------------------ Evaluator
def _composition_images(kind, seed, n_images=10):
    """n_images synthetic images for metrics.Evaluator: 2-D joints from the matching builder at the reference's IoU
    threshold 0.05, predicted SMPL-X meshes (10475 vertices) and ground-truth meshes of `kind` ('smplx': 10475,
    'smpl': 6890), pelvis near vertex 0.  P and G are drawn from {0..48} x {1..48}, the extremes included."""
    rng = np.random.default_rng(seed)
    Vg = 10475 if kind == "smplx" else 6890
    shape = [0.25, 0.5, 0.12]
    base_p, base_g = rng.normal(size=(10475, 3)) * shape, rng.normal(size=(Vg, 3)) * shape
    edges = [(0, 5), (48, 48), (48, 1), (1, 48)]
    out = []
    for i in range(n_images):
        P, G = edges[i] if i < len(edges) else (int(rng.integers(0, 49)), int(rng.integers(1, 49)))
        pj, gj, _, _ = ek.match_case(P, G, 17, False, seed=seed * 100 + i, fixed_thresh=True)
        mesh = lambda base, k: (base[None] * rng.uniform(0.9, 1.1, size=(k, 1, 1)) + rng.normal(size=(k, 1, 3))
                                + [0.0, 0.0, 6.0] + rng.normal(size=(k,) + base.shape) * 0.01).astype(np.float32)
        pv, gv = mesh(base_p, P), mesh(base_g, G)
        pp = (pv[:, :1] + rng.normal(size=(P, 1, 3)) * 0.01).astype(np.float32)
        gp = (gv[:, :1] + rng.normal(size=(G, 1, 3)) * 0.01).astype(np.float32)
        out.append(dict(pj=pj, pv=pv, pp=pp, gj=gj, gv=gv, gp=gp))
    return out


def _dev(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _stage_check(got, ref, tol, what):
    assert ((got - ref).abs() <= tol).all(), f"{what}: {((got - ref).abs() / tol.clamp_min(1e-300)).max().item()}"


def _evaluator_reference(kind, imgs, T, Jr, dev, shift=False):
    """fp64 restatement of Trainer.evaluate's loop over `imgs`: matching by eval_ref, then per matched pair the
    kernel-level oracles.  On the SMPL path each regression stage (the transfer of the centred prediction, the H36M
    joints of both sides) is run on the device once, checked against its fp64 bound, and its fp32 output is the
    input of the next stage's oracle, so every per-pair value has the bound of its own last stage.  `shift` takes
    pair m's prediction-side rows from pair m + 1 (the index plumbing mistake the test must see).
    Returns count, miss, fp, {meter: [(value, tol)]}, [pairs per image]."""
    from multihmr_b200 import metrics

    count = miss = fp = 0
    vals = {k: [] for k in ("pve", "pa_pve", "mpjpe", "pa_mpjpe")}
    all_pairs = []
    for im in imgs:
        P, G = len(im["pj"]), len(im["gj"])
        best, _, _ = ek.match_reference(im["pj"], im["gj"], None, float(np.float32(0.05)))
        n = len(best)
        count, miss, fp = count + G, miss + G - n, fp + P - n
        all_pairs.append(best)
        if n == 0:
            continue
        sh = (np.arange(n) + (1 if shift else 0)) % n
        if kind == "smplx":
            for m in range(n):
                p, g = best[sh[m], 0], best[m, 1]
                pve, pa, tp, ta, _ = ek.points_reference(im["pv"][p], im["pp"][p, 0], im["gv"][g], im["gp"][g, 0])
                vals["pve"].append((pve, tp))
                vals["pa_pve"].append((pa, ta))
            continue
        pr = best.astype(np.int32)
        # stage 1: the SMPL-X -> SMPL transfer of the centred predictions, pair m in row m
        ys, _ = run_regress(T.rowptr, T.col, T.val, 6890, 10475, None, -1, _dev(im["pv"], dev),
                            im["pp"][:, 0], pr, 0, n, n, None, dev)
        rp_T = T.rowptr.cpu().numpy()
        for m in range(n):
            ref, tol = ek.regress_reference(T.A, rp_T, im["pv"][pr[m, 0]], im["pp"][pr[m, 0], 0], None, -1)
            _stage_check(ys[m], ref, tol, f"transfer of pair {m}")
        ys32 = ys.float().numpy()
        # stage 2: H36M joints (J14, root-centred) of the transferred predictions and of the ground truths
        same = np.stack([np.arange(n), np.arange(n)], 1).astype(np.int32)
        hh, _ = run_regress(Jr.rowptr, Jr.col, Jr.val, 17, 6890, metrics.H36M_TO_J14, 0, _dev(ys32, dev), None, same,
                            0, n, n, None, dev)
        hg, _ = run_regress(Jr.rowptr, Jr.col, Jr.val, 17, 6890, metrics.H36M_TO_J14, 0, _dev(im["gv"], dev),
                            im["gp"][:, 0], pr, 1, n, n, None, dev)
        rp_J = Jr.rowptr.cpu().numpy()
        for m in range(n):
            ref, tol = ek.regress_reference(Jr.A, rp_J, ys32[m], None, metrics.H36M_TO_J14, 0)
            _stage_check(hh[m], ref, tol, f"H36M of transferred pair {m}")
            g = pr[m, 1]
            ref, tol = ek.regress_reference(Jr.A, rp_J, im["gv"][g], im["gp"][g, 0], metrics.H36M_TO_J14, 0)
            _stage_check(hg[m], ref, tol, f"H36M of ground truth {g}")
        hh32, hg32 = hh.float().numpy(), hg.float().numpy()
        for m in range(n):
            g = pr[m, 1]
            pve, pa, tp, ta, _ = ek.points_reference(ys32[sh[m]], None, im["gv"][g], im["gp"][g, 0])
            vals["pve"].append((pve, tp))
            vals["pa_pve"].append((pa, ta))
            e, pe, te, tpe, _ = ek.points_reference(hh32[sh[m]], None, hg32[m], None)
            vals["mpjpe"].append((e, te))
            vals["pa_mpjpe"].append((pe, tpe))
    return count, miss, fp, vals, all_pairs


@pytest.mark.parametrize("kind", ["smplx", "smpl"])
def test_evaluator_composition_vs_fp64(kind, cuda_device):
    """Ten images per ground-truth kind (twenty in all) through metrics.Evaluator against the fp64 restatement of the
    loop: counts, matched pairs and precision / recall / F1 exact, every per-pair value within its bound, each meter
    the mean of its values; the restatement with the prediction-side pair rows shifted by one misses."""
    from multihmr_b200 import metrics
    from oracle import eval_bench_ref

    assets = eval_bench_ref.eval_assets(0)
    T, Jr = metrics.CSR(assets["smplx2smpl"], cuda_device), metrics.CSR(assets["j_regressor_h36m"], cuda_device)
    T.A, Jr.A = assets["smplx2smpl"], assets["j_regressor_h36m"]
    imgs = _composition_images(kind, seed=41 if kind == "smplx" else 42)
    ev = metrics.Evaluator(smplx2smpl=T if kind == "smpl" else None,
                           j_regressor_h36m=Jr if kind == "smpl" else None, device=cuda_device)
    got_pairs = []
    for im in imgs:
        persons = [dict(j2d=_dev(im["pj"][p], cuda_device), v3d=_dev(im["pv"][p], cuda_device),
                        transl_pelvis=_dev(im["pp"][p], cuda_device)) for p in range(len(im["pj"]))]
        gt = dict(j2d=_dev(im["gj"], cuda_device), v3d=_dev(im["gv"], cuda_device),
                  transl_pelvis=_dev(im["gp"], cuda_device))
        got_pairs.append(ev.update(persons, gt).cpu().numpy().astype(np.int64))
    count, miss, fp, vals, ref_pairs = _evaluator_reference(kind, imgs, T, Jr, cuda_device)
    assert (ev.count, ev.miss, ev.fp) == (count, miss, fp)
    assert all(np.array_equal(a, b) for a, b in zip(got_pairs, ref_pairs))
    s = ev.summary()
    prf = ek.eval_ref.compute_prf1(count, miss, fp)
    assert (s["precision"], s["recall"], s["f1_score"]) == tuple(prf)
    keys = ("pve", "pa_pve") + (("mpjpe", "pa_mpjpe") if kind == "smpl" else ())
    n_pairs = sum(len(p) for p in ref_pairs)
    for k in keys:
        got = np.asarray(ev.values[k], np.float64)
        ref = np.asarray(vals[k], np.float64).reshape(-1, 2)
        assert got.shape == (n_pairs,) and ref.shape[0] == n_pairs, k
        r = np.abs(got - ref[:, 0]) / ref[:, 1]
        assert (r <= 1).all(), (k, r.max())
        assert s[k] == ev.meters[k].avg and abs(s[k] - got.mean()) <= 1e-9 * abs(got.mean()), k
        print(f"Evaluator {kind} {k}: {n_pairs} pairs over {len(imgs)} images, worst err/tol {r.max():.3f}")
    # the index plumbing: with the prediction-side rows shifted by one the values miss their bounds
    _, _, _, wrong, _ = _evaluator_reference(kind, imgs, T, Jr, cuda_device, shift=True)
    for k in keys:
        got = np.asarray(ev.values[k], np.float64)
        w = np.asarray(wrong[k], np.float64).reshape(-1, 2)
        r = (np.abs(got - w[:, 0]) / np.asarray(vals[k], np.float64).reshape(-1, 2)[:, 1]).max()
        print(f"Evaluator {kind} {k} with shifted pair rows: misses by {r:.3g}x")
        assert r > 1.0, k
