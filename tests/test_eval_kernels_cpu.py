"""The premises of tests/test_eval_kernels_gpu.py, without a GPU: the case builders of eval_kernels_util keep their
promises (error separation in fp32 and fp64, exact IoUs at the threshold edges, the designed d sign and sigma gaps), a
numpy port of the kernel's eig_sym3 / procrustes_from_cov agrees with roma_ref within the PA bound on every geometry
(the bound is achievable by the algorithm), and each planted mistake moves the fp64 oracle outside its bound on the
cases the GPU test uses."""
import numpy as np
import pytest

import eval_kernels_util as ek



def _separated(e):
    """Consecutive distinct errors >= MIN_SEP apart (relative); equal ones only as exact ties."""
    v = np.sort(e.ravel())
    if v.size < 2:
        return True
    d = np.diff(v)
    return bool(((d == 0) | (d >= ek.MIN_SEP * v[1:])).all())


@pytest.mark.parametrize("P,G,J,masked", [c for c in ek.MATCH_CASES if c[0] in (0, 1, 33, 48) or c[1] in (2, 48)]
                         + [(48, 48, J, m) for J in ek.J_SWEEP for m in (False, True)])
def test_match_builder_promises(P, G, J, masked):
    # the seeds of tests/test_eval_kernels_gpu.py
    pred, gt, vm, thr = ek.match_case(P, G, J, masked, seed=P * 64 + G + 4096 * J)
    assert pred.dtype == np.float32 and np.array_equal(pred, np.round(pred)) and np.array_equal(gt, np.round(gt))
    # boxes at least 1 px in each direction, as the reference asserts
    for a in (pred, gt):
        if len(a):
            assert ((a.max(1) - a.min(1)) >= 1).all()
    iou = ek.iou_matrix(pred, gt)
    assert iou.size == 0 or np.abs(iou - thr).min() >= ek.IOU_MARGIN
    if P:
        e64, e32 = ek.pair_errors(pred, gt, vm, np.float64), ek.pair_errors(pred, gt, vm, np.float32)
        assert _separated(e64) and _separated(e32)
        # the reference's fp32 norm orders the pairs exactly as the fp64 one
        assert np.array_equal(np.argsort(e64.ravel(), kind="stable"), np.argsort(e32.ravel(), kind="stable"))
    if masked:
        assert (~vm).any(axis=1).all()
        # one whole lane-stride slice j = l (mod 32) is dropped for every ground truth
        assert any((~vm[:, l::32]).all() for l in range(min(J, 32)))


def test_dedicated_match_cases():
    cases = ek.dedicated_match_cases()
    for name, (pred, gt, vm, thr) in cases.items():
        e64, e32 = ek.pair_errors(pred, gt, vm, np.float64), ek.pair_errors(pred, gt, vm, np.float32)
        assert np.array_equal(np.argsort(e64.ravel(), kind="stable"), np.argsort(e32.ravel(), kind="stable")), name
        iou = ek.iou_matrix(pred, gt)
        if name.startswith("iou_edge"):
            # exact in fp32: integer areas, dyadic quotient
            assert iou[0, 0] == thr and np.float32(iou[0, 0]) == np.float32(thr) and iou[1, 0] < thr, name
        else:
            assert np.abs(iou - thr).min() >= ek.IOU_MARGIN, name
    best, p2g, _ = ek.match_reference(*cases["ties"])
    assert best.tolist() == [[1, 0], [2, 1]]
    for k in ("iou_edge_0.5", "iou_edge_0.25", "iou_edge_0.5_fp_first", "iou_edge_0.25_fp_first"):
        best, p2g, _ = ek.match_reference(*cases[k])
        assert best.tolist() == [[0, 0]] and p2g[1] == -1, k
    e = ek.pair_errors(*cases["iou_edge_0.5_fp_first"][:3], np.float64)
    assert e[1, 0] < e[0, 0]  # the narrower box is popped (and counted) first
    best, _, _ = ek.match_reference(*cases["early_fp_end"])
    assert best.size == 0  # the loop ends on two false positives of prediction 0
    assert ek.match_reference(*cases["spectral_vs_frobenius"])[0].tolist() == [[0, 0]]


def test_match_mistakes_move_the_oracle():
    cases = ek.dedicated_match_cases()
    where = {"frobenius": "spectral_vs_frobenius", "no_plus1": "iou_edge_0.5", "tie_last": "ties",
             "fp_per_prediction": "early_fp_end"}
    for mistake in ek.MATCH_MISTAKES:
        c = cases[where[mistake]]
        ref, wrong = ek.match_reference(*c), ek.match_variant(*c, mistake)
        assert not all(np.array_equal(a, b) for a, b in zip(ref, wrong)), mistake
        # and the variant machinery itself is faithful without the mistake
        assert all(np.array_equal(a, b) for a, b in zip(ref, ek.match_variant(*c, None))), mistake


def _pairs():
    return [(g, n) for g in ek.GEOMETRIES for n in ek.N_SWEEP if ek.applicable(g, n)]


@pytest.mark.parametrize("geom", ek.GEOMETRIES)
def test_geometry_promises_and_port(geom):
    worst = worst_base = 0.0
    for n in ek.N_SWEEP:
        if not ek.applicable(geom, n):
            continue
        X, cx, Y, cy = ek.placed_pair(geom, n, seed=n)
        d, sig = ek.cov_facts(X, cx, Y, cy)
        if n >= 4:
            if geom.startswith("mirror"):
                assert d == -1 and sig[1] - sig[2] >= 1e-3 * sig[0], (geom, n, sig)
            elif geom not in ("coplanar", "collinear"):
                assert d == 1, (geom, n)
            if geom == "isotropic":
                assert sig[2] >= 0.99 * sig[0], (n, sig)
            if geom == "tpose":
                assert sig[1] >= 0.99 * sig[0] and sig[2] < 0.5 * sig[0], (n, sig)
            if geom == "coplanar":
                assert sig[2] <= 1e-6 * sig[0], (n, sig)
        if geom == "collinear":
            assert sig[1] <= 1e-6 * sig[0], (n, sig)
        pve, pa, tp, ta, tb = ek.points_reference(X, cx, Y, cy)
        if geom == "exact":
            assert pa <= ta, (n, pa, ta)
        dev = abs(ek.points_port(X, cx, Y, cy) - pa)
        worst, worst_base = max(worst, dev / ta), max(worst_base, dev / tb)
        assert dev <= ta, (geom, n, dev / ta)
    print(f"{geom}: numpy port of the kernel's Procrustes vs roma_ref, worst err/tol {worst:.3g} "
          f"({worst_base:.3g} of the bound without the rank-deficiency term)")


def test_point_mistakes_move_the_oracle():
    """On the batches of the GPU sensitivity test (same builders, same seeds)."""
    for mistake in ek.POINT_MISTAKES:
        best = 0.0
        for geom, npt, seed in ek.SENSITIVITY_POINTS:
            pred, pc, gt, gc, pairs = ek.points_batch(geom, npt, 3, seed=seed, centres=(True, True))
            ref = ek.points_refs(pred, pc, gt, gc, pairs)
            w = ek.points_refs(pred, pc, gt, gc, pairs, mistake)
            best = max(best, (np.abs(w[:, 0] - ref[:, 0]) / ref[:, 2]).max(), (np.abs(w[:, 1] - ref[:, 1]) / ref[:, 3]).max())
        print(f"points mistake {mistake}: oracle moves by {best:.3g} x the bound")
        assert best > 1.0, mistake


def test_regression_bound_and_mistakes():
    """The bound holds for an fp32 evaluation in the kernel's order, and each planted mistake moves the fp64 oracle
    outside it on the inputs of the GPU sensitivity test."""
    N = 700
    Am, rpm, _, _ = ek.make_csr(list(ek.NNZ_EDGES) * 2, N, seed=23)
    assert np.array_equal(np.diff(rpm), list(ek.NNZ_EDGES) * 2)
    X, c, K, pairs = ek.reg_inputs(N, 22)
    rows, root = ek.ROOT_ROWS, 4
    xc = (X[0] - c[0]).astype(np.float32)
    f32 = lambda r: np.array([sum(np.float32(Am[r, k]) * xc[k, q] for k in np.nonzero(Am[r])[0]) for q in range(3)],
                             np.float32) if np.count_nonzero(Am[r]) else np.zeros(3, np.float32)
    y, tol = ek.regress_reference(Am, rpm, X[0], c[0], rows, root)
    got = np.stack([f32(r) - f32(root) for r in rows]).astype(np.float64)
    assert (np.abs(got - y.numpy()) <= tol.numpy()).all()
    moved = {k: 0.0 for k in ek.REG_MISTAKES}
    for side in (0, 1):
        for m in range(4):
            s = pairs[m, side]
            y, tol = ek.regress_reference(Am, rpm, X[s], c[s], rows, root)
            for mistake in ("before_centring", "no_root"):
                w, _ = ek.regress_reference(Am, rpm, X[s], c[s], rows, root, mistake)
                moved[mistake] = max(moved[mistake], ((w - y).abs() / tol.clamp_min(1e-300)).max().item())
    A, rp, _, _ = ek.make_csr([1, 31, 32, 33, 200, 3, 48, 7, 9], N, seed=21, positive=True)
    for side in (0, 1):
        for m in range(4):
            s, o = pairs[m, side], pairs[m, 1 - side]
            y, tol = ek.regress_reference(A, rp, X[s], c[s], ek.PROJ_ROWS, -1)
            q, qt = ek.project_reference(y, tol, K[s])
            qo, _ = ek.project_reference(y, tol, K[o])
            moved["other_K"] = max(moved["other_K"], ((qo - q).abs() / qt).max().item())
    for k, r in moved.items():
        print(f"regression mistake {k}: oracle moves by {r:.3g} x the bound")
        assert r > 1.0, k
