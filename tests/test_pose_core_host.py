"""centerpose_b200/csrc/pose_core.h is __host__ __device__: the exact code the
CUDA decode kernel runs per detection is compiled with g++ here and checked
against the oracle and cv2 without a GPU."""
import ctypes

import numpy as np
import pytest

from centerpose_b200 import synth
from oracle import decode_ref, pnp_ref

dp = ctypes.POINTER(ctypes.c_double)
fp = ctypes.POINTER(ctypes.c_float)
ip = ctypes.POINTER(ctypes.c_int)


def _solve(Lh, pts, scale, K, w, h, vis=6, ocv=0):
    pts = np.ascontiguousarray(pts, np.float64)
    scale = np.ascontiguousarray(scale, np.float32)
    K = np.ascontiguousarray(K, np.float64)
    out = np.zeros(80)
    st, npt = ctypes.c_int(), ctypes.c_int()
    Lh.host_solve_and_shell(pts.ctypes.data_as(dp), ctypes.c_int(pts.shape[0]), scale.ctypes.data_as(fp),
                            K.ctypes.data_as(dp), ctypes.c_double(w), ctypes.c_double(h), vis, ocv,
                            out.ctypes.data_as(dp), ctypes.byref(st), ctypes.byref(npt))
    return st.value, npt.value, out


def test_pnp_matches_oracle_and_cv2(pose_host):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    cam = synth.default_camera(512, 512)
    worst = np.zeros(4)
    M = np.array([[0, 1, 0], [1, 0, 0], [0, 0, -1.]])
    for trial in range(120):
        scale = np.array([rng.uniform(0.3, 2), rng.uniform(0.5, 1.5), rng.uniform(0.3, 2)], np.float32)
        V = pnp_ref.cuboid_vertices(scale)
        R = synth._rand_rot(rng)
        tz = rng.uniform(2.5, 7)
        t = np.array([rng.uniform(-.3, .3) * tz, rng.uniform(-.3, .3) * tz, tz])
        pts = np.repeat(pnp_ref.project(V, R, t, cam), 2, axis=0) + rng.normal(0, rng.choice([0.0, 0.5, 2.0, 5.0]), (16, 2))
        for j in range(8):
            if rng.uniform() < 0.3:
                pts[2 * j + 1] = [-10000, -10000]
        det = {"obj_scale": scale, "kps": pts[0::2].reshape(-1)}
        st_o, _ = pnp_ref.pnp_shell(det, pts, cam, 512, 512, "chair")
        st, npt, out = _solve(pose_host, pts, scale, cam, 512, 512, 6, 0)
        assert st == st_o and npt == int((pts[:, 0] > -5000).sum())
        ok = pts[:, 0] > -5000
        X = np.array([V[i // 2] for i in range(16)])[ok]
        _, rv, tv, err = cv2.solvePnPGeneric(X, pts[ok], cam, np.zeros((4, 1)), flags=cv2.SOLVEPNP_ITERATIVE)
        qcv = pnp_ref.mat_to_quat(M @ pnp_ref.rodrigues(rv[0].reshape(3)))
        lcv = M @ tv[0].reshape(3)
        if st in (1, 2):
            q = out[3:7]
            if q @ qcv < 0:
                q = -q
            worst[0] = max(worst[0], np.abs(out[0:3] - lcv).max() / np.linalg.norm(lcv))
            worst[1] = max(worst[1], np.abs(q - qcv).max())
            worst[2] = max(worst[2], abs(out[7] - err.flatten()[0]))
            worst[3] = max(worst[3], np.abs(out[24:51].reshape(9, 3) - det["kps_3d_cam"]).max())
    assert worst[0] <= 1e-6 and worst[1] <= 1e-6 and worst[2] <= 1e-8 and worst[3] <= 1e-6, worst


def test_pnp_failure_paths(pose_host):
    cam = synth.default_camera(512, 512)
    scale = np.array([1.0, 1.0, 1.0], np.float32)
    pts = np.full((16, 2), -10000.0)
    pts[:6:2] = np.random.default_rng(1).uniform(100, 400, (3, 2))     # only 3 valid points
    st, npt, _ = _solve(pose_host, pts, scale, cam, 512, 512)
    assert st == 4 and npt == 3                                        # < 4 points: cuboid_pnp_solver.py:157-160
    # a cuboid far outside the image: pose found, visibility gate rejects it (cuboid_pnp_shell.py:59-79)
    V = pnp_ref.cuboid_vertices(scale)
    uv = pnp_ref.project(V, np.eye(3), np.array([6.0, 0.0, 4.0]), cam)
    st, _, out = _solve(pose_host, np.repeat(uv, 2, 0), scale, cam, 512, 512, 6, 0)
    assert st == 2
    st3, _, _ = _solve(pose_host, np.repeat(uv, 2, 0), scale, cam, 512, 512, 0, 0)     # bike/laptop/shoe: only centre gate
    assert st3 == 2


def test_nonfinite_input_is_solver_failure(pose_host):
    """A NaN / inf image point or cuboid vertex (scale[1] = 0, denormal or inf; a width that overflows fp32) is
    SOLVER_FAIL in pose_core.h and in the oracle -- on the DLT + LM path (8 points) and on the EPnP path (5 points)."""
    cam = synth.default_camera(512, 512)
    V = pnp_ref.cuboid_vertices(np.ones(3, np.float32))
    uv = pnp_ref.project(V, synth._rand_rot(np.random.default_rng(5)), np.array([0.1, -0.2, 4.0]), cam)
    cases = [(uv, s) for s in ((1, 0, 1), (1, 1e-40, 1), (1, np.inf, 1), (3e38, 1e-3, 1), (1, -0.0, 1))]
    for bad in (np.inf, np.nan):
        p = uv.copy()
        p[2, 1] = bad
        cases.append((p, (1, 1, 1)))
    for pts, sc in cases:
        for keep in (8, 5):
            p = pts.copy()
            p[keep:] = -10000.0
            scale = np.array(sc, np.float32)
            st, npt, out = _solve(pose_host, p, scale, cam, 512, 512, 6, 0)
            assert (st, npt) == (pnp_ref.ST_SOLVER_FAIL, keep), (sc, keep, st)
            with np.errstate(all="ignore"):
                assert pnp_ref.pnp_shell({"obj_scale": scale, "kps": p.reshape(-1)}, p, cam, 512, 512)[0] == st


def _epnp_case(rng, n, noise):
    import cv2
    K = np.array([[663.0, 0, 300.3], [0, 663.0, 395.0], [0, 0, 1.0]])
    scale = rng.uniform(0.3, 2, 3).astype(np.float32)
    V = pnp_ref.cuboid_vertices(scale)
    rv = rng.normal(size=3) * 0.7
    t = np.array([rng.uniform(-.3, .3), rng.uniform(-.3, .3), rng.uniform(2, 4)])
    R = cv2.Rodrigues(rv)[0]
    idx = np.sort(rng.choice(8, n, replace=False))
    uv = pnp_ref.project(V, R, t, K) + rng.normal(size=(8, 2)) * noise
    pts = np.full((8, 2), -10000.0)
    pts[idx] = uv[idx]
    ok, rvs, tvs, _ = cv2.solvePnPGeneric(V[idx].reshape(-1, 1, 3), uv[idx].reshape(-1, 1, 2), K, np.zeros(4),
                                          flags=cv2.SOLVEPNP_EPNP)
    return K, scale, V, idx, uv, pts, cv2.Rodrigues(rvs[0])[0], tvs[0].reshape(3)


def _reproj(V, idx, uv, R, t, K):
    return np.sqrt(((pnp_ref.project(V[idx], R, t, K) - uv[idx]) ** 2).sum(1)).mean()


def test_epnp_five_consistent_points_match_cv2(pose_host):
    """4 - 5 valid points take EPnP (cuboid_pnp_solver.py:162-163).  On consistent 5-point input the pose is unique and
    both the C++ (host build of the device code) and the numpy restatement agree with cv2.SOLVEPNP_EPNP to 1e-8."""
    pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    n_ok = 0
    for _ in range(20):
        K, scale, V, idx, uv, pts, Rc, tc = _epnp_case(rng, 5, 0.0)
        if tc[2] < 0 or _reproj(V, idx, uv, Rc, tc, K) > 1e-6:
            continue                                           # cv2 itself did not find the exact pose
        st, npt, out = _solve(pose_host, pts, scale, K, 600, 800, 0, 1)
        assert npt == 5 and st in (1, 2)
        Ro = pnp_ref.quat_to_mat(out[3:7])
        assert np.abs(Ro - Rc).max() <= 1e-8 and np.abs(out[0:3] - tc).max() <= 1e-8
        sol = pnp_ref.epnp(V[idx], uv[idx], K)
        assert np.abs(sol[0] - Rc).max() <= 1e-8 and np.abs(sol[1] - tc).max() <= 1e-8
        n_ok += 1
    assert n_ok >= 15


def test_epnp_degenerate_cases_stay_valid(pose_host):
    """4 points / noisy points: M has a structurally degenerate null space, cv2 (LAPACK basis) and this code (Jacobi basis)
    return different valid EPnP poses.  Bound: a pose is produced and its reprojection error is of the order of cv2's."""
    pytest.importorskip("cv2")
    rng = np.random.default_rng(4)
    ratios = []
    for trial in range(40):
        n, noise = (5, 1.0) if trial % 2 else (4, 0.5)
        K, scale, V, idx, uv, pts, Rc, tc = _epnp_case(rng, n, noise)
        st, npt, out = _solve(pose_host, pts, scale, K, 600, 800, 0, 1)
        assert npt == n and st in (1, 2, 3, 5)
        if st in (1, 2) and tc[2] > 0:
            ours = _reproj(V, idx, uv, pnp_ref.quat_to_mat(out[3:7]), out[0:3], K)
            ratios.append((ours + 0.5) / (_reproj(V, idx, uv, Rc, tc, K) + 0.5))
    print("EPnP reprojection error vs cv2 (ratio of error + 0.5 px): median %.2f  90th pct %.2f  n %d"
          % (np.median(ratios), np.percentile(ratios, 90), len(ratios)))
    assert len(ratios) >= 25 and np.median(ratios) <= 1.5


def test_soft_nms_matches_oracle(pose_host):
    rng = np.random.default_rng(2)
    for trial in range(100):
        n = int(rng.integers(1, 40))
        ctr = rng.uniform(100, 400, size=(n, 2))
        wh = rng.uniform(20, 150, size=(n, 2))
        bb = np.concatenate([ctr - wh / 2, ctr + wh / 2], 1)
        sc = np.sort(rng.uniform(0.3001, 1, size=n))[::-1].copy()
        boxes = [{"bbox": bb[i].copy(), "score": float(sc[i]), "id": i} for i in range(n)]
        nn = decode_ref.soft_nms(boxes, threshold=0.3)
        b2, s2, perm = bb.copy(), sc.copy(), np.arange(n, dtype=np.int32)
        n2 = pose_host.host_soft_nms(b2.ctypes.data_as(dp), s2.ctypes.data_as(dp), perm.ctypes.data_as(ip), n,
                                     ctypes.c_double(0.3))
        assert nn == n2 and [b["id"] for b in boxes[:nn]] == list(perm[:n2])
        assert np.allclose([b["score"] for b in boxes[:nn]], s2[:n2], rtol=0, atol=1e-15)


def test_moments_matches_oracle(pose_host):
    rng = np.random.default_rng(4)
    for trial in range(100):
        nr, nc = int(rng.integers(1, 12)), int(rng.integers(1, 12))
        w = np.ascontiguousarray(rng.uniform(0, 1, size=(nr, nc)) * (rng.uniform(size=(nr, nc)) > 0.3))
        if w.sum() == 0:
            continue
        out5 = np.zeros(5)
        ok = pose_host.host_moments(w.ctypes.data_as(dp), nr, nc, out5.ctypes.data_as(dp))
        with np.errstate(all="ignore"):
            ref = decode_ref.moments(w)
        if not np.all(np.isfinite(ref)):
            continue
        assert ok and np.allclose(out5, ref, rtol=1e-12, atol=1e-14)


def test_moments_rejects_what_fitgaussian_rejects(pose_host):
    """Raw (opt.mse_loss) windows mix signs: a non-positive total or centroid row / column sum, a centroid outside the
    window, a NaN or negative width.  pose::moments accepts exactly the windows whose start point
    scipy.optimize.least_squares takes with fitgaussian's bounds (decode_ref.fit_start), with the same values."""
    opt = pytest.importorskip("scipy.optimize")
    rng = np.random.default_rng(14)
    seen = {True: 0, False: 0}
    for trial in range(400):
        nr, nc = int(rng.integers(1, 12)), int(rng.integers(1, 12))
        w = rng.uniform(-0.3, 1.0, size=(nr, nc)) * (rng.uniform(size=(nr, nc)) > 0.3)
        w[rng.uniform(size=(nr, nc)) < 0.2] = -rng.uniform(0.0, 0.5)
        w = np.ascontiguousarray(w)
        out5 = np.zeros(5)
        ok = bool(pose_host.host_moments(w.ctypes.data_as(dp), nr, nc, out5.ctypes.data_as(dp)))
        fit = decode_ref.fit_start(w)
        assert ok == (fit is not None), (trial, w)
        seen[ok] += 1
        with np.errstate(all="ignore"):
            try:
                ref = decode_ref.moments(w)
            except (ValueError, IndexError, OverflowError):
                assert not ok
                continue
        x0 = np.array(ref, np.float64)
        fitgaussian = lambda: opt.least_squares(lambda p: np.zeros(1), x0, bounds=(0, [np.inf, nr, nc, np.inf, np.inf]),
                                                max_nfev=1)
        if not ok:
            with pytest.raises(ValueError):
                fitgaussian()
            continue
        assert np.allclose(out5, ref, rtol=1e-12, atol=1e-14)
        fitgaussian()
    assert seen[True] > 20 and seen[False] > 20, seen


def test_cuboid_vertices_order(pose_host):
    scale = np.array([0.4, 0.8, 1.2], np.float32)
    V = np.zeros(24)
    pose_host.host_cuboid_vertices(scale.ctypes.data_as(fp), V.ctypes.data_as(dp))
    assert np.array_equal(V.reshape(8, 3), pnp_ref.cuboid_vertices(scale))
