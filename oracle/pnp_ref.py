"""TEST INFRASTRUCTURE ONLY -- numpy (float64) restatement of the reference's
per-object PnP stage.  Never imported by the product path.

The arithmetic of this stage lives in a third-party dependency that is NOT
under /root/reference: OpenCV (`requirements.txt:11` pins only
`opencv-python>=4.5.3.56`; the build container has 4.13.0).  Call sites:
`cv2.solvePnPGeneric(flags=SOLVEPNP_ITERATIVE)` at
utils/pnp/cuboid_pnp_solver.py:165-171 and `cv2.projectPoints` at :203-204.
Published algorithm of SOLVEPNP_ITERATIVE for >=6 non-planar points, zero
distortion (OpenCV calib3d `findExtrinsicCameraParams2`):
  1. normalise image points with K^-1;
  2. DLT: stack the 2n x 12 system, take the right singular vector of the
     smallest singular value of L^T L, fix the sign by det(R) > 0, project the
     3x3 block onto SO(3) with an SVD and rescale t by ||R_orth|| / ||R_dlt||;
  3. Levenberg-Marquardt on the 6-DoF reprojection error (pixels).
The answer is the local least-squares minimum reached from the DLT start.

With 4 or 5 valid points the reference passes `cv2.SOLVEPNP_EPNP` (cuboid_pnp_solver.py:162-163).  `epnp` restates the
published algorithm of OpenCV's calib3d epnp.cpp (Lepetit, Moreno-Noguer, Fua 2009): control points from the PCA of the
object points, barycentric coordinates, the 2n x 12 system and the 4 smallest singular vectors of M^T M, three beta
approximations each refined by 5 Gauss-Newton steps, absolute orientation, smallest mean reprojection error.  M has
rank <= 2n < 12 there, so its null space is degenerate by construction and its basis is whatever the SVD routine
returns: pinned against cv2 on CONSISTENT 5-point input (1e-9); on 4 points or noisy input cv2 and this file return
different, equally valid EPnP poses (tests/test_oracle_pnp.py reports the gap).

Parity status: PINNED against cv2 4.13 (`tests/test_oracle_pnp.py` compares
with `cv2.solvePnPGeneric` directly -- cv2 is part of the image on both the
build container and the GPU box) and against the reference's own
`pnp_shell` through `oracle/ref_shims.py` / `tests/golden/pnp_*.npz`.

Reference lines followed (relative to /root/reference/src/lib):
  utils/pnp/cuboid_objectron.py:83-109   Cuboid3d.generate_vertexes -> cuboid_vertices
  detectors/base_detector.py:548-566     point assembly by rep_mode -> assemble_points
  utils/pnp/cuboid_pnp_solver.py:91-239  solve_pnp                  -> solve_pnp
  utils/pnp/cuboid_pnp_solver.py:241-247 convert_rvec_to_quaternion -> rvec_to_quat
  utils/pnp/cuboid_pnp_shell.py:11-93    pnp_shell                  -> pnp_shell
"""
import numpy as np

F32 = np.float32

ST_NOT_RUN = 0
ST_OK = 1            # pnp_shell returned a tuple (goes into `boxes`)
ST_INVISIBLE = 2     # pose written into the result dict, but a visibility gate returned None
ST_BEHIND = 3        # z < 0 on the OpenCV tvec  (cuboid_pnp_solver.py:208-220)
ST_FEW_POINTS = 4    # < 4 valid points (4-5 points: EPnP, restated in `epnp`)
ST_SOLVER_FAIL = 5


def cuboid_vertices(obj_scale):
    """Cuboid3d(scale / scale[1]).get_vertices(); float32 arithmetic like the
    reference (obj_scale is a float32 numpy row), order (-x-y-z, -x-y+z, ...)."""
    sc = np.asarray(obj_scale, F32)
    size = (F32(1) * sc / sc[1]).astype(F32)
    w, h, d = size
    r, l = w / F32(2), -w / F32(2)
    t, b = h / F32(2), -h / F32(2)
    f, re = d / F32(2), -d / F32(2)
    v = np.array([[l, b, re], [l, b, f], [l, t, re], [l, t, f],
                  [r, b, re], [r, b, f], [r, t, re], [r, t, f]], dtype=F32)
    return v.astype(np.float64)


def assemble_points(det, rep_mode):
    """base_detector.py:551-566: 8 points (rep 0/3/4) or 16 interleaved (rep 1)."""
    if rep_mode in (0, 3, 4):
        return np.asarray(det["kps"], np.float64).reshape(-1, 2)
    if rep_mode == 1:
        p1 = np.asarray(det["kps_displacement_mean"], np.float64).reshape(-1, 2)
        p2 = np.asarray(det["kps_heatmap_mean"], np.float64).reshape(-1, 2)
        return np.hstack((p1, p2)).reshape(-1, 2)
    raise NotImplementedError("rep_mode 2 samples from a random GMM; excluded from parity (SURVEY 8a-9)")


def rodrigues(rvec):
    th = np.linalg.norm(rvec)
    if th < 1e-300:
        return np.eye(3)
    k = rvec / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)


def mat_to_quat(R):
    """Rotation matrix -> unit quaternion xyzw with w >= 0 (what
    scipy `from_matrix().as_rotvec()` + convert_rvec_to_quaternion produce)."""
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    q = np.zeros(4)
    c = [R[0, 0], R[1, 1], R[2, 2], tr]
    i = int(np.argmax(c))
    if i == 3:
        q[3] = 1 + tr
        q[0] = R[2, 1] - R[1, 2]
        q[1] = R[0, 2] - R[2, 0]
        q[2] = R[1, 0] - R[0, 1]
    else:
        j, k = (i + 1) % 3, (i + 2) % 3
        q[i] = 1 - tr + 2 * R[i, i]
        q[j] = R[j, i] + R[i, j]
        q[k] = R[k, i] + R[i, k]
        q[3] = R[k, j] - R[j, k]
    q /= np.linalg.norm(q)
    if q[3] < 0:
        q = -q
    return q


def mat_to_rvec(R):
    q = mat_to_quat(R)
    s = np.linalg.norm(q[:3])
    if s < 1e-300:
        return np.zeros(3)
    ang = 2 * np.arctan2(s, q[3])
    return q[:3] / s * ang


def rvec_to_quat(rvec):
    th = np.sqrt(rvec[0] * rvec[0] + rvec[1] * rvec[1] + rvec[2] * rvec[2])
    ax = np.asarray(rvec, np.float64) / th
    return np.array([ax[0] * np.sin(th / 2), ax[1] * np.sin(th / 2), ax[2] * np.sin(th / 2), np.cos(th / 2)])


def quat_to_mat(q):
    x, y, z, w = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def project(X, R, t, Kc):
    P = X @ R.T + t
    return np.stack([Kc[0, 0] * P[:, 0] / P[:, 2] + Kc[0, 2], Kc[1, 1] * P[:, 1] / P[:, 2] + Kc[1, 2]], 1)


def dlt_init(X, uv, Kc):
    n = X.shape[0]
    x = (uv[:, 0] - Kc[0, 2]) / Kc[0, 0]
    y = (uv[:, 1] - Kc[1, 2]) / Kc[1, 1]
    L = np.zeros((2 * n, 12))
    for i in range(n):
        Xi, Yi, Zi = X[i]
        L[2 * i] = [Xi, Yi, Zi, 1, 0, 0, 0, 0, -x[i] * Xi, -x[i] * Yi, -x[i] * Zi, -x[i]]
        L[2 * i + 1] = [0, 0, 0, 0, Xi, Yi, Zi, 1, -y[i] * Xi, -y[i] * Yi, -y[i] * Zi, -y[i]]
    w, V = np.linalg.eigh(L.T @ L)
    p = V[:, 0]
    RR = np.array([[p[0], p[1], p[2]], [p[4], p[5], p[6]], [p[8], p[9], p[10]]])
    tt = np.array([p[3], p[7], p[11]])
    if np.linalg.det(RR) < 0:
        RR, tt = -RR, -tt
    sc = np.linalg.norm(RR)
    U, _, Vt = np.linalg.svd(RR)
    R = U @ Vt
    tt = tt * (np.linalg.norm(R) / sc)
    return R, tt


def refine_lm(X, uv, Kc, R, t, max_iter=20):
    """Levenberg-Marquardt on the pixel reprojection error with a left
    multiplicative rotation update R <- exp([dw]x) R (the minimiser does not
    depend on the parametrisation).  max_iter = 20 accepted steps mirrors cv2's
    TermCriteria(MAX_ITER + EPS, 20, FLT_EPSILON): converged cases are unaffected
    (agreement with cv2 <= 1e-8), unconverged ones stay close to what cv2 returns."""
    def resid(R, t):
        return (project(X, R, t, Kc) - uv).reshape(-1)

    lam = 1e-3
    r = resid(R, t)
    cost = r @ r
    for _ in range(max_iter):
        P = X @ R.T + t
        J = np.zeros((2 * X.shape[0], 6))
        for i in range(X.shape[0]):
            px, py, pz = P[i]
            du = np.array([Kc[0, 0] / pz, 0, -Kc[0, 0] * px / (pz * pz)])
            dv = np.array([0, Kc[1, 1] / pz, -Kc[1, 1] * py / (pz * pz)])
            q = P[i] - t
            dPdw = -np.array([[0, -q[2], q[1]], [q[2], 0, -q[0]], [-q[1], q[0], 0]])
            J[2 * i, :3] = du @ dPdw
            J[2 * i, 3:] = du
            J[2 * i + 1, :3] = dv @ dPdw
            J[2 * i + 1, 3:] = dv
        A = J.T @ J
        g = J.T @ r
        improved = False
        for _ in range(30):
            try:
                d = -np.linalg.solve(A + lam * np.diag(np.diag(A)), g)
            except np.linalg.LinAlgError:
                lam *= 10
                continue
            Rn = rodrigues(d[:3]) @ R
            tn = t + d[3:]
            rn = resid(Rn, tn)
            cn = rn @ rn
            if np.isfinite(cn) and cn <= cost:
                improved = True
                break
            lam *= 10
        if not improved:
            break
        step = np.linalg.norm(d)
        R, t, r = Rn, tn, rn
        dec = cost - cn
        cost = cn
        lam = max(lam * 0.1, 1e-12)
        if step < 1e-10 or dec <= 1e-28 * max(cost, 1e-300):
            break
    return R, t, cost


def epnp(pws, us, Kc):
    """cv2.solvePnP(..., flags=SOLVEPNP_EPNP) without distortion: (R, t, mean reprojection error in pixels)."""
    pws = np.asarray(pws, np.float64)
    us = np.asarray(us, np.float64)
    n = len(pws)
    fu, fv, uc, vc = Kc[0, 0], Kc[1, 1], Kc[0, 2], Kc[1, 2]
    cws = np.zeros((4, 3))
    cws[0] = pws.mean(0)
    PW0 = pws - cws[0]
    U, D, _ = np.linalg.svd(PW0.T @ PW0)
    for i in range(1, 4):
        cws[i] = cws[0] + np.sqrt(D[i - 1] / n) * U[:, i - 1]
    CC = (cws[1:] - cws[0]).T
    if abs(np.linalg.det(CC)) < 1e-300:
        return None
    CCi = np.linalg.inv(CC)
    al = np.zeros((n, 4))
    al[:, 1:] = (pws - cws[0]) @ CCi.T
    al[:, 0] = 1 - al[:, 1:].sum(1)
    M = np.zeros((2 * n, 12))
    for j in range(4):
        M[0::2, 3 * j] = al[:, j] * fu
        M[0::2, 3 * j + 2] = al[:, j] * (uc - us[:, 0])
        M[1::2, 3 * j + 1] = al[:, j] * fv
        M[1::2, 3 * j + 2] = al[:, j] * (vc - us[:, 1])
    U, D, _ = np.linalg.svd(M.T @ M)
    v = [U[:, 11], U[:, 10], U[:, 9], U[:, 8]]
    pairs = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    dv = np.array([[vi[3 * a:3 * a + 3] - vi[3 * b:3 * b + 3] for a, b in pairs] for vi in v])     # [4, 6, 3]
    L = np.zeros((6, 10))
    for i in range(6):
        d = dv[:, i]
        L[i] = [d[0] @ d[0], 2 * d[0] @ d[1], d[1] @ d[1], 2 * d[0] @ d[2], 2 * d[1] @ d[2], d[2] @ d[2],
                2 * d[0] @ d[3], 2 * d[1] @ d[3], 2 * d[2] @ d[3], d[3] @ d[3]]
    rho = np.array([((cws[a] - cws[b]) ** 2).sum() for a, b in pairs])
    lsq = lambda A, b: np.linalg.lstsq(A, b, rcond=None)[0]      # noqa: E731

    def start(ap):
        be = np.zeros(4)
        if ap == 0:
            b4 = lsq(L[:, [0, 1, 3, 6]], rho)
            be[0] = np.sqrt(abs(b4[0]))
            be[1:] = (-b4[1:] if b4[0] < 0 else b4[1:]) / be[0]
            return be
        b = lsq(L[:, :3] if ap == 1 else L[:, :5], rho)
        if b[0] < 0:
            be[0], be[1] = np.sqrt(-b[0]), (np.sqrt(-b[2]) if b[2] < 0 else 0.0)
        else:
            be[0], be[1] = np.sqrt(b[0]), (np.sqrt(b[2]) if b[2] > 0 else 0.0)
        if b[1] < 0:
            be[0] = -be[0]
        if ap == 2:
            be[2] = b[3] / be[0]
        return be

    best = None
    for ap in range(3):
        be = start(ap)
        if not np.isfinite(be).all() or be[0] == 0:
            continue
        for _ in range(5):
            A = np.zeros((6, 4))
            r = L
            A[:, 0] = 2 * r[:, 0] * be[0] + r[:, 1] * be[1] + r[:, 3] * be[2] + r[:, 6] * be[3]
            A[:, 1] = r[:, 1] * be[0] + 2 * r[:, 2] * be[1] + r[:, 4] * be[2] + r[:, 7] * be[3]
            A[:, 2] = r[:, 3] * be[0] + r[:, 4] * be[1] + 2 * r[:, 5] * be[2] + r[:, 8] * be[3]
            A[:, 3] = r[:, 6] * be[0] + r[:, 7] * be[1] + r[:, 8] * be[2] + 2 * r[:, 9] * be[3]
            b = rho - (r[:, 0] * be[0] ** 2 + r[:, 1] * be[0] * be[1] + r[:, 2] * be[1] ** 2 + r[:, 3] * be[0] * be[2] +
                       r[:, 4] * be[1] * be[2] + r[:, 5] * be[2] ** 2 + r[:, 6] * be[0] * be[3] + r[:, 7] * be[1] * be[3] +
                       r[:, 8] * be[2] * be[3] + r[:, 9] * be[3] ** 2)
            be = be + lsq(A, b)
        ccs = sum(be[i] * v[i].reshape(4, 3) for i in range(4))
        pcs = al @ ccs
        if pcs[0, 2] < 0:
            pcs = -pcs
        pc0, pw0 = pcs.mean(0), pws.mean(0)
        Uo, _, Vt = np.linalg.svd((pcs - pc0).T @ (pws - pw0))
        R = Uo @ Vt
        if np.linalg.det(R) < 0:
            R[2] = -R[2]
        t = pc0 - R @ pw0
        P = pws @ R.T + t
        err = np.sqrt((us[:, 0] - (uc + fu * P[:, 0] / P[:, 2])) ** 2 + (us[:, 1] - (vc + fv * P[:, 1] / P[:, 2])) ** 2).mean()
        if np.isfinite(err) and (best is None or err < best[2]):
            best = (R, t, err)
    return best


def solve_pnp(points2d, vertices, Kc, opencv_return=False):
    """cuboid_pnp_solver.py:91-239.  Returns dict(status, location, quaternion,
    projected_points[8,2], reproj_err, R_cv, t_cv)."""
    pts = np.asarray(points2d, np.float64).reshape(-1, 2)
    n_in = pts.shape[0]
    o2, o3 = [], []
    for i in range(n_in):
        if pts[i, 0] < -5000 or pts[i, 1] < -5000:
            continue
        o2.append(pts[i])
        o3.append(vertices[int(i // (n_in / 8))])
    out = {"status": ST_FEW_POINTS, "location": None, "quaternion": None,
           "projected_points": pts, "reproj_err": None, "n_pts": len(o2)}
    if len(o2) < 4:
        return out          # cuboid_pnp_solver.py:157-160
    o2 = np.array(o2)
    o3 = np.array(o3)
    if not (np.isfinite(o2).all() and np.isfinite(o3).all()):
        # a NaN / inf point or cuboid vertex (scale[1] = 0, denormal or inf, an overflowing width): cv2 asserts on
        # such input, the device solvers end in SOLVER_FAIL -- the rule of DESIGN.md section 5
        out["status"] = ST_SOLVER_FAIL
        return out
    if len(o2) < 6:         # :162-163 SOLVEPNP_EPNP
        sol = epnp(o3, o2, np.asarray(Kc, np.float64))
        if sol is None:
            out["status"] = ST_SOLVER_FAIL
            return out
        R, t = sol[0], sol[1]
        cost = float(((project(o3, R, t, Kc) - o2) ** 2).sum())
    else:
        R, t = dlt_init(o3, o2, Kc)
        R, t, cost = refine_lm(o3, o2, Kc, R, t)
    if not np.all(np.isfinite(R)) or not np.all(np.isfinite(t)):
        out["status"] = ST_SOLVER_FAIL
        return out
    out["reproj_err"] = np.sqrt(cost / (2 * len(o2)))      # cv2: RMSE over the 2n residuals
    out["R_cv"], out["t_cv"] = R, t
    out["projected_points"] = project(vertices, R, t, Kc)
    if t[2] < 0:
        out["status"] = ST_BEHIND
        return out
    if opencv_return:
        out["location"] = list(t)
        out["quaternion"] = mat_to_quat(R)
    else:
        M = np.array([[0, 1, 0], [1, 0, 0], [0, 0, -1.0]])
        out["location"] = list(M @ t)
        out["quaternion"] = mat_to_quat(M @ R)
    out["status"] = ST_OK
    return out


def pnp_shell(det, points, Kc, width, height, category="chair", opencv_return=False):
    """cuboid_pnp_shell.py:11-93.  Mutates `det` like the reference and returns
    (status, tuple-or-None)."""
    V = cuboid_vertices(det["obj_scale"])
    sol = solve_pnp(points, V, np.asarray(Kc, np.float64), opencv_return)
    det["pnp_status"] = sol["status"]
    det["pnp_n_pts"] = sol["n_pts"]
    if sol["location"] is None:
        return sol["status"], None
    det["location"] = sol["location"]
    det["quaternion_xyzw"] = sol["quaternion"]
    det["projected_cuboid"] = sol["projected_points"]
    det["reproj_err"] = sol["reproj_err"]
    ori = quat_to_mat(sol["quaternion"])
    p3 = V @ ori.T + np.asarray(sol["location"])
    p3 = np.vstack([p3.mean(0, keepdims=True), p3])
    det["kps_3d_cam"] = p3
    pp = np.vstack([sol["projected_points"].mean(0, keepdims=True), sol["projected_points"]]).copy()
    pp[:, 0] /= width
    pp[:, 1] /= height
    det["kps_pnp"] = pp
    if category not in ("bike", "laptop", "shoe"):
        thr = 6 if category in ("book", "chair", "cereal_box") else 3
        nv = int(np.sum((pp[:, 0] < 0) | (pp[:, 0] > 1) | (pp[:, 1] < 0) | (pp[:, 1] > 1)))
        if nv >= thr:
            det["pnp_status"] = ST_INVISIBLE
            return ST_INVISIBLE, None
    if not (pp[0, 0] > 0 and pp[0, 0] < 1 and pp[0, 1] > 0 and pp[0, 1] < 1):
        det["pnp_status"] = ST_INVISIBLE
        return ST_INVISIBLE, None
    kp = np.asarray(det["kps"], np.float64).reshape(-1, 2)
    po = np.vstack([kp.mean(0, keepdims=True), kp]).copy()
    po[:, 0] /= width
    po[:, 1] /= height
    return ST_OK, (pp, p3, np.array(det["obj_scale"]), po, det)
