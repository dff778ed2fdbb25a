"""The warp-cooperative PnP of the decode kernel (pnp_warp.cuh, phase G of decode.cu) at its edges, driven through
`cp_decode_pnp` by the scenes of tests/pnp_scenes.py, detection by detection against

  (a) the host build of pose_core.h on the identical fp64 points: equal status and point count, and the pose fields
      within HOST_BAR -- over 300x tighter than the stated tolerances, and below what one LM iteration less or points
      rounded to fp32 (in a frame where that rounding is not exact) move them;
  (b) the fp64 oracle (pnp_ref.pnp_shell) through compare_records at the stated tolerances, and its reprojection
      error at ORACLE_REPROJ_REL;
  (c) cv2.solvePnPGeneric (ITERATIVE for >= 6 points, EPNP for 4 - 5) at the 1e-6 bar of tests/test_pose_core_host.py
      on converged, well-posed detections (noise-free targets; cv2's reprojection error < 1e-3 px, the fp32 rounding
      of the decoded map coordinates).

Where the problem itself does not fix one answer, only validity is asserted: EPnP on 4 points or on 5 noisy points has a
degenerate null space whose basis the Jacobi order picks (DESIGN.md section 5), and degenerate point sets (all points
equal, collinear points, a cuboid collapsed onto a line; `free` in the scene) have no unique pose.  There a pose is
produced and the median reprojection error stays within EPNP_RATIO of both cv2's and the host's.

The tracker's second PnP (tracker.cu: solve_and_shell_warp_v on the filtered keypoints, vertices from the fp64 pooled
scale) is scored the same way against the host build of track_core.h (test_tracker_second_pnp_matches_host).

The bars of (a) were set from a run on one H100 80GB HBM3; the worst value per class is in the comment above HOST_BAR."""
import collections
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from oracle import pnp_ref
from tests import pnp_scenes as ps
from tests.test_track_core_host import track_host  # noqa: F401  (fixture)
from tests.util import compare_records

pytestmark = pytest.mark.gpu

dp = ctypes.POINTER(ctypes.c_double)
fp = ctypes.POINTER(ctypes.c_float)

# (a) device vs the host build of pose_core.h, on detections with a pose (OK / INVISIBLE) or a projection (BEHIND):
#   quat      max |q_dev - q_host|, sign-aligned
#   loc_rel   max |t_dev - t_host| / |t_host|
#   kps3d_rel max |kps_3d_cam_dev - kps_3d_cam_host| / max(|t_host|, max |kps_3d_cam_host|)
#   proj_rel  max |proj_dev - proj_host| / max(1, max |proj_host|)  (pixels)
#   kps_pnp   max |kps_pnp_dev - kps_pnp_host| / max(1, max |kps_pnp_host|)
#   reproj    |reproj_dev - reproj_host| / (reproj_host + 1 px)
# The device writes fp32 records, so the floor of every relative field is fp32 rounding (6e-8).  Measured on one
# H100 80GB HBM3 (700 W), worst field per class: point_count 5.5e-8, mixed 5.9e-8, depth 5.5e-8, shape 5.6e-8,
# nonfinite 3.9e-8, rotation 5.1e-8, noise 5.7e-8, camera 5.3e-8, gates 8.0e-8, tracker 3.7e-9 (its host reference
# writes the same fp32 record); the reproj of consistent 5-point EPnP, which has no LM polish, is 4.5e-7 (gates class),
# hence EPNP_REPROJ_BAR.  Worst against the oracle: reproj 4.9e-7 of reproj + 1 px.
# The bite, on builds with one change each (every test of this file):
#   DLT moment weight of one block wrong       11 tests fail (every class, the tracker)
#   EPnP below 5 points in the decode path     point_count, gates
#   EPnP below 5 points in the tracker path    the tracker test
#   no identity start of V in the EPnP Jacobi  point_count, mixed, gates, scratch reuse, the tracker test
#   the visibility gate at `nv > thr`          depth, shape, gates, gate thresholds, the tracker test
#   19 LM iterations                           shape, noise, gates
#   points rounded to fp32 before the PnP      camera only: in the 600 x 800 frame (a = 6.25, tx = -100); at 512 x 512
#                                              a = 4 and tx = 0 make the fp32 rounding exact
#   not caught: the Jacobi stopping at off <= 1e-20 diag (the LM start moves, its minimum does not, and EPnP's shift
#   stays below the fp32 record), and `t[2] <= 0` for `t[2] < 0` (no scene reaches t[2] == 0 exactly).
HOST_BAR = {"quat": 3e-7, "loc_rel": 3e-7, "proj_rel": 3e-7, "kps3d_rel": 3e-7, "kps_pnp": 3e-7, "reproj": 3e-7}
EPNP_REPROJ_BAR = 2e-6      # reproj of 4 - 5 point EPnP (no LM polish): the Jacobi order's eigenvector rounding
CV2_BAR = 1e-6
ORACLE_REPROJ_REL = 1e-4    # |reproj_dev - reproj_oracle| / (reproj_oracle + 1 px), the stated 1e-4 of a relative field
EPNP_RATIO = 1.5            # median (reproj + 0.5 px) ratio, as tests/test_pose_core_host.py bounds degenerate EPnP


def _host(Lh, pts, scale, cam, w, h, vis, ocv):
    pts = np.ascontiguousarray(pts, np.float64)
    scale = np.ascontiguousarray(scale, np.float32)
    cam = np.ascontiguousarray(cam, np.float64)
    out = np.zeros(80)
    st, npt = ctypes.c_int(), ctypes.c_int()
    Lh.host_solve_and_shell(pts.ctypes.data_as(dp), ctypes.c_int(pts.shape[0]), scale.ctypes.data_as(fp),
                            cam.ctypes.data_as(dp), ctypes.c_double(w), ctypes.c_double(h), vis, ocv,
                            out.ctypes.data_as(dp), ctypes.byref(st), ctypes.byref(npt))
    return st.value, npt.value, out


def _device(sc):
    prm = cpb.decode_params(None, **sc.decode_kwargs())
    heads = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in sc.heads.items()}
    meta = cpb.make_meta(sc.B, sc.c, sc.s, sc.img_w, sc.img_h, sc.cam)
    dets, poses, n_valid = cpb.decode_pnp(heads, meta, prm, want_dets=True)
    torch.cuda.synchronize()
    return dets.cpu().numpy(), poses.cpu().numpy(), n_valid.cpu().numpy()


def _pnp_fields(r):
    return r[L.P_STATUS:L.P_NPTS + 1], r[L.P_LOCATION:L.P_KPS_PNP + 18]


def _cv2_pose(cv2, X, uv, cam, ocv):
    flags = cv2.SOLVEPNP_ITERATIVE if len(X) >= 6 else cv2.SOLVEPNP_EPNP
    ok, rv, tv, err = cv2.solvePnPGeneric(X, uv, cam, np.zeros(4), flags=flags)
    if not ok:
        return None
    R, t = pnp_ref.rodrigues(rv[0].reshape(3)), tv[0].reshape(3)
    if t[2] < 0:
        return None
    if not ocv:
        R, t = ps.M_GL @ R, ps.M_GL @ t
    return pnp_ref.mat_to_quat(R), t, float(err.reshape(-1)[0])


def _qdiff(a, b):
    if np.dot(a, b) < 0:
        b = -b
    return float(np.abs(a - b).max())


def _free(o, n):
    """No unique answer: EPnP with a degenerate null space (4 points, or 5 inconsistent ones), or a point / vertex set
    the scene marks degenerate."""
    return bool(o.get("free")) or n == 4 or (n == 5 and (o.get("noise", 0) > 0 or bool(o.get("loose"))))


def _pose_fields(r):
    """The PnP fields of a pose or track record as fp64 arrays."""
    r = np.asarray(r, np.float64)
    return {"loc": r[L.P_LOCATION:L.P_LOCATION + 3], "quat": r[L.P_QUAT:L.P_QUAT + 4], "reproj": r[L.P_REPROJ],
            "proj": r[L.P_PROJ_CUBOID:L.P_PROJ_CUBOID + 16], "kps3d": r[L.P_KPS_3D_CAM:L.P_KPS_3D_CAM + 27],
            "kpspnp": r[L.P_KPS_PNP:L.P_KPS_PNP + 18]}


def _host_fields(out):
    return {"loc": out[0:3], "quat": out[3:7], "reproj": out[7], "proj": out[8:24], "kps3d": out[24:51],
            "kpspnp": out[51:69]}


def _gaps(dev, ref, has_pose):
    """The HOST_BAR measures of device fields `dev` against reference fields `ref` (dicts of _pose_fields)."""
    e = {"proj_rel": np.abs(dev["proj"] - ref["proj"]).max() / max(1.0, np.abs(ref["proj"]).max()),
         "reproj": abs(dev["reproj"] - ref["reproj"]) / (ref["reproj"] + 1.0)}
    if has_pose:
        tn = np.linalg.norm(ref["loc"])
        e["quat"] = _qdiff(ref["quat"], dev["quat"])
        e["loc_rel"] = np.abs(dev["loc"] - ref["loc"]).max() / tn
        e["kps3d_rel"] = np.abs(dev["kps3d"] - ref["kps3d"]).max() / max(tn, np.abs(ref["kps3d"]).max())
        e["kps_pnp"] = np.abs(dev["kpspnp"] - ref["kpspnp"]).max() / max(1.0, np.abs(ref["kpspnp"]).max())
    return e


def _check_gaps(e, n, worst, prefix, what):
    for key, v in e.items():
        worst[prefix + key] = max(worst[prefix + key], v)
        bar = EPNP_REPROJ_BAR if key == "reproj" and n < 6 else HOST_BAR[key]
        assert v <= bar, what + (key, v)


def _score_scene(sc, dets, poses, n_valid, pose_host, cv2):
    """Every detection of a scene against (a), (b), (c).  Returns (worst dict, counts Counter, rows)."""
    worst = collections.defaultdict(float)
    cnt = collections.Counter()
    rows = []
    ratios, ratios_host = [], []
    for b in range(sc.B):
        assert n_valid[b] == len(sc.objs[b]), (sc.name, b, n_valid[b])
        got, want = [], []
        for i, o in enumerate(sc.objs[b]):
            rec = poses[b, i].astype(np.float64)
            k = int(rec[L.P_SRC_INDEX])
            assert k == i, (sc.name, b, i, k)
            pts = ps.used_points(dets[b, k], sc.rep_mode, sc.c, sc.s, sc.out_w, sc.out_h, L)
            # the image points of the record are the kernel's aff * x + tx, rounded to fp32: bit-equal to the oracle's
            kps = ps.decode_ref.map_to_image(dets[b, k, L.D_KPS:L.D_KPS + 16], sc.c, sc.s, sc.out_w, sc.out_h)
            assert np.array_equal(poses[b, i, L.P_KPS:L.P_KPS + 16], kps.reshape(-1).astype(np.float32),
                                  equal_nan=True), (sc.name, i)
            scale = dets[b, k, L.D_OBJ_SCALE:L.D_OBJ_SCALE + 3].copy()
            st = int(rec[L.P_STATUS])
            n = int(rec[L.P_NPTS])
            # (a) host
            st_h, n_h, out = _host(pose_host, pts, scale, sc.cam, sc.img_w, sc.img_h, sc.visible_thresh, sc.opencv_return)
            free = _free(o, n)
            assert n == n_h == ps.n_valid_points(pts), (sc.name, i, o["tag"], n, n_h)
            if o.get("npts") is not None:
                assert n == o["npts"], (sc.name, i, o["tag"], n)
            if o["want"] is not None:
                assert st in o["want"], (sc.name, i, o["tag"], st)
            cnt["dev==host"] += st == st_h
            cnt["n"] += 1
            if not free:
                assert st == st_h, (sc.name, i, o["tag"], st, st_h)
            # no pose with a NaN or inf in it
            if st in ps.HAS_POSE:
                assert np.isfinite(rec[L.P_LOCATION:L.P_KPS_PNP + 18]).all(), (sc.name, i, o["tag"])
            if st == st_h and st in ps.HAS_POSE + (ps.BEHIND,) and not free:
                _check_gaps(_gaps(_pose_fields(rec), _host_fields(out), st != ps.BEHIND), n, worst, "host_",
                            (sc.name, i, o["tag"]))
            if free and n in (4, 5) and st in ps.HAS_POSE and st_h in ps.HAS_POSE:
                ratios_host.append((rec[L.P_REPROJ] + 0.5) / (out[7] + 0.5))
            # (b) oracle
            det = {"obj_scale": scale, "kps": pts[::sc.n_in // 8].reshape(-1)}
            with np.errstate(all="ignore"):
                st_o, _ = pnp_ref.pnp_shell(det, pts, sc.cam, sc.img_w, sc.img_h, category=ps.VISIBLE[sc.visible_thresh],
                                            opencv_return=bool(sc.opencv_return))
            cnt["dev==oracle"] += st == st_o
            w = rec.copy()
            w[L.P_STATUS] = st_o
            if "location" in det and st_o in ps.HAS_POSE:
                w[L.P_LOCATION:L.P_LOCATION + 3] = det["location"]
                w[L.P_QUAT:L.P_QUAT + 4] = det["quaternion_xyzw"]
                w[L.P_PROJ_CUBOID:L.P_PROJ_CUBOID + 16] = np.asarray(det["projected_cuboid"]).reshape(-1)
                w[L.P_KPS_3D_CAM:L.P_KPS_3D_CAM + 27] = np.asarray(det["kps_3d_cam"]).reshape(-1)
                w[L.P_KPS_PNP:L.P_KPS_PNP + 18] = np.asarray(det["kps_pnp"]).reshape(-1)
            if not free:
                assert st == st_o, (sc.name, i, o["tag"], st, st_o)
            if not free and np.isfinite(rec[:L.P_LOCATION]).all():      # non-finite inputs: status only
                if "location" in det and st_o in ps.HAS_POSE:
                    dr = abs(rec[L.P_REPROJ] - det["reproj_err"]) / (det["reproj_err"] + 1.0)
                    worst["oracle_reproj"] = max(worst["oracle_reproj"], dr)
                    assert dr <= ORACLE_REPROJ_REL, (sc.name, i, o["tag"], dr)
                got.append(rec)
                want.append(w)
            # (c) cv2
            ok = ~((pts[:, 0] < -5000) | (pts[:, 1] < -5000))
            with np.errstate(all="ignore"):
                V = pnp_ref.cuboid_vertices(scale)
            if cv2 is not None and n >= 4 and np.isfinite(pts[ok]).all() and np.isfinite(V).all():
                X = np.array([V[j // (sc.n_in // 8)] for j in range(sc.n_in)])[ok]
                cvp = _cv2_pose(cv2, X, pts[ok], sc.cam, sc.opencv_return)
                if cvp is not None and st in ps.HAS_POSE:
                    if free and n in (4, 5):
                        ratios.append((rec[L.P_REPROJ] + 0.5) / (cvp[2] + 0.5))
                    elif o.get("noise", 0) == 0 and not o.get("loose") and cvp[2] < 1e-3 and not free:
                        dq = _qdiff(cvp[0], rec[L.P_QUAT:L.P_QUAT + 4])
                        dl = np.abs(rec[L.P_LOCATION:L.P_LOCATION + 3] - cvp[1]).max() / np.linalg.norm(cvp[1])
                        worst["cv2_quat"] = max(worst["cv2_quat"], dq)
                        worst["cv2_loc_rel"] = max(worst["cv2_loc_rel"], dl)
                        cnt["cv2_compared"] += 1
                        assert dq <= CV2_BAR and dl <= CV2_BAR, (sc.name, i, o["tag"], dq, dl)
            rows.append((b, i, st, n, o["tag"]))
        if got:
            err = compare_records(np.stack(got), np.stack(want), L)
            for key in ("quat", "loc_rel", "proj_px", "kps3d_rel", "kps_pnp"):
                worst["oracle_" + key] = max(worst["oracle_" + key], err.get(key, 0.0))
    for key, r in (("epnp_ratio_cv2", ratios), ("epnp_ratio_host", ratios_host)):
        if r:
            worst[key] = max(worst[key], float(np.median(r)))
            assert np.median(r) <= EPNP_RATIO, (sc.name, key, np.median(r))
    return worst, cnt, rows


@pytest.fixture(scope="module")
def results(cplib, pose_host):
    try:
        import cv2
    except ImportError:      # pragma: no cover
        cv2 = None
    out = {}
    for cls in ps.CLASSES:
        for sc in ps.BUILDERS[cls]():
            dets, poses, n_valid = _device(sc)
            out[sc.name] = (sc, dets, poses, n_valid)
    return out, pose_host, cv2


def _report(cls, worst, cnt, statuses):
    keys = sorted(worst)
    print("\n[pnp %s] %s  statuses %s  agree: host %d/%d oracle %d/%d  cv2 compared %d" % (
        cls, "  ".join("%s %.2e" % (k, worst[k]) for k in keys), dict(sorted(statuses.items())), cnt["dev==host"],
        cnt["n"], cnt["dev==oracle"], cnt["n"], cnt["cv2_compared"]))


@pytest.mark.parametrize("cls", ps.CLASSES)
def test_class_matches_host_oracle_cv2(cls, results):
    res, pose_host, cv2 = results
    worst = collections.defaultdict(float)
    cnt = collections.Counter()
    statuses = collections.Counter()
    for name, (sc, dets, poses, n_valid) in res.items():
        if sc.cls != cls:
            continue
        w, c, rows = _score_scene(sc, dets, poses, n_valid, pose_host, cv2)
        for k, v in w.items():
            worst[k] = max(worst[k], v)
        cnt.update(c)
        statuses.update((st, n) for _, _, st, n, _ in rows)
    _report(cls, worst, cnt, statuses)
    # coverage: what each class exists to reach
    need = {
        "point_count": [(ps.FEW_POINTS, 3)] + [(s, n) for n in (4, 5, 6, 7, 8, 16) for s in (ps.OK,)],
        "depth": [(ps.BEHIND, 8), (ps.OK, 8), (ps.INVISIBLE, 8)],
        "nonfinite": [(ps.SOLVER_FAIL, 8)],
        "gates": [(ps.OK, 8), (ps.INVISIBLE, 8), (ps.OK, 7), (ps.OK, 5)],
        "rotation": [(ps.OK, 8)], "shape": [(ps.OK, 8)], "noise": [(ps.OK, 8), (ps.OK, 16)], "camera": [(ps.OK, 8)],
        "mixed": [(ps.OK, n) for n in (4, 5, 6, 7, 8)], "degenerate": [],
    }[cls]
    missing = [k for k in need if statuses[k] == 0]
    assert not missing, (cls, missing, dict(statuses))
    assert sum(statuses.values()) > 0


def test_gate_thresholds_reached(results):
    """Each visible_thresh scene has detections at thr - 1 and thr points outside the frame, with the intended
    statuses (asserted per detection above); the centre gate has both sides of every border it tests."""
    res, _, _ = results
    for thr in (3, 6):
        sc, dets, poses, n_valid = res["visible_%d" % thr]
        got = collections.Counter((o["tag"], int(poses[0, i, L.P_STATUS])) for i, o in enumerate(sc.objs[0]))
        assert got[("thr %d nv %d" % (thr, thr - 1), ps.OK)] >= 3 and got[("thr %d nv %d" % (thr, thr), ps.INVISIBLE)] >= 3
    sc, dets, poses, n_valid = res["centre"]
    assert sorted(int(v) for v in poses[0, :4, L.P_STATUS]) == [ps.OK, ps.OK, ps.INVISIBLE, ps.INVISIBLE]


def test_scratch_reuse_is_invisible(cplib):
    """Each warp of group_pose_kernel solves detections w, w + 8, ... in one PNP_SCRATCH region, alternating between
    EPnP and DLT + LM in the mixed scenes.  Every record equals, bit for bit, the record of the same detection solved
    alone in its own image (same cell, same map, so the same fp32 keypoints and fp64 points)."""
    for sc in ps.scenes_mixed():
        dets, poses, n_valid = _device(sc)
        solo, index = ps.solo_scene(sc)
        d1, p1, n1 = _device(solo)
        assert (n1 == 1).all()
        for k, (b, i) in enumerate(index):
            a_st, a_f = _pnp_fields(poses[b, i])
            b_st, b_f = _pnp_fields(p1[k, 0])
            assert np.array_equal(a_st, b_st) and np.array_equal(a_f.view(np.uint32), b_f.view(np.uint32)), (sc.name, b, i)


def test_no_nonfinite_pose(results):
    """No OK / INVISIBLE record of any scene holds a NaN or inf; non-finite points or cuboid vertices end in
    SOLVER_FAIL on the device, in the host build and in the oracle (DESIGN.md section 5)."""
    res, pose_host, _ = results
    for name, (sc, dets, poses, n_valid) in res.items():
        for b in range(sc.B):
            for i in range(n_valid[b]):
                r = poses[b, i]
                if int(r[L.P_STATUS]) in ps.HAS_POSE:
                    assert np.isfinite(r[L.P_LOCATION:L.P_KPS_PNP + 18]).all(), (name, b, i)
    sc, dets, poses, n_valid = res["nonfinite"]
    for i, o in enumerate(sc.objs[0]):
        with np.errstate(all="ignore"):
            V = pnp_ref.cuboid_vertices(dets[0, i, L.D_OBJ_SCALE:L.D_OBJ_SCALE + 3])
        pts = ps.used_points(dets[0, i], 0, sc.c, sc.s, sc.out_w, sc.out_h, L)
        ok = ~((pts[:, 0] < -5000) | (pts[:, 1] < -5000))
        if not (np.isfinite(V).all() and np.isfinite(pts[ok]).all()):
            assert int(poses[0, i, L.P_STATUS]) == ps.SOLVER_FAIL, o["tag"]


def test_tracker_second_pnp_matches_host(cplib, pose_host, track_host):
    """The tracker's second PnP (tracker.cu steps 5 - 6: solve_and_shell_warp_v on the filtered keypoints, vertices from
    the fp64 pooled scale) against the host build of track_core.h + pose_core.h on the same records.  Fresh streams take
    the detections of ps.track_objs as their first frame; keypoints whose filter confidence is below 0.15 reach the PnP
    as -10000, so 3 - 8 points survive.  The host harness runs the same read-out in fp64, so the comparison is at
    HOST_BAR, not at the stated tolerances."""
    import json
    from tests.test_gpu_tracker import _opt_from_gold
    from tests.test_track_core_host import GOLD
    gold = json.load(open(GOLD))
    o = gold["opt"]
    assert o["kalman"] and o["scale_pool"] and o["use_pnp"] and o["hps_uncertainty"] and list(o["conf_border"]) == [3, 9]
    opt = _opt_from_gold(o)
    objs, cam = ps.track_objs()
    S, K = len(objs), max(len(r) for r in objs)
    recs = np.zeros((S, K, L.CP_POSE_RECORD), np.float32)
    for s, row in enumerate(objs):
        for i, d in enumerate(row):
            recs[s, i] = ps.track_record(d["pts"], d["keep"], d["scale"], 0.9 - 0.01 * i, L)
    trk = cpb.Tracker(opt, streams=S)
    meta = cpb.make_meta(S, np.array([256., 256.], np.float32), 512.0, 512, 512, cam).cuda()
    nv = torch.full((S,), K, dtype=torch.int32).cuda()
    tr, n = trk.step_records(torch.from_numpy(recs).cuda(), nv, meta)
    tr, n = tr.cpu().numpy(), n.cpu().numpy()
    vis = ps.VISIBLE_OF[o["c"]]
    worst = collections.defaultdict(float)
    reached = collections.Counter()
    ratios = []
    agree = 0
    for s, row in enumerate(objs):
        h = track_host.trk_create(1, 1, 1, 1, int(o["max_age"]), float(o["new_thresh"]), float(o["R"]), 3.0, 9.0, vis,
                                  int(o["show_axes"]), 128)
        out = np.zeros((128, L.CP_TRACK_RECORD), np.float32)
        rs = np.ascontiguousarray(recs[s])
        cam64 = np.ascontiguousarray(cam, np.float64)
        nh = track_host.trk_step(h, rs.ctypes.data_as(ctypes.c_void_p), K, cam64.ctypes.data_as(ctypes.c_void_p), 512.0,
                                 512.0, out.ctypes.data_as(ctypes.c_void_p))
        track_host.trk_destroy(h)
        assert int(n[s]) == nh == len(row)
        for i, d in enumerate(row):
            dev, ref = tr[s, i].astype(np.float64), out[i].astype(np.float64)
            what = (s, i, d["tag"])
            assert dev[L.T_ID] == ref[L.T_ID] == i + 1, what
            # the read-out the PnP sees: the fp32 point where kept, -10000 where the confidence is below 0.15
            kf = dev[L.T_KPS_MEAN_KF:L.T_KPS_MEAN_KF + 16].reshape(8, 2)
            want = np.where(d["keep"][:, None], d["pts"].astype(np.float64), -10000.0)
            assert np.array_equal(kf, want), what
            assert abs(dev[L.T_CONF_AVG] - ref[L.T_CONF_AVG]) <= 1e-6, what
            st, st_h = int(dev[L.T_PNP2_STATUS]), int(ref[L.T_PNP2_STATUS])
            agree += st == st_h
            free = _free(d, d["npts"])
            if not free:
                assert st == st_h, what + (st, st_h)
            if st in ps.HAS_POSE:
                assert int(dev[L.P_NPTS]) == d["npts"], what
                assert np.isfinite(dev[L.P_LOCATION:L.P_KPS_PNP + 18]).all(), what
            if st == st_h and st in ps.HAS_POSE and not free:
                _check_gaps(_gaps(_pose_fields(dev), _pose_fields(ref), True), d["npts"], worst, "host_", what)
                if st == ps.OK:
                    for off, m in ((L.T_KPS_PNP_KF, 18), (L.T_KPS_3D_CAM_KF, 27)):
                        a, b = dev[off:off + m], ref[off:off + m]
                        g = np.abs(a - b).max() / max(1.0, np.abs(b).max())
                        worst["host_kf_fields"] = max(worst["host_kf_fields"], g)
                        assert g <= HOST_BAR["kps_pnp"], what + (off, g)
                assert dev[L.T_IN_BOXES] == ref[L.T_IN_BOXES], what
            if free and st in ps.HAS_POSE and st_h in ps.HAS_POSE:
                ratios.append((dev[L.P_REPROJ] + 0.5) / (ref[L.P_REPROJ] + 0.5))
            reached[(st, d["npts"])] += 1
    if ratios:
        worst["epnp_ratio_host"] = float(np.median(ratios))
        assert np.median(ratios) <= EPNP_RATIO, np.median(ratios)
    total = sum(reached.values())
    print("\n[pnp tracker] %s  statuses %s  agree: host %d/%d" % (
        "  ".join("%s %.2e" % (k, worst[k]) for k in sorted(worst)), dict(sorted(reached.items())), agree, total))
    need = [(ps.FEW_POINTS, 3)] + [(ps.OK, k) for k in (4, 5, 6, 7, 8)]
    missing = [k for k in need if reached[k] == 0]
    assert not missing, (missing, dict(reached))
