"""CPU tests of the ground-truth seeding and the optimal association in centerpose_b200/csrc/track_core.h (compiled for
the host by tests/host/track_gt_host.cpp): the solver core returns the pairs scipy.optimize.linear_sum_assignment returns,
ties included, and a serial replay reproduces what the unmodified reference tracker produced on the seeded sequences
(tests/golden/tracker_seq_{gt_first,gt_every,hungarian}.json, oracle/make_golden_tracker_gt.py)."""
import ctypes
import json
import os
import subprocess
import types

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

from centerpose_b200 import _lib as L
from centerpose_b200.tracker import seed_records
from oracle import make_golden_tracker as mg
from oracle import make_golden_tracker_gt as mgt
from tests.test_track_core_host import VISIBLE, compare_to_golden, det_to_record, summarize_tracks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def gt_host():
    src = os.path.join(ROOT, "tests", "host", "track_gt_host.cpp")
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    so = os.path.join(out_dir, "libtrack_gt_host.so")
    hdrs = [os.path.join(ROOT, "centerpose_b200", "csrc", h) for h in ("track_core.h", "pose_core.h")]
    hdrs.append(os.path.join(ROOT, "include", "centerpose_b200.h"))
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    vp, i32, f64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    lib.gth_create.restype = vp
    lib.gth_create.argtypes = [i32] * 5 + [f64] * 4 + [i32] * 4
    lib.gth_destroy.argtypes = [vp]
    lib.gth_seed.argtypes = [vp, vp, i32]
    lib.gth_step.argtypes = [vp, vp, i32, vp, f64, f64, vp]
    lib.gth_lsa.argtypes = [vp, i32, i32, vp, vp]
    return lib


def host_lsa(lib, cost):
    cost = np.ascontiguousarray(cost, np.float64)
    nr, nc = cost.shape
    rows = np.zeros(max(1, min(nr, nc)), np.int32)
    cols = np.zeros_like(rows)
    n = lib.gth_lsa(cost.ctypes.data_as(ctypes.c_void_p), nr, nc, rows.ctypes.data_as(ctypes.c_void_p),
                    cols.ctypes.data_as(ctypes.c_void_p))
    assert n >= 0
    return rows[:n], cols[:n]


def random_costs(rng, count):
    """Seeded matrices of sizes 0..40 both ways: continuous costs, small integers (many ties) and ~30 % 1e18 entries
    (the invalid pairs of the tracker's dist), plus the tracker's own mix of squared distances under 64 and 1e18."""
    for t in range(count):
        nr, nc = int(rng.integers(0, 41)), int(rng.integers(0, 41))
        kind = t % 4
        if kind == 0:
            c = rng.random((nr, nc)) * 100
        elif kind == 1:
            c = rng.integers(0, 4, size=(nr, nc)).astype(np.float64)
        elif kind == 2:
            c = rng.integers(0, 50, size=(nr, nc)).astype(np.float64)
            c[rng.random((nr, nc)) < 0.3] = 1e18
        else:
            c = (rng.random((nr, nc)) * 64).astype(np.float32).astype(np.float64)
            c[rng.random((nr, nc)) < 0.3] = 1e18
        yield c


def test_solver_matches_scipy_linear_sum_assignment(gt_host):
    rng = np.random.default_rng(2024)
    n = 0
    for c in random_costs(rng, 2400):
        r_want, c_want = linear_sum_assignment(c)
        r_got, c_got = host_lsa(gt_host, c)
        assert r_got.tolist() == r_want.tolist() and c_got.tolist() == c_want.tolist(), (c.shape, c.tolist())
        n += 1
    assert n == 2400


def replay(lib, name, pose_host):
    """The host build through one of the ground-truth / hungarian sequences -> (got, golden frames)."""
    gold = json.load(open(os.path.join(GOLDEN, "tracker_seq_%s.json" % name)))
    o = gold["opt"]
    opt = types.SimpleNamespace(kalman=o["kalman"], scale_pool=o["scale_pool"], use_pnp=o["use_pnp"])
    meta, frames0 = mg.make_sequence()
    frames = mgt.scenario_frames(name, frames0)
    seeds = mgt.seed_schedule(name, frames0)
    cam = np.ascontiguousarray(meta["camera_matrix"], np.float64)
    h = lib.gth_create(int(o["kalman"]), int(o["scale_pool"]), int(o["use_pnp"]), int(o["hps_uncertainty"]), int(o["max_age"]),
                       float(o["new_thresh"]), float(o["R"]), float(o["conf_border"][0]), float(o["conf_border"][1]),
                       int(o["hungarian"]), VISIBLE[o["c"]], int(o["show_axes"]), 128)
    out = np.zeros((128, L.CP_TRACK_RECORD), np.float32)
    got = []
    for f, dets in enumerate(frames):
        if seeds[f] is not None:
            rec = np.ascontiguousarray(seed_records(seeds[f], opt), np.float32)
            lib.gth_seed(h, rec.ctypes.data_as(ctypes.c_void_p), rec.shape[0])
        recs = np.stack([det_to_record(d, cam, meta["width"], meta["height"], pose_host, VISIBLE[o["c"]]) for d in dets])
        recs = np.ascontiguousarray(recs, np.float32)
        n = lib.gth_step(h, recs.ctypes.data_as(ctypes.c_void_p), recs.shape[0], cam.ctypes.data_as(ctypes.c_void_p),
                         float(meta["width"]), float(meta["height"]), out.ctypes.data_as(ctypes.c_void_p))
        got.append(summarize_tracks(out.copy(), n))
    lib.gth_destroy(h)
    return got, gold["frames"]


@pytest.mark.parametrize("name", mgt.SCENARIOS)
def test_host_replay_matches_reference_golden(name, gt_host, pose_host):
    got, want = replay(gt_host, name, pose_host)
    compare_to_golden(got, want)


def test_seed_records_name_missing_keys():
    opt = types.SimpleNamespace(kalman=True, scale_pool=True, use_pnp=True)
    meta, frames = mg.make_sequence()
    d = mgt.gt_list(frames[0])[0]
    rec = seed_records([d], opt)
    assert rec.shape == (1, L.CP_SEED_RECORD) and rec[0, L.S_HAS_KPS_GT] == 1 and rec[0, L.S_HAS_CT] == 0
    assert np.allclose(rec[0, L.S_KPS_GT:L.S_KPS_GT + 18], np.asarray(d["kps_gt"]).reshape(-1))
    for key in ("kps_fusion_std", "obj_scale_uncertainty", "score"):
        bad = dict(d)
        del bad[key]
        with pytest.raises(ValueError, match=key):
            seed_records([bad], opt)
