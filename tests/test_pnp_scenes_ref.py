"""The PnP edge scenes of tests/pnp_scenes.py decode, in the oracle, to what they were built for: the intended number
of valid points at the intended image positions (to fp32 rounding of the map coordinates) and a status of the intended
class.  This keeps the scenes of tests/test_gpu_pnp_edges.py honest without a GPU."""
import collections

import numpy as np
import pytest

from oracle import pnp_ref
from tests import pnp_scenes as ps


@pytest.mark.parametrize("cls", ps.CLASSES)
def test_scene_decodes_as_built(cls):
    reached = collections.Counter()
    for sc in ps.BUILDERS[cls]():
        for b in range(sc.B):
            res = ps.oracle_decode(sc, b)
            assert len(res) == len(sc.objs[b]), (sc.name, b, len(res))
            for i, (d, o) in enumerate(zip(res, sc.objs[b])):
                assert d["_k"] == i
                pts = pnp_ref.assemble_points(d, sc.rep_mode)
                assert o["npts"] is None or ps.n_valid_points(pts) == o["npts"], (sc.name, b, i, o["tag"])
                if not o.get("loose"):
                    want = np.asarray(o["pts"], np.float64)
                    fin = np.isfinite(want) & (want > -5000)
                    tol = 1e-6 * (np.abs(want[fin]) + 4 * max(sc.out_w, sc.out_h))
                    assert (np.abs(pts[fin] - want[fin]) <= tol).all(), (sc.name, i, o["tag"])
                    assert np.array_equal(np.isnan(pts), np.isnan(want)), (sc.name, i, o["tag"])
                    assert ((pts < -5000) == (want < -5000)).all(), (sc.name, i, o["tag"])
                with np.errstate(all="ignore"):
                    st, _ = pnp_ref.pnp_shell(dict(d), pts, sc.cam, sc.img_w, sc.img_h,
                                              category=ps.VISIBLE[sc.visible_thresh], opencv_return=bool(sc.opencv_return))
                if o["want"] is not None:
                    assert st in o["want"], (sc.name, i, o["tag"], st)
                reached[(st, ps.n_valid_points(pts))] += 1
    assert sum(reached.values()) > 0
    print(cls, dict(reached))


def test_mixed_scene_alternates_solvers_in_every_warp():
    """Warp w of group_pose_kernel (8 warps) solves detections w, w + 8, ...: in the mixed scenes each of those
    sequences alternates between EPnP (4 - 5 points) and DLT + LM (6 - 8 points)."""
    for sc in ps.scenes_mixed():
        for row in sc.objs:
            for w in range(8):
                epnp = [row[i]["npts"] < 6 for i in range(w, len(row), 8)]
                assert all(a != b for a, b in zip(epnp, epnp[1:])), (sc.name, w)


def test_solo_scene_keeps_the_cell_and_bits():
    sc = ps.scenes_mixed()[0]
    solo, index = ps.solo_scene(sc)
    cells = ps._cells(sc.out_h, sc.out_w, sc.K)
    for k, (b, i) in enumerate(index):
        cx, cy = cells[i]
        for name in sc.heads:
            assert np.array_equal(solo.heads[name][k, :, cy, cx], sc.heads[name][b, :, cy, cx])


def test_nonfinite_inputs_are_solver_failures():
    """A NaN / inf image point or cuboid vertex is SOLVER_FAIL in the oracle (cv2 asserts on such input)."""
    cv2 = pytest.importorskip("cv2")
    sc = ps.scenes_nonfinite()[0]
    for o in sc.objs[0]:
        with np.errstate(all="ignore"):
            V = pnp_ref.cuboid_vertices(o["scale"])
            sol = pnp_ref.solve_pnp(o["pts"], V, sc.cam)
        ok = np.all(o["pts"] > -5000, axis=1)
        finite = np.isfinite(V).all() and np.isfinite(o["pts"][ok]).all()
        if not finite:
            assert sol["status"] == ps.SOLVER_FAIL, o["tag"]
            with pytest.raises(cv2.error):
                cv2.solvePnPGeneric(V[ok], o["pts"][ok], sc.cam, np.zeros(4), flags=cv2.SOLVEPNP_ITERATIVE)
