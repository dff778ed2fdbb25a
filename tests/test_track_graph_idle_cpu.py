"""The tracking graphs with idle slots, without a GPU: cp_preprocess_slots_rows_dev, cp_gather_rows_dev,
cp_tracker_render_dev2 and cp_tracker_step_dev are declared, exported and bound with their documented signatures and
refuse bad arguments with CP_ERR_INVALID before touching the device; TrackGraph and MultiCategoryTrackGraph built with
idle_slots=True refuse pre_dets, the ground-truth heat maps and multi-scale with the messages of the default graphs; the
control block of a step maps rows, tracker streams and slots as run_batch(list, track=True) orders them."""
import ctypes
import os

import numpy as np
import pytest

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from tests.test_track_graph_cpu import _header, _shell
from tests.test_track_graph_multi_cpu import _multi_shell
from tests.util import ROOT

INVALID = -1      # CP_ERR_INVALID
SIGNATURES = {
    "cp_preprocess_slots_rows_dev": "int cp_preprocess_slots_rows_dev(const uint8_t* frames, const void* table, "
                                    "int32_t format, const int32_t* rows, int32_t B, int32_t dst_h, int32_t dst_w, "
                                    "const float mean[3], const float std[3], const int32_t* start, float* store, "
                                    "float* out, float* prev, void* stream);",
    "cp_gather_rows_dev": "int cp_gather_rows_dev(const void* src, void* dst, int64_t row_bytes, int32_t n, "
                          "const int32_t* map, void* stream);",
    "cp_tracker_render_dev2": "int cp_tracker_render_dev2(cp_tracker* trk, int32_t batch, const int32_t* stream_ids, "
                              "const double* meta, const double* trans_input, int32_t inp_h, int32_t inp_w, "
                              "const int32_t* modes, float* pre_hm, float* pre_hm_hp, void* stream);",
    "cp_tracker_step_dev": "int cp_tracker_step_dev(cp_tracker* trk, int32_t batch, const int32_t* stream_ids, "
                           "const float* poses, const int32_t* n_valid, int32_t K, const double* meta, "
                           "float* tracks_out, int32_t* n_tracks, void* stream);",
}


def test_entry_points_declared_exported_and_bound(cplib):
    hdr = _header()
    for name, sig in SIGNATURES.items():
        assert sig in hdr, name
        assert name in _lib.EXPORTS and hasattr(cplib, name)
        assert len(getattr(cplib, name).argtypes) == sig.count(",") + 1, name
        assert getattr(cplib, name).restype is ctypes.c_int, name
    # the device maps are read unchecked: the header says so where each is declared
    raw = open(os.path.join(ROOT, "include", "centerpose_b200.h")).read()
    for name in SIGNATURES:
        doc = raw[:raw.index("int %s(" % name)].rsplit("*/", 2)[-2]
        assert "WITHOUT checking" in doc, name


def _err(cplib):
    return cplib.cp_last_error()


def _rows(cplib, fmt=_lib.CP_PIX_BGR, B=2, dh=512, dw=512, frames=8, table=8, rows=8, out=8, start=8, store=8, prev=8,
          mean=True, std=True):
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4) if mean else None
    s = (ctypes.c_float * 3)(0.3, 0.3, 0.3) if std else None
    p = ctypes.c_void_p
    return cplib.cp_preprocess_slots_rows_dev(p(frames), p(table), fmt, p(rows), B, dh, dw, m, s, p(start), p(store),
                                              p(out), p(prev), None)


def test_slots_rows_validates_its_arguments(cplib):
    for kw in ({"frames": 0}, {"table": 0}, {"rows": 0}, {"out": 0}, {"mean": False}, {"std": False}):
        assert _rows(cplib, **kw) == INVALID and b"null argument" in _err(cplib), kw
    for kw in ({"store": 0}, {"prev": 0}):
        assert _rows(cplib, **kw) == INVALID and b"store and prev go together" in _err(cplib), kw
    for fmt in (-1, 3, 7):
        assert _rows(cplib, fmt=fmt) == INVALID and b"unknown pixel format %d" % fmt in _err(cplib)
    for kw in ({"B": 0}, {"B": -3}, {"dh": 0}, {"dw": -1}):
        assert _rows(cplib, **kw) == INVALID and b"bad shape" in _err(cplib), kw
    assert b"cp_preprocess_slots_rows_dev" in _err(cplib)


def test_gather_rows_validates_its_arguments(cplib):
    p = ctypes.c_void_p
    for args in ((0, 8, 8), (8, 0, 8), (8, 8, 0)):
        assert cplib.cp_gather_rows_dev(p(args[0]), p(args[1]), 16, 2, p(args[2]), None) == INVALID
        assert b"cp_gather_rows_dev: null argument" in _err(cplib), args
    for row_bytes, n in ((0, 2), (-4, 2), (6, 2), (16, 0), (16, -1)):
        assert cplib.cp_gather_rows_dev(p(8), p(8), row_bytes, n, p(8), None) == INVALID
        assert b"cp_gather_rows_dev: bad shape" in _err(cplib), (row_bytes, n)


def test_tracker_dev2_entries_validate_their_arguments(cplib):
    p = ctypes.c_void_p
    assert cplib.cp_tracker_render_dev2(None, 1, p(8), p(8), p(8), 64, 64, None, p(8), p(8), None) == INVALID
    assert b"cp_tracker_render: null argument" in _err(cplib)
    assert cplib.cp_tracker_step_dev(None, 1, p(8), p(8), p(8), 4, p(8), p(8), p(8), None) == INVALID
    assert b"cp_tracker_step: null argument" in _err(cplib)


# ---- the graphs' refusals with idle slots (all raised before any device work) ------------------------------------------
@pytest.mark.parametrize("over, exc, msg", [
    ({"test_scales": [1.0, 0.5]}, NotImplementedError, r"test_scales=\[1\]"),
    ({"gt_pre_hm_hmhp": True}, NotImplementedError, r"ground-truth heat maps .* run through (MultiCategoryTracker\.)?"
                                                    r"run_batch"),
    ({"gt_pre_hm_hmhp_first": True}, NotImplementedError, r"ground-truth heat maps"),
])
def test_idle_graph_refuses_options(over, exc, msg):
    with pytest.raises(exc, match=msg):
        cpb.TrackGraph(_shell(**over), slots=2, frame_hw=(480, 640), camera_matrix=None, idle_slots=True)
    det = _multi_shell()
    for k, v in over.items():
        setattr(det.opt, k, v)
    with pytest.raises(exc, match=msg):
        cpb.MultiCategoryTrackGraph(det, slots=2, frame_hw=[(480, 640), (720, 1280)], camera_matrix=None,
                                    idle_slots=True)


def _built_shell(cls=cpb.TrackGraph, S=3, M=1):
    """A graph object with the host state of one built with idle_slots=True (no device buffers)."""
    g = cls.__new__(cls)
    g.idle_slots, g.per_slot, g.slots, g.streams = True, False, S, M * S
    g.frame_hw, g.frame_shape, g.pixel_format = (480, 640), (S, 480, 640, 3), "bgr"
    g._slot_hw, g._slot_shapes = [(480, 640)] * S, [(480, 640, 3)] * S
    g._fresh, g._started = True, [False] * S
    return g


@pytest.mark.parametrize("cls, msg", [(cpb.TrackGraph, "pre_dets seeding runs through run_batch"),
                                      (cpb.MultiCategoryTrackGraph, "pre_dets seeding runs through "
                                                                    "MultiCategoryTracker.run_batch")])
def test_idle_graph_refuses_pre_dets(cls, msg):
    with pytest.raises(NotImplementedError, match=msg):
        _built_shell(cls)([None, None, None], pre_dets=[[], [], []])


def test_idle_graph_checks_the_frames_of_a_call():
    g = _built_shell()
    with pytest.raises(ValueError, match=r"frames is a list of 3 frames \(None for an idle slot\) or one uint8 "
                                         r"\[3, 480, 640, 3\] array, got dict"):
        g({})
    with pytest.raises(ValueError, match=r"frames must be uint8 \[3, 480, 640, 3\] \(bgr\), got torch.uint8 "
                                         r"\(2, 480, 640, 3\)"):
        g(np.zeros((2, 480, 640, 3), np.uint8))
    with pytest.raises(ValueError, match="built with idle slots: frames is a list of 3 frames, got 2 frames"):
        g([None, None])
    with pytest.raises(ValueError, match=r"slot 2 takes uint8 \[480, 640, 3\] frames \(bgr, frame_hw \(480, 640\)\)"):
        g([None, None, np.zeros((480, 641, 3), np.uint8)])
    with pytest.raises(ValueError, match="2 new_video entries for 3 slots"):
        g([None, None, None], new_video=[True, False])


@pytest.mark.parametrize("M", [1, 3])
def test_control_block_orders_rows_as_run_batch(M):
    """rows: the live slots in slot order (run_batch(list)'s batch); ids: stream m * S + slot of row m * n + k (its
    tracker rows); inv: the row of each stream, -1 for an idle slot; start tiled per category."""
    S = 4
    g = _built_shell(S=S, M=M)
    live, start = [1, 3], np.array([0, 1, 0, 0], np.int32)
    c = g._control(live, start)
    MS = M * S
    assert c.dtype == np.int32 and c.shape == (3 * MS + S,)
    assert list(c[:MS]) == list(np.tile(start, M))
    assert list(c[MS:MS + 2]) == live
    ids = c[MS + S:2 * MS + S][:M * 2]
    assert list(ids) == [m * S + i for m in range(M) for i in live]
    inv = c[2 * MS + S:]
    for m in range(M):
        for s in range(S):
            want = m * 2 + live.index(s) if s in live else -1
            assert inv[m * S + s] == want, (m, s)
