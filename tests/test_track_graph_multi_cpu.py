"""The graph-safe ragged slot pre-process and the graphs over several categories and per-slot frame sizes, without a GPU:
cp_preprocess_frame_table_bytes, cp_preprocess_frame_table and cp_preprocess_slots_ragged_dev are declared, exported and
bound with their documented signatures and refuse bad arguments with CP_ERR_INVALID before touching the device;
TrackGraph and MultiCategoryTrackGraph refuse what they do not take before any device work."""
import ctypes

import numpy as np
import pytest

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.detector import MultiCategoryDetector, MultiCategoryTracker, ObjectPoseDetector
from tests.test_track_graph_cpu import _header

INVALID = -1      # CP_ERR_INVALID
SIGNATURES = {
    "cp_preprocess_frame_table_bytes": "int64_t cp_preprocess_frame_table_bytes(int32_t B);",
    "cp_preprocess_frame_table": "int cp_preprocess_frame_table(int64_t frames_bytes, const int64_t* offsets, "
                                 "const int32_t* src_hw, int32_t format, int32_t B, int32_t dst_h, int32_t dst_w, "
                                 "const double* trans_input, void* table, void* stream);",
    "cp_preprocess_slots_ragged_dev": "int cp_preprocess_slots_ragged_dev(const uint8_t* frames, const void* table, "
                                      "int32_t format, int32_t B, int32_t dst_h, int32_t dst_w, const float mean[3], "
                                      "const float std[3], const int32_t* start, float* out, float* prev, "
                                      "void* stream);",
}


def test_entry_points_declared_exported_and_bound(cplib):
    hdr = _header()
    for name, sig in SIGNATURES.items():
        assert sig in hdr, name
        assert name in _lib.EXPORTS and hasattr(cplib, name)
        assert len(getattr(cplib, name).argtypes) == sig.count(",") + 1, name
    assert cplib.cp_preprocess_frame_table_bytes.restype is ctypes.c_int64


def test_frame_table_bytes(cplib):
    one = cplib.cp_preprocess_frame_table_bytes(1)
    assert one >= 6 * 8 + 8 + 2 * 4 and one % 8 == 0       # the inverted affine, the byte offset and the size
    assert cplib.cp_preprocess_frame_table_bytes(5) == 5 * one
    for B in (0, -2):
        assert cplib.cp_preprocess_frame_table_bytes(B) == INVALID
        assert b"B must be > 0" in cplib.cp_last_error()


def _table(cplib, hw=((480, 640), (720, 1280)), fmt=_lib.CP_PIX_BGR, offsets=None, frames_bytes=None, B=None,
           table=8, null=(), trans=False):
    hw = np.ascontiguousarray(hw, np.int32).reshape(-1, 2)
    per = hw[:, 0].astype(np.int64) * hw[:, 1] * (3 if fmt == _lib.CP_PIX_BGR else 1.5)
    offs = np.ascontiguousarray(offsets if offsets is not None else np.concatenate([[0], np.cumsum(per)[:-1]]), np.int64)
    nbytes = int(per.sum()) if frames_bytes is None else frames_bytes
    tr = np.tile(np.array([0.5, 0, 0, 0, 0.5, 0], np.float64), (hw.shape[0], 1)) if trans else None
    p64 = None if "offsets" in null else offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
    p32 = None if "src_hw" in null else hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
    ptr = None if tr is None else tr.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    return cplib.cp_preprocess_frame_table(nbytes, p64, p32, fmt, hw.shape[0] if B is None else B, 512, 512, ptr,
                                           None if "table" in null else ctypes.c_void_p(table), None)


def _err(cplib):
    return cplib.cp_last_error()


def test_frame_table_validates_its_arguments(cplib):
    for what in ("offsets", "src_hw", "table"):
        assert _table(cplib, null=(what,)) == INVALID and b"null argument" in _err(cplib), what
    for B in (0, -1):
        assert _table(cplib, B=B) == INVALID and b"bad shape" in _err(cplib), B
    assert _table(cplib, frames_bytes=0) == INVALID and b"bad shape" in _err(cplib)
    for fmt in (-1, 3, 9):
        assert _table(cplib, fmt=fmt) == INVALID and b"unknown pixel format %d" % fmt in _err(cplib)
    # a frame running past the buffer: one byte short, a negative offset, an offset past the end
    assert _table(cplib, frames_bytes=480 * 640 * 3 + 720 * 1280 * 3 - 1) == INVALID
    assert b"frame 1 (720 x 1280 at byte 921600) lies outside the 3686399-byte buffer" in _err(cplib)
    assert _table(cplib, offsets=[-1, 0]) == INVALID and b"frame 0" in _err(cplib) and b"lies outside" in _err(cplib)
    assert _table(cplib, offsets=[0, 1 << 40]) == INVALID and b"lies outside" in _err(cplib)
    for fmt in (_lib.CP_PIX_NV12, _lib.CP_PIX_I420):
        assert _table(cplib, hw=((480, 640), (721, 1280)), fmt=fmt) == INVALID
        assert b"frame 1 has size 721 x 1280 (YUV 4:2:0 needs even sizes)" in _err(cplib)
        assert _table(cplib, hw=((480, 641),), fmt=fmt) == INVALID and b"even sizes" in _err(cplib)
    assert _table(cplib, hw=((480, 640), (0, 1280))) == INVALID and b"frame 1 has size 0 x 1280" in _err(cplib)
    assert b"cp_preprocess_frame_table" in _err(cplib)


def _ragged(cplib, fmt=_lib.CP_PIX_BGR, B=2, dh=512, dw=512, frames=8, table=8, out=8, start=0, prev=0, mean=True,
            std=True):
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4) if mean else None
    s = (ctypes.c_float * 3)(0.3, 0.3, 0.3) if std else None
    return cplib.cp_preprocess_slots_ragged_dev(ctypes.c_void_p(frames), ctypes.c_void_p(table), fmt, B, dh, dw, m, s,
                                                ctypes.c_void_p(start), ctypes.c_void_p(out), ctypes.c_void_p(prev), None)


def test_slots_ragged_validates_its_arguments(cplib):
    for kw in ({"frames": 0}, {"table": 0}, {"out": 0}, {"mean": False}, {"std": False}):
        assert _ragged(cplib, **kw) == INVALID and b"null argument" in _err(cplib), kw
    for kw in ({"start": 8}, {"prev": 8}):
        assert _ragged(cplib, **kw) == INVALID and b"start and prev go together" in _err(cplib), kw
    for fmt in (-1, 3, 7):
        assert _ragged(cplib, fmt=fmt) == INVALID and b"unknown pixel format %d" % fmt in _err(cplib)
    for kw in ({"B": 0}, {"B": -3}, {"dh": 0}, {"dw": -1}):
        assert _ragged(cplib, **kw) == INVALID and b"bad shape" in _err(cplib), kw
    assert b"cp_preprocess_slots_ragged_dev" in _err(cplib)


# ---- the graphs' refusals (all raised before any device work) --------------------------------------------------------
def _opt():
    return cpb.default_opt("dla_34", tracking_task=True)


def _shell():
    det = ObjectPoseDetector.__new__(ObjectPoseDetector)
    det.opt = _opt()
    return det


def _multi_shell(cls=MultiCategoryTracker):
    det = cls.__new__(cls)
    det.opt = _opt()
    det.categories = ["chair", "cup", "laptop"]
    return det


@pytest.mark.parametrize("make, cls", [(_shell, cpb.TrackGraph), (_multi_shell, cpb.MultiCategoryTrackGraph)],
                         ids=["TrackGraph", "MultiCategoryTrackGraph"])
def test_graphs_refuse_per_slot_sizes_they_cannot_take(make, cls):
    name = cls.__name__
    with pytest.raises(ValueError, match=r"%s: frame_hw is one \(H, W\) for every slot or one per slot, got 3 for 2 "
                                         r"slots" % name):
        cls(make(), slots=2, frame_hw=[(480, 640), (720, 1280), (512, 512)], camera_matrix=None)
    with pytest.raises(ValueError, match=r"got 1 for 2 slots"):
        cls(make(), slots=2, frame_hw=[(480, 640)], camera_matrix=None)
    with pytest.raises(ValueError, match=r"frame_hw is one \(H, W\) for every slot or one per slot, got"):
        cls(make(), slots=2, frame_hw=[(480, 640), (720, 1280, 3)], camera_matrix=None)
    for fmt in ("nv12", "i420"):
        with pytest.raises(ValueError, match="%s frames need an even, positive image size; got 721 x 1280" % fmt):
            cls(make(), slots=2, frame_hw=[(480, 640), (721, 1280)], camera_matrix=None, pixel_format=fmt)
        with pytest.raises(ValueError, match="got 480 x 641"):
            cls(make(), slots=2, frame_hw=np.array([[480, 641], (720, 1280)]), camera_matrix=None, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"camera_matrix must be \[3,3\] or one \[3,3\] per frame \(\[2,3,3\]\)"):
        cls(make(), slots=2, frame_hw=[(480, 640), (720, 1280)], camera_matrix=np.eye(3)[None].repeat(3, 0))


@pytest.mark.parametrize("over, exc, msg", [
    ({"tracking_task": False}, ValueError, r"MultiCategoryTrackGraph needs a tracking model"),
    ({"test_scales": [1.0, 0.5]}, NotImplementedError, r"test_scales=\[1\]"),
    ({"gt_pre_hm_hmhp": True}, NotImplementedError, r"ground-truth heat maps .* run through MultiCategoryTracker.run_batch"),
    ({"gt_pre_hm_hmhp_first": True}, NotImplementedError, r"ground-truth heat maps"),
])
def test_multi_category_graph_refuses_options(over, exc, msg):
    det = _multi_shell()
    for k, v in over.items():
        setattr(det.opt, k, v)
    with pytest.raises(exc, match=msg):
        cpb.MultiCategoryTrackGraph(det, slots=2, frame_hw=(480, 640), camera_matrix=None)


def test_multi_category_graph_takes_a_multi_category_tracker_only():
    with pytest.raises(ValueError, match="needs a MultiCategoryTracker; a MultiCategoryDetector is not a tracking model"):
        cpb.MultiCategoryTrackGraph(_multi_shell(MultiCategoryDetector), slots=1, frame_hw=(480, 640),
                                    camera_matrix=None)
    with pytest.raises(NotImplementedError, match="one category's ObjectPoseDetector goes to TrackGraph"):
        cpb.MultiCategoryTrackGraph(_shell(), slots=1, frame_hw=(480, 640), camera_matrix=None)
    # and TrackGraph, given several categories, names the graph that takes them
    with pytest.raises(NotImplementedError, match="several run through MultiCategoryTracker.run_batch or a "
                                                  "MultiCategoryTrackGraph"):
        cpb.TrackGraph(_multi_shell(), slots=1, frame_hw=(480, 640), camera_matrix=None)
    assert issubclass(cpb.MultiCategoryTrackGraph, cpb.TrackGraph)
