"""The graph-safe tracking step without a GPU: the entry points TrackGraph captures (cp_preprocess_slots_dev,
cp_tracker_reset_dev, cp_tracker_render_dev) are declared, exported and bound with their documented signatures and
refuse bad arguments with CP_ERR_INVALID before touching the device; TrackGraph refuses every option its fixed-shape
form does not take, with a message that names where that option runs."""
import ctypes
import os
import re

import pytest

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.detector import MultiCategoryTracker, ObjectPoseDetector
from tests.util import ROOT

INVALID = -1      # CP_ERR_INVALID
SIGNATURES = {
    "cp_preprocess_slots_dev": "int cp_preprocess_slots_dev(const uint8_t* frames, int32_t format, int32_t B, "
                               "int32_t src_h, int32_t src_w, int32_t dst_h, int32_t dst_w, const double* trans_input, "
                               "const float mean[3], const float std[3], const int32_t* start, float* out, float* prev, "
                               "void* stream);",
    "cp_tracker_reset_dev": "int cp_tracker_reset_dev(cp_tracker* trk, int32_t batch, const int32_t* flags, void* stream);",
    "cp_tracker_render_dev": "int cp_tracker_render_dev(cp_tracker* trk, int32_t batch, const double* meta, "
                             "const double* trans_input, int32_t inp_h, int32_t inp_w, const int32_t* modes, "
                             "float* pre_hm, float* pre_hm_hp, void* stream);",
}


def _header():
    txt = open(os.path.join(ROOT, "include", "centerpose_b200.h")).read()
    return re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", txt, flags=re.S))


def test_entry_points_declared_exported_and_bound(cplib):
    hdr = _header()
    for name, sig in SIGNATURES.items():
        assert sig in hdr, name
        assert name in _lib.EXPORTS and hasattr(cplib, name)
        assert len(getattr(cplib, name).argtypes) == sig.count(",") + 1, name
    assert (_lib.CP_PIX_NV12, _lib.CP_PIX_I420, _lib.CP_PIX_BGR) == (0, 1, 2)
    assert "CP_PIX_BGR = 2" in hdr


def _pre(cplib, fmt=_lib.CP_PIX_BGR, B=2, h=64, w=64, frames=1, out=1, start=0, prev=0, mean=True, std=True):
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4) if mean else None
    s = (ctypes.c_float * 3)(0.3, 0.3, 0.3) if std else None
    return cplib.cp_preprocess_slots_dev(ctypes.c_void_p(frames), fmt, B, h, w, 32, 32, None, m, s,
                                         ctypes.c_void_p(start), ctypes.c_void_p(out), ctypes.c_void_p(prev), None)


def test_preprocess_slots_validates_its_arguments(cplib):
    for kw in ({"frames": 0}, {"out": 0}, {"mean": False}, {"std": False}):
        assert _pre(cplib, **kw) == INVALID and b"null argument" in cplib.cp_last_error(), kw
    for kw in ({"start": 8}, {"prev": 8}):
        assert _pre(cplib, **kw) == INVALID and b"start and prev go together" in cplib.cp_last_error(), kw
    for fmt in (-1, 3, 7):
        assert _pre(cplib, fmt=fmt) == INVALID
        assert b"unknown pixel format %d" % fmt in cplib.cp_last_error()
    for kw in ({"B": 0}, {"B": -3}, {"h": 0}, {"w": -1}):
        assert _pre(cplib, **kw) == INVALID and b"bad shape" in cplib.cp_last_error(), kw
    for fmt in (_lib.CP_PIX_NV12, _lib.CP_PIX_I420):
        assert _pre(cplib, fmt=fmt, h=63) == INVALID
        assert b"YUV 4:2:0 frames need an even size, got 63 x 64" in cplib.cp_last_error()
        assert _pre(cplib, fmt=fmt, w=9) == INVALID and b"even size" in cplib.cp_last_error()
    assert b"cp_preprocess_slots_dev" in cplib.cp_last_error()


def test_tracker_dev_entries_validate_their_arguments(cplib):
    fake = ctypes.c_void_p(8)       # never dereferenced: the checks that need no tracker come first
    for batch in (0, -1):
        assert cplib.cp_tracker_reset_dev(fake, batch, ctypes.c_void_p(8), None) == INVALID
        assert b"cp_tracker_reset_dev: batch must be > 0" in cplib.cp_last_error()
    assert cplib.cp_tracker_reset_dev(None, 2, ctypes.c_void_p(8), None) == INVALID
    assert b"cp_tracker_reset_dev: null argument" in cplib.cp_last_error()
    assert cplib.cp_tracker_reset_dev(fake, 2, None, None) == INVALID
    assert b"null argument" in cplib.cp_last_error()
    assert cplib.cp_tracker_render_dev(None, 1, *([ctypes.c_void_p(8)] * 2), 64, 64, None,
                                       *([ctypes.c_void_p(8)] * 2), None) == INVALID
    assert b"cp_tracker_render: null argument" in cplib.cp_last_error()


# ---- TrackGraph's refusals (all raised before any device work) ------------------------------------------------------
def _shell(**over):
    """An ObjectPoseDetector of a tracking opt that never touched a device: TrackGraph reads only its opt before it
    refuses."""
    opt = cpb.default_opt("dla_34", tracking_task=True)
    for k, v in over.items():
        setattr(opt, k, v)
    det = ObjectPoseDetector.__new__(ObjectPoseDetector)
    det.opt = opt
    return det


@pytest.mark.parametrize("over, exc, msg", [
    ({"tracking_task": False}, ValueError, r"needs a tracking model \(opt.tracking_task\)"),
    ({"test_scales": [1.0, 0.5]}, NotImplementedError, r"test_scales=\[1\]"),
    ({"gt_pre_hm_hmhp": True}, NotImplementedError, r"ground-truth heat maps .* run through run_batch"),
    ({"gt_pre_hm_hmhp_first": True}, NotImplementedError, r"ground-truth heat maps"),
])
def test_track_graph_refuses_options(over, exc, msg):
    with pytest.raises(exc, match=msg):
        cpb.TrackGraph(_shell(**over), slots=2, frame_hw=(480, 640), camera_matrix=None)


def test_track_graph_refuses_shapes_and_formats():
    det = _shell()
    with pytest.raises(ValueError, match="slots must be >= 1"):
        cpb.TrackGraph(det, slots=0, frame_hw=(480, 640), camera_matrix=None)
    with pytest.raises(ValueError, match=r"frame_hw is one \(H, W\) for every slot"):
        cpb.TrackGraph(det, slots=2, frame_hw=[(480, 640), (600, 800), (512, 512)], camera_matrix=None)
    with pytest.raises(ValueError, match="pixel_format must be one of bgr, nv12, i420"):
        cpb.TrackGraph(det, slots=2, frame_hw=(480, 640), camera_matrix=None, pixel_format="yuyv")
    with pytest.raises(ValueError, match="even"):
        cpb.TrackGraph(det, slots=2, frame_hw=(481, 640), camera_matrix=None, pixel_format="nv12")
    with pytest.raises(ValueError, match=r"camera_matrix must be \[3,3\] or one \[3,3\] per frame \(\[2,3,3\]\)"):
        cpb.TrackGraph(det, slots=2, frame_hw=(480, 640), camera_matrix=[[1, 0], [0, 1]])


def test_track_graph_refuses_several_categories():
    det = MultiCategoryTracker.__new__(MultiCategoryTracker)
    det.opt = cpb.default_opt("dla_34", tracking_task=True)
    det.categories = ["chair", "cup"]
    with pytest.raises(NotImplementedError, match="one category; several run through MultiCategoryTracker.run_batch"):
        cpb.TrackGraph(det, slots=2, frame_hw=(480, 640), camera_matrix=None)
    with pytest.raises(NotImplementedError, match="one category"):
        cpb.TrackGraph(object(), slots=2, frame_hw=(480, 640), camera_matrix=None)
