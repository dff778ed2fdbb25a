"""The detection graphs without a GPU: DetectGraph and MultiCategoryDetectGraph are exported, share TrackGraph's frame
checking, capture and call (one base, no copy), refuse every option and argument they do not take with a message that
names where it runs, before any device work, and check the frames of a call as TrackGraph does; the control block of a
step with idle slots gathers the live rows' meta rows and scatters the compact outputs of run_batch(list) of the live
frames back to their slots."""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.detector import MultiCategoryDetector, MultiCategoryTracker
from centerpose_b200.graph import _SlotGraph
from tests.test_yuv_input_cpu import _host_detector


@pytest.fixture
def no_device(monkeypatch):
    """Every refusal comes before the library is loaded or a device is touched."""
    def touched(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(_lib, "load", touched)
    monkeypatch.setattr(torch.cuda, "current_device", touched)


def test_exported_and_sharing_one_base():
    assert cpb.DetectGraph.__module__ == cpb.MultiCategoryDetectGraph.__module__ == "centerpose_b200.graph"
    for cls in (cpb.DetectGraph, cpb.MultiCategoryDetectGraph, cpb.TrackGraph, cpb.MultiCategoryTrackGraph):
        assert issubclass(cls, _SlotGraph)
        for name in ("_build", "_plan", "_frames", "_control", "_replay", "_call_rows", "_preprocess",
                     "_preprocess_rows", "_gather"):
            assert getattr(cls, name) is getattr(_SlotGraph, name), (cls, name)


def _multi(tracking=False, cats=("chair", "cup")):
    cls = MultiCategoryTracker if tracking else MultiCategoryDetector
    det = cls.__new__(cls)
    det.opt = cpb.default_opt("dla_34", tracking_task=tracking)
    det.categories = list(cats)
    return det


def _with(det, **over):
    for k, v in over.items():
        setattr(det.opt, k, v)
    return det


@pytest.mark.parametrize("over, exc, msg", [
    ({"tracking_task": True}, ValueError, r"runs a detection model; a tracking model \(opt.tracking_task\) runs through "
                                          r"(MultiCategory)?TrackGraph"),
    ({"test_scales": [1.0, 0.5]}, NotImplementedError,
     r"runs at test_scales=\[1\]; multi-scale detection runs through run\(\)"),
    ({"fix_short": 512}, NotImplementedError,
     r"pre-processes in the fix_res mode only, as run_batch\(list\); keep_res and fix_short run through run\(\)"),
    ({"fix_res": False}, NotImplementedError, r"pre-processes in the fix_res mode only"),
])
def test_refuses_options(over, exc, msg, no_device):
    with pytest.raises(exc, match="DetectGraph " + msg):
        cpb.DetectGraph(_with(_host_detector(), **over), slots=2, frame_hw=(480, 640), camera_matrix=np.eye(3))
    with pytest.raises(exc, match="MultiCategoryDetectGraph " + msg):
        cpb.MultiCategoryDetectGraph(_with(_multi(), **over), slots=2, frame_hw=[(480, 640), (720, 1280)],
                                     camera_matrix=np.eye(3), idle_slots=True)


def test_refuses_the_wrong_detector(no_device):
    with pytest.raises(NotImplementedError, match="DetectGraph detects one category; several run through a "
                                                  "MultiCategoryDetectGraph"):
        cpb.DetectGraph(_multi(), slots=1, frame_hw=(480, 640), camera_matrix=np.eye(3))
    with pytest.raises(NotImplementedError, match="takes an ObjectPoseDetector, got object"):
        cpb.DetectGraph(object(), slots=1, frame_hw=(480, 640), camera_matrix=np.eye(3))
    with pytest.raises(ValueError, match="needs a MultiCategoryDetector; a MultiCategoryTracker runs through "
                                         "MultiCategoryTrackGraph"):
        cpb.MultiCategoryDetectGraph(_multi(tracking=True), slots=1, frame_hw=(480, 640), camera_matrix=np.eye(3))
    with pytest.raises(NotImplementedError, match="ObjectPoseDetector goes to DetectGraph"):
        cpb.MultiCategoryDetectGraph(_host_detector(), slots=1, frame_hw=(480, 640), camera_matrix=np.eye(3))
    # the tracking graphs keep refusing a detection model with their own messages
    with pytest.raises(ValueError, match=r"TrackGraph needs a tracking model \(opt.tracking_task\)"):
        cpb.TrackGraph(_host_detector(), slots=1, frame_hw=(480, 640), camera_matrix=np.eye(3))


def test_refuses_shapes_and_formats(no_device):
    det = _host_detector()
    with pytest.raises(ValueError, match="DetectGraph: slots must be >= 1"):
        cpb.DetectGraph(det, slots=0, frame_hw=(480, 640), camera_matrix=np.eye(3))
    with pytest.raises(ValueError, match=r"frame_hw is one \(H, W\) for every slot or one per slot, got 3 for 2 slots"):
        cpb.DetectGraph(det, slots=2, frame_hw=[(480, 640), (600, 800), (512, 512)], camera_matrix=np.eye(3))
    with pytest.raises(ValueError, match="pixel_format must be one of bgr, nv12, i420"):
        cpb.DetectGraph(det, slots=2, frame_hw=(480, 640), camera_matrix=np.eye(3), pixel_format="yuyv")
    with pytest.raises(ValueError, match="even"):
        cpb.DetectGraph(det, slots=2, frame_hw=[(480, 640), (721, 1280)], camera_matrix=np.eye(3), pixel_format="i420")
    with pytest.raises(ValueError, match=r"camera_matrix must be \[3,3\] or one \[3,3\] per frame \(\[2,3,3\]\)"):
        cpb.DetectGraph(det, slots=2, frame_hw=(480, 640), camera_matrix=np.stack([np.eye(3)] * 3))


def _built(cls=cpb.DetectGraph, S=3, M=1, idle=False, per_slot=False, fmt="bgr"):
    """A graph object with the host state of a built one (no device buffers): calls that are refused never reach
    them."""
    g = cls.__new__(cls)
    g.idle_slots, g.per_slot, g.slots, g.streams, g.pixel_format = idle, per_slot, S, M * S, fmt
    shape = (480, 640, 3) if fmt == "bgr" else (720, 640)
    g._slot_hw, g._slot_shapes = [(480, 640)] * S, [shape] * S
    g.frame_hw, g.frame_shape = ((g._slot_hw, g._slot_shapes) if per_slot else ((480, 640), (S,) + shape))
    g._fresh, g._started = True, [False] * S
    return g


@pytest.mark.parametrize("cls", [cpb.DetectGraph, cpb.MultiCategoryDetectGraph])
def test_refuses_tracking_arguments(cls):
    g = _built(cls)
    for kw in ({"new_video": [True, False, False]}, {"pre_dets": [[], [], []]}):
        with pytest.raises(ValueError, match="%s keeps nothing from one frame to the next: new_video and pre_dets are "
                                             r"tracking arguments \(TrackGraph, run_batch\(track=True\)\)" % cls.__name__):
            g(np.zeros((3, 480, 640, 3), np.uint8), **kw)


def test_checks_the_frames_of_a_call():
    g = _built()
    with pytest.raises(ValueError, match=r"DetectGraph steps every slot at one frame size: frames must be uint8 "
                                         r"\[3, 480, 640, 3\] \(bgr\), got torch.float32 \(3, 480, 640, 3\); idle slots "
                                         r"and mixed sizes run through run_batch\(list\) of the live frames or a "
                                         r"DetectGraph built with one frame_hw per slot"):
        g(np.zeros((3, 480, 640, 3), np.float32))
    with pytest.raises(ValueError, match=r"got list"):
        g([np.zeros((480, 640, 3), np.uint8)] * 3)
    g = _built(cpb.MultiCategoryDetectGraph, per_slot=True, fmt="nv12", M=2)
    with pytest.raises(ValueError, match="built with one frame_hw per slot: frames is a list of 3 frames, got 2 frames"):
        g([np.zeros((720, 640), np.uint8)] * 2)
    with pytest.raises(ValueError, match=r"MultiCategoryDetectGraph steps every slot: slot 1 is idle; idle slots run "
                                         r"through MultiCategoryDetector.run_batch\(list\) of the live frames"):
        g([np.zeros((720, 640), np.uint8), None, np.zeros((720, 640), np.uint8)])
    with pytest.raises(ValueError, match=r"slot 2 takes uint8 \[720, 640\] frames \(nv12, frame_hw \(480, 640\)\), got "
                                         r"torch.uint8 \(480, 640, 3\)"):
        g([np.zeros((720, 640), np.uint8)] * 2 + [np.zeros((480, 640, 3), np.uint8)])
    g = _built(idle=True)
    with pytest.raises(ValueError, match="built with idle slots: frames is a list of 3 frames, got 4 frames"):
        g([None] * 4)
    with pytest.raises(ValueError, match=r"frames must be uint8 \[3, 480, 640, 3\] \(bgr\), got torch.uint8 "
                                         r"\(2, 480, 640, 3\)"):
        g(np.zeros((2, 480, 640, 3), np.uint8))


def _scatter(src, m):
    """cp_gather_rows_dev on the host: row i = src[m[i]], zeros where m[i] < 0."""
    out = np.zeros((len(m),) + src.shape[1:], src.dtype)
    for i, r in enumerate(m):
        if r >= 0:
            out[i] = src[r]
    return out


@pytest.mark.parametrize("M", [1, 2, 3])
@pytest.mark.parametrize("live", [[0], [1, 3], [0, 1, 2, 3], [2, 3], [0, 2, 3]])
def test_control_block_maps_rows_and_slots(M, live):
    """rows: the live slots in slot order (the batch of run_batch(list) of the live frames), whose meta rows the step
    gathers; inv: for category m's slot s the row m * n + k of its frame in the compact [M, n] outputs, -1 for an idle
    slot, so the scatter gives every slot its own records and zeros for the idle ones."""
    S = 4
    g = _built(cpb.MultiCategoryDetectGraph if M > 1 else cpb.DetectGraph, S=S, M=M, idle=True)
    n, MS = len(live), M * S
    c = g._control(live, np.zeros(S, np.int32))
    assert c.dtype == np.int32 and c.shape == (3 * MS + S,)
    assert not c[:MS].any()                                      # no start flags: a detection step keeps no state
    rows, inv = c[MS:MS + S], c[2 * MS + S:]
    assert list(rows[:n]) == live
    meta = np.arange(S * 16, dtype=np.float64).reshape(S, 16)     # per-slot meta rows -> the live rows' meta rows
    assert np.array_equal(_scatter(meta, rows[:n]), meta[live])
    compact = np.arange(1, M * n + 1, dtype=np.float32).reshape(M * n, 1) * np.ones((1, 5), np.float32)
    out = _scatter(compact, inv).reshape(M, S, 5)
    for m in range(M):
        for s in range(S):
            want = compact[m * n + live.index(s)] if s in live else np.zeros(5, np.float32)
            assert np.array_equal(out[m, s], want), (m, s)
