"""Multi-category tracking without a GPU: argument validation of cp_plan_create_multi_track, cp_infer_multi_track and
cp_tracker_create_multi (error codes, no device touched) and MultiCategoryTracker's checks of its opt, checkpoints,
categories and pre_dets."""
import ctypes

import pytest

import centerpose_b200 as cpb
from centerpose_b200 import _lib, synth
from centerpose_b200.detector import MultiCategoryTracker
from centerpose_b200.tracker import _tracker_config

INVALID = -1      # CP_ERR_INVALID


def _cfg(tracking=1):
    cfg = _lib.CpConfig()
    cfg.arch = _lib.CP_ARCH_DLA34
    cfg.tracking = tracking
    cfg.max_batch, cfg.height, cfg.width = 1, 64, 64
    cfg.precision = _lib.PRECISIONS["fp32"]
    cfg.head_conv = 256
    cfg.num_heads = 1
    cfg._name = b"hm"
    cfg.head_names[0] = cfg._name
    cfg.head_channels[0] = 1
    return cfg


def test_plan_create_multi_track_validates(cplib):
    plan = ctypes.c_void_p()
    assert cplib.cp_plan_create_multi_track(ctypes.byref(_cfg(tracking=0)), 2, ctypes.byref(plan)) == INVALID
    assert b"tracking" in cplib.cp_last_error()
    for n in (0, _lib.CP_MAX_MODELS + 1):
        assert cplib.cp_plan_create_multi_track(ctypes.byref(_cfg()), n, ctypes.byref(plan)) == INVALID
        assert b"num_models" in cplib.cp_last_error()
    assert cplib.cp_plan_create_multi_track(None, 2, ctypes.byref(plan)) == INVALID
    assert b"null" in cplib.cp_last_error()
    assert not plan.value
    # the detection call still refuses several tracking models, and says where they go
    assert cplib.cp_plan_create_multi(ctypes.byref(_cfg()), 2, ctypes.byref(plan)) == INVALID
    assert b"cp_plan_create_multi_track" in cplib.cp_last_error()


def test_infer_multi_track_refuses_null_arguments(cplib):
    assert cplib.cp_infer_multi_track(None, 1, *([None] * 11)) == INVALID
    assert b"null argument" in cplib.cp_last_error()


def _tcfgs(opt, cats, streams=2):
    return [_tracker_config(opt, c, streams, _lib.CP_MAX_K, 0) for c in cats]


def test_tracker_create_multi_validates(cplib):
    opt = cpb.default_opt("dla_34", tracking_task=True)
    opt.conf_border = {"chair": [3, 9], "cup": [2, 8], "laptop": [4, 10]}
    h = ctypes.c_void_p()
    assert cplib.cp_tracker_create_multi(None, 2, ctypes.byref(h)) == INVALID
    cfgs = _tcfgs(opt, ("chair", "cup"))
    arr = (_lib.CpTrackerConfig * 2)(*cfgs)
    assert cplib.cp_tracker_create_multi(arr, 2, None) == INVALID
    for n in (0, _lib.CP_MAX_MODELS + 1):
        assert cplib.cp_tracker_create_multi(arr, n, ctypes.byref(h)) == INVALID
    # anything but visible_thresh / conf_lo / conf_hi differing is refused before any allocation
    for field, value in (("max_age", 7), ("hungarian", 1), ("streams", 3), ("new_thresh", 0.5), ("kalman", 0)):
        cfgs = _tcfgs(opt, ("chair", "cup", "laptop"))
        setattr(cfgs[2], field, value)
        arr = (_lib.CpTrackerConfig * 3)(*cfgs)
        assert cplib.cp_tracker_create_multi(arr, 3, ctypes.byref(h)) == INVALID, field
        assert b"differ in more than visible_thresh" in cplib.cp_last_error(), field
        assert not h.value
    cfgs = _tcfgs(opt, ("chair", "cup"))
    cfgs[1].conf_lo = cfgs[1].conf_hi
    assert cplib.cp_tracker_create_multi((_lib.CpTrackerConfig * 2)(*cfgs), 2, ctypes.byref(h)) == INVALID
    assert b"conf_border" in cplib.cp_last_error()


def _save(tmp_path, name, opt, seed):
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=seed))
    path = str(tmp_path / name)
    cpb.save_model(path, 1, m)
    return path


def test_tracker_rejects_bad_setups(tmp_path):
    opt = cpb.default_opt("dla_34", tracking_task=True)
    ok = _save(tmp_path, "chair.pth", opt, 1)
    other = cpb.default_opt("dla_34", tracking_task=True)
    other.head_conv = 64
    bad = _save(tmp_path, "cup.pth", other, 2)
    with pytest.raises(ValueError, match="tracking"):
        MultiCategoryTracker(cpb.default_opt("dla_34"), {"chair": ok})
    with pytest.raises(ValueError, match="MultiCategoryTracker: the checkpoint of 'cup'.*does not match"):
        MultiCategoryTracker(opt, {"chair": ok, "cup": bad})
    with pytest.raises(ValueError, match="unknown category"):
        MultiCategoryTracker(opt, {"chair": ok, "teapot": ok})
    with pytest.raises(ValueError, match="categories"):
        MultiCategoryTracker(opt, {})
    kal = cpb.default_opt("dla_34", tracking_task=True)
    kal.refined_Kalman = True
    with pytest.raises(NotImplementedError, match="refined_Kalman"):
        MultiCategoryTracker(kal, {"chair": ok})
    ms = cpb.default_opt("dla_34", tracking_task=True)
    ms.test_scales = [1.0, 0.5]
    with pytest.raises(NotImplementedError, match="test_scales"):
        MultiCategoryTracker(ms, {"chair": ok})
    # the detection class keeps refusing tracking and names the tracking one
    with pytest.raises(ValueError, match="MultiCategoryTracker"):
        cpb.MultiCategoryDetector(opt, {"chair": ok})


def test_tracker_pre_dets_checked():
    det = object.__new__(MultiCategoryTracker)          # the check reads only the categories
    det.categories = ["chair", "cup"]
    assert det._slot_pre_dets(None, 2) is None
    got = det._slot_pre_dets({"cup": [None, [{"score": 1.0}]]}, 2)
    assert det._cat_pre_dets(got) == [None, [None, [{"score": 1.0}]]]
    with pytest.raises(ValueError, match="unknown category 'laptop'"):
        det._slot_pre_dets({"laptop": [None, None]}, 2)
    with pytest.raises(ValueError, match="3 entries for 2 slots"):
        det._slot_pre_dets({"chair": [None, None, None]}, 2)
    with pytest.raises(ValueError, match="maps a category"):
        det._slot_pre_dets([None, None], 2)
