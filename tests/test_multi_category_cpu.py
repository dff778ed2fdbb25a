"""Multi-model plans and MultiCategoryDetector without a GPU: argument validation of the new C calls (error codes, no
device touched) and the detector's checkpoint checks."""
import ctypes

import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib, synth

INVALID = -1      # CP_ERR_INVALID


def _cfg(tracking=0):
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


@pytest.mark.parametrize("n", [0, -1, _lib.CP_MAX_MODELS + 1])
def test_bad_model_count(cplib, n):
    plan = ctypes.c_void_p()
    assert cplib.cp_plan_create_multi(ctypes.byref(_cfg()), n, ctypes.byref(plan)) == INVALID
    assert b"num_models" in cplib.cp_last_error()
    assert not plan.value


def test_tracking_takes_one_model(cplib):
    plan = ctypes.c_void_p()
    assert cplib.cp_plan_create_multi(ctypes.byref(_cfg(tracking=1)), 2, ctypes.byref(plan)) == INVALID
    assert b"tracking" in cplib.cp_last_error()


def test_model_calls_validate_arguments(cplib):
    d = _lib.CpOpDesc()
    assert cplib.cp_plan_op_desc_model(None, 0, 0, ctypes.byref(d)) == INVALID
    assert cplib.cp_plan_load_weights_model(None, 0, None, None, None, 0, None) == INVALID
    assert cplib.cp_infer_multi(None, 1, None, None, None, None, None, None, None, None) == INVALID
    assert cplib.cp_plan_num_models(None) == 0


def _save(tmp_path, name, opt, seed):
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=seed))
    path = str(tmp_path / name)
    cpb.save_model(path, 1, m)
    return path


def test_detector_rejects_incompatible_checkpoints(tmp_path):
    opt = cpb.default_opt("dla_34")
    ok = _save(tmp_path, "chair.pth", opt, 1)
    other = cpb.default_opt("dla_34")
    other.head_conv = 64
    bad = _save(tmp_path, "cup.pth", other, 2)
    with pytest.raises(ValueError, match="does not match"):
        cpb.MultiCategoryDetector(opt, {"chair": ok, "cup": bad})
    with pytest.raises(ValueError, match="unknown category"):
        cpb.MultiCategoryDetector(opt, {"chair": ok, "teapot": ok})
    trk = cpb.default_opt("dla_34", tracking_task=True)
    with pytest.raises(ValueError, match="tracking"):
        cpb.MultiCategoryDetector(trk, {"chair": ok})
    with pytest.raises(ValueError, match="categories"):
        cpb.MultiCategoryDetector(opt, {})
