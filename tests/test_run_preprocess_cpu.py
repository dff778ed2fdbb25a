"""run()'s device pre-process without a GPU: the numpy restatement of cv2.resize (tests/resize_ref.py) against cv2
itself, bit for bit, on every pair of lengths 1..48 along each axis, on a seeded sample of joint sizes up to 64 and on
the Objectron frame sizes at the test scales, with random, all-0, all-255 and checkerboard content; the chain
resize -> warp -> normalise through the restatements against pre_process in each mode; cp_preprocess_resize_affine
declared, exported and bound, and its refusals of bad sizes before any device work; and run()'s refusal of a test
scale that resizes the frame to nothing, before any upload."""
import ctypes

import numpy as np
import pytest

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.detector import ObjectPoseDetector
from oracle import preprocess_ref
from tests import resize_ref
from tests.test_abi import _declared_symbols
from tests.test_meta_geometry import _detector

INVALID = -1
CONTENTS = ("random", "zeros", "full", "checker")
OBJECTRON = [(1440, 1920), (1920, 1440), (480, 640), (600, 800)]
SCALES = (0.33, 0.5, 0.6, 0.75, 0.9, 1.25, 1.5, 2.0)


def _frame(h, w, content, seed):
    if content == "random":
        return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if content == "zeros":
        return np.zeros((h, w, 3), np.uint8)
    if content == "full":
        return np.full((h, w, 3), 255, np.uint8)
    yy, xx = np.mgrid[:h, :w]
    return np.repeat((((yy + xx) & 1) * 255).astype(np.uint8)[..., None], 3, axis=2)


def _same(f, rw, rh):
    import cv2
    return np.array_equal(resize_ref.resize_u8(f, rw, rh), cv2.resize(f, (rw, rh)))


@pytest.mark.parametrize("content", CONTENTS)
@pytest.mark.parametrize("axis", ["x", "y"])
def test_oracle_is_cv2_along_each_axis(axis, content):
    """Every (src, dst) pair of lengths 1..48 along one axis; the other axis stays at 5, so its pass runs too."""
    bad = []
    for src in range(1, 49):
        f = _frame(5, src, content, src) if axis == "x" else _frame(src, 5, content, src)
        for dst in range(1, 49):
            rw, rh = (dst, 5) if axis == "x" else (5, dst)
            if not _same(f, rw, rh):
                bad.append((src, dst))
    assert not bad, bad[:8]


@pytest.mark.parametrize("content", CONTENTS)
def test_oracle_is_cv2_on_joint_sizes(content):
    rng = np.random.default_rng(17)
    bad = []
    for _ in range(400):
        sh, sw, rh, rw = (int(v) for v in rng.integers(1, 65, 4))
        if not _same(_frame(sh, sw, content, sh * 64 + sw), rw, rh):
            bad.append((sh, sw, rh, rw))
    assert not bad, bad[:8]


@pytest.mark.parametrize("h, w", OBJECTRON)
def test_oracle_is_cv2_on_objectron_sizes(h, w):
    for content in ("random", "checker"):              # (constant frames: the axis and joint tests)
        f = _frame(h, w, content, h + w)
        for scale in SCALES:
            rw, rh = int(w * scale), int(h * scale)
            assert _same(f, rw, rh), (content, scale)
    # exactly one half (cv2 may take an area path there) and the unchanged size (a copy) follow the same rule
    f = _frame(h, w, "random", 1)
    assert _same(f, w // 2, h // 2) and _same(f, w, h)


def test_oracle_refusals():
    with pytest.raises(ValueError, match="positive"):
        resize_ref.resize_u8(np.zeros((4, 4, 3), np.uint8), 0, 3)
    with pytest.raises(ValueError, match="uint8"):
        resize_ref.resize_u8(np.zeros((4, 4, 3), np.float32), 3, 3)


@pytest.mark.parametrize("mode", ["fix_res", "keep_res", "fix_short"])
@pytest.mark.parametrize("scale", [0.5, 0.75, 1.25])
def test_restated_chain_is_pre_process(mode, scale):
    """warp(resize(frame)) through the restatements, normalised, is pre_process's network input at a test scale."""
    det = _detector(mode)
    img = _frame(61, 83, "random", 5)
    want, meta = det.pre_process(img, scale, {})
    resized = resize_ref.resize_u8(img, int(83 * scale), int(61 * scale))
    got = preprocess_ref.pre_process(resized, meta["inp_width"], meta["inp_height"], det.opt.mean, det.opt.std,
                                     trans_input=meta["trans_input"])
    assert np.array_equal(got, want.numpy())


def _resize_call(cplib, B=1, src=(20, 30), rs=(10, 15), dst=(16, 16), frames=1, out=1, trans=True):
    T = (ctypes.c_double * 6)(1, 0, 0, 0, 1, 0) if trans else None
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    s = (ctypes.c_float * 3)(0.3, 0.3, 0.3)
    return cplib.cp_preprocess_resize_affine(ctypes.c_void_p(frames), ctypes.c_void_p(out), B, src[0], src[1], rs[0],
                                             rs[1], dst[0], dst[1], T, m, s, None)


def test_resize_entry_declared_exported_and_bound(cplib):
    name = "cp_preprocess_resize_affine"
    assert name in _declared_symbols() and name in _lib.EXPORTS and hasattr(cplib, name)


@pytest.mark.parametrize("kw", [dict(B=0), dict(src=(0, 30)), dict(src=(20, -1)), dict(rs=(0, 15)), dict(rs=(10, 0)),
                                dict(dst=(16, 0)), dict(dst=(-2, 16))])
def test_resize_entry_refuses_bad_sizes(cplib, kw):
    assert _resize_call(cplib, **kw) == INVALID
    assert b"cp_preprocess_resize_affine: bad shape" in cplib.cp_last_error()


@pytest.mark.parametrize("kw", [dict(frames=0), dict(out=0), dict(trans=False)])
def test_resize_entry_refuses_null_arguments(cplib, kw):
    assert _resize_call(cplib, **kw) == INVALID
    assert b"cp_preprocess_resize_affine: null argument" in cplib.cp_last_error()


def test_run_refuses_a_scale_that_resizes_to_nothing():
    """cv2.resize raised for these; run() refuses them before it uploads the frame (the shell has no device)."""
    opt = cpb.default_opt("dla_34")
    det = ObjectPoseDetector.__new__(ObjectPoseDetector)
    det.opt, det.scales, det._stage = opt, [1.0, 0.004], None
    with pytest.raises(ValueError, match=r"test scale 0.004 resizes the 200 x 300 frame to 0 x 1 pixels"):
        det.run(np.zeros((200, 300, 3), np.uint8))
    # other inputs keep the host pre_process: no device frame
    for img in (np.zeros((200, 300, 3), np.float32), np.zeros((200, 300), np.uint8), np.zeros((200, 300, 4), np.uint8)):
        assert det._device_frame(img) is None
