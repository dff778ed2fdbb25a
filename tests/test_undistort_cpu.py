"""Lens distortion without a GPU: the numpy restatement of cv2.remap (tests/remap_ref.py) is cv2.remap bit for bit on
undistortion maps of all three models and on hand-made maps with half ties, far-outside and non-finite entries; the
product's map builder is the documented recipe; LensDistortion checks its arguments; run_batch, the pipelines and the
four graphs refuse what they do not take before any device work; the new entry points check their arguments."""
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.detector import affine_from_center_scale
from centerpose_b200.lens import LensDistortion, MapCache, slot_distortions, undistort_map
from tests import remap_ref
from tests.test_abi import _declared_symbols
from tests.test_detect_graph_cpu import _multi, no_device  # noqa: F401  (fixture)
from tests.test_yuv_input_cpu import _host_detector

INVALID = -1      # CP_ERR_INVALID
FRAMES = [(1440, 1920), (720, 1280), (480, 640)]
INPUTS = [(512, 512), (384, 512)]


def _K(h, w):
    return np.array([[0.8 * w, 0, w / 2 + 3.3], [0, 0.8 * w, h / 2 - 2.1], [0, 0, 1]])


LENSES = {
    "plumb_bob": LensDistortion([-0.28, 0.07, 1e-3, -5e-4, -0.01]),
    "plumb_bob4": LensDistortion([-0.2, 0.05, 1e-3, 2e-4]),
    "rational_polynomial": LensDistortion([0.3, -0.1, 1e-3, -5e-4, 0.02, 0.6, -0.05, 0.05], "rational_polynomial"),
    "equidistant": LensDistortion([0.05, -0.01, 0.002, -0.0005], "equidistant"),
}


def _frame(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _cv2_remap(img, m):
    import cv2
    return cv2.remap(img, np.ascontiguousarray(m[..., 0]), np.ascontiguousarray(m[..., 1]), cv2.INTER_LINEAR,
                     borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def _recipe(dist, K, hw, ihw):
    """The recipe of the issue, written out with cv2 alone."""
    import cv2
    (h, w), (ih, iw) = hw, ihw
    A = affine_from_center_scale(np.array([w / 2., h / 2.], np.float32), float(max(h, w)), iw, ih)
    Kn = K if dist.new_camera_matrix is None else dist.new_camera_matrix
    P = np.vstack([A, [0, 0, 1]]) @ Kn
    if dist.model == "equidistant":
        mx, my = cv2.fisheye.initUndistortRectifyMap(K, dist.coeffs, np.eye(3), P, (iw, ih), cv2.CV_32FC1)
    else:
        mx, my = cv2.initUndistortRectifyMap(K, dist.coeffs, None, P, (iw, ih), cv2.CV_32FC1)
    return mx, my


# ---- the restatement and the map builder ------------------------------------------------------------------------------
@pytest.mark.parametrize("lens", sorted(LENSES))
@pytest.mark.parametrize("hw", FRAMES)
@pytest.mark.parametrize("ihw", INPUTS)
def test_restatement_is_cv2_remap_and_the_builder_is_the_recipe(lens, hw, ihw):
    dist, K = LENSES[lens], _K(*hw)
    m = undistort_map(dist, K, hw, ihw)
    assert m.dtype == np.float32 and m.shape == ihw + (2,) and m.flags.c_contiguous
    mx, my = _recipe(dist, K, hw, ihw)
    assert np.array_equal(m[..., 0], mx) and np.array_equal(m[..., 1], my)
    img = _frame(*hw, seed=hw[0] + ihw[1])
    assert np.array_equal(remap_ref.remap_u8(img, mx, my), _cv2_remap(img, m))


@pytest.mark.parametrize("scale", [0.6, 1.4])          # K_new that widens the view, and one that crops
def test_new_camera_matrix(scale):
    hw, ihw = (720, 1280), (512, 512)
    K = _K(*hw)
    Kn = K.copy()
    Kn[0, 0] *= scale
    Kn[1, 1] *= scale
    for base in ("plumb_bob", "equidistant"):
        d = LENSES[base]
        dist = LensDistortion(d.coeffs, d.model, new_camera_matrix=Kn)
        assert np.array_equal(dist.camera(K), Kn) and np.array_equal(LENSES[base].camera(K), K)
        m = undistort_map(dist, K, hw, ihw)
        mx, my = _recipe(dist, K, hw, ihw)
        assert np.array_equal(m[..., 0], mx) and np.array_equal(m[..., 1], my)
        img = _frame(*hw, seed=7)
        assert np.array_equal(remap_ref.remap_u8(img, mx, my), _cv2_remap(img, m))


def test_restatement_on_hand_made_maps():
    rng = np.random.default_rng(0)
    img = _frame(300, 400, seed=3)
    # exact half ties of the 1/32 grid, negative and far-outside positions
    mx = (rng.integers(-200, 800 * 32, (256, 256)) / 32 + rng.choice([0, 1 / 64, -1 / 64], (256, 256))).astype(np.float32)
    my = (rng.integers(-200, 600 * 32, (256, 256)) / 32 + rng.choice([0, 1 / 64, -1 / 64], (256, 256))).astype(np.float32)
    # non-finite and huge entries, next to in-frame ones
    bad = np.array([np.nan, np.inf, -np.inf, 1e10, -1e10, 6.7e7, -6.7e7, 2 ** 26, -2 ** 26, 2 ** 26 - 1], np.float32)
    mx[:10, 0], my[:10, 0] = bad, 100.5
    mx[10:20, 0], my[10:20, 0] = 200.25, bad
    mx[20:30, 0], my[20:30, 0] = bad, bad
    m = np.stack([mx, my], -1)
    assert np.array_equal(remap_ref.remap_u8(img, mx, my), _cv2_remap(img, m))
    assert not remap_ref.remap_u8(img, mx, my)[:30, 0].any()          # every non-finite or far entry is the border


def test_zero_distortion_is_the_inverse_affine():
    """D = 0, K_new = K: the map is the fix_res affine's inverse, to 1e-3 px (the composition, not a bit claim)."""
    hw, ihw = (720, 1280), (384, 512)
    m = undistort_map(LensDistortion([0, 0, 0, 0, 0]), _K(*hw), hw, ihw)
    A = affine_from_center_scale(np.array([640., 360.], np.float32), 1280.0, ihw[1], ihw[0])
    Ai = np.linalg.inv(np.vstack([A, [0, 0, 1]]))
    ys, xs = np.mgrid[0:ihw[0], 0:ihw[1]]
    want = np.einsum("ij,jhw->hwi", Ai[:2], np.stack([xs, ys, np.ones_like(xs)]).astype(np.float64))
    assert np.abs(m - want).max() < 1e-3


def test_map_cache_keys_and_bound():
    c = MapCache(capacity=2)
    built = []
    import centerpose_b200.lens as lens_mod
    orig = lens_mod.undistort_map
    try:
        lens_mod.undistort_map = lambda *a: built.append(a[1:]) or np.zeros((2, 2, 2), np.float32)
        d = LENSES["plumb_bob"]
        K1, K2 = _K(480, 640), _K(480, 640) * 1.01
        a = c.get(d, K1, (480, 640), (2, 2), "cpu")
        assert c.get(d, K1, (480, 640), (2, 2), "cpu") is a and len(built) == 1       # once per camera
        c.get(d, K2, (480, 640), (2, 2), "cpu")                                        # a changed camera: its own map
        c.get(d, K1, (720, 1280), (2, 2), "cpu")                                       # another frame size
        assert len(built) == 3 and len(c._maps) == 2
        c.get(d, K1, (480, 640), (2, 2), "cpu")                                        # dropped, least recently used
        assert len(built) == 4
    finally:
        lens_mod.undistort_map = orig


# ---- LensDistortion and the distortion argument --------------------------------------------------------------------
def test_lens_distortion_validates():
    assert cpb.LensDistortion is LensDistortion
    for model, n in (("plumb_bob", 4), ("plumb_bob", 5), ("rational_polynomial", 8), ("equidistant", 4)):
        LensDistortion(np.zeros(n), model)
    for model, n in (("plumb_bob", 8), ("plumb_bob", 3), ("rational_polynomial", 5), ("equidistant", 5),
                     ("plumb_bob", 12), ("rational_polynomial", 14)):
        with pytest.raises(ValueError, match="%s takes .* coefficients, got shape \\(%d,\\)" % (model, n)):
            LensDistortion(np.zeros(n), model)
    with pytest.raises(ValueError, match="model must be one of plumb_bob, rational_polynomial, equidistant"):
        LensDistortion(np.zeros(5), "fisheye")
    with pytest.raises(ValueError, match="coefficients must be finite"):
        LensDistortion([0.1, np.nan, 0, 0, 0])
    with pytest.raises(ValueError, match="takes 4 or 5 coefficients, got shape \\(1, 5\\)"):
        LensDistortion(np.zeros((1, 5)))
    with pytest.raises(ValueError, match="new_camera_matrix must be a finite 3x3 matrix"):
        LensDistortion(np.zeros(5), new_camera_matrix=np.eye(4))
    with pytest.raises(ValueError, match="new_camera_matrix must be a finite 3x3 matrix"):
        LensDistortion(np.zeros(5), new_camera_matrix=np.full((3, 3), np.inf))


def test_slot_distortions():
    d = LENSES["plumb_bob"]
    assert slot_distortions(None, 3) is None and slot_distortions([None] * 3, 3) is None
    assert slot_distortions(d, 2) == [d, d] and slot_distortions([None, d], 2) == [None, d]
    with pytest.raises(ValueError, match="run_batch: distortion is one LensDistortion or one per frame or slot, got 2 "
                                         "for 3"):
        slot_distortions([d, d], 3)
    with pytest.raises(TypeError, match="a distortion entry is a LensDistortion or None, got ndarray"):
        slot_distortions([d, np.zeros(5)], 2)
    with pytest.raises(TypeError, match="distortion is a LensDistortion or a list"):
        slot_distortions(np.zeros(5), 2)


D = LENSES["plumb_bob"]


def test_run_batch_refusals(no_device):
    det = _host_detector()
    cam = np.eye(3)
    with pytest.raises(ValueError, match="pre-processed fp32 input has no frame to remap"):
        det.run_batch(torch.zeros((2, 3, 64, 64)), cam, distortion=D)
    with pytest.raises(ValueError, match="got 3 for 2"):
        det.run_batch(np.zeros((2, 48, 64, 3), np.uint8), cam, distortion=[D] * 3)
    with pytest.raises(ValueError, match="got 1 for 2"):
        det.run_batch([np.zeros((48, 64, 3), np.uint8)] * 2, cam, distortion=[D])
    det.opt.fix_short = 512
    for frames in (np.zeros((2, 48, 64, 3), np.uint8), [np.zeros((48, 64, 3), np.uint8)] * 2):
        with pytest.raises(NotImplementedError, match="fix_short|fix_res mode only"):
            det.run_batch(frames, cam, distortion=D)
    trk = _host_detector(tracking=True)
    with pytest.raises(ValueError, match="got 2 for 3"):
        trk.run_batch([np.zeros((48, 64, 3), np.uint8), None, None], cam, track=True, distortion=[D, None])
    trk.opt.fix_res = False
    with pytest.raises(NotImplementedError, match="the keep_res and fix_short pre-process take no distortion"):
        trk.run_batch([np.zeros((48, 64, 3), np.uint8), None], cam, track=True, distortion=[D, None])
    for tracking in (False, True):
        m = _multi(tracking=tracking)
        m.opt.device, m.scales, m._slots = torch.device("cuda"), m.opt.test_scales, None
        with pytest.raises(ValueError, match="pre-processed fp32 input has no frame to remap"):
            m.run_batch(torch.zeros((2, 3, 64, 64)), cam, distortion=D)
        with pytest.raises(ValueError, match="got 3 for 2"):
            m.run_batch([np.zeros((48, 64, 3), np.uint8)] * 2, cam, distortion=[D] * 3)


@pytest.mark.parametrize("cls, tracking, multi", [(cpb.DetectGraph, False, False), (cpb.TrackGraph, True, False),
                                                  (cpb.MultiCategoryDetectGraph, False, True),
                                                  (cpb.MultiCategoryTrackGraph, True, True)])
def test_graphs_refuse_before_device_work(cls, tracking, multi, no_device):
    det = _multi(tracking=tracking) if multi else _host_detector(tracking=tracking)
    for kw in ({"frame_hw": (480, 640)}, {"frame_hw": [(480, 640), (720, 1280)]},
               {"frame_hw": (480, 640), "idle_slots": True}):
        with pytest.raises(ValueError, match="%s: distortion is one LensDistortion or one per frame or slot, got 3 "
                                             "for 2" % cls.__name__):
            cls(det, slots=2, camera_matrix=np.eye(3), distortion=[D] * 3, **kw)
        with pytest.raises(TypeError, match="%s: a distortion entry is a LensDistortion or None" % cls.__name__):
            cls(det, slots=2, camera_matrix=np.eye(3), distortion=[D, "plumb_bob"], **kw)
    det.opt.fix_short = 512
    with pytest.raises(NotImplementedError, match="fix_res mode only|fix_short"):
        cls(det, slots=2, frame_hw=(480, 640), camera_matrix=np.eye(3), distortion=D)


def test_pipelines_refuse(no_device):
    det = _host_detector()
    with pytest.raises(ValueError, match="BatchPipeline: distortion is one LensDistortion or one per frame or slot, got "
                                         "2 for 4"):
        cpb.BatchPipeline(det, batch=4, height=48, width=64, camera_matrix=np.eye(3), distortion=[D, D])
    with pytest.raises(ValueError, match="TrackPipeline: distortion is one LensDistortion or one per frame or slot, got "
                                         "3 for 2"):
        cpb.TrackPipeline(_host_detector(tracking=True), slots=2, camera_matrix=np.eye(3), distortion=[D] * 3)


# ---- the C ABI ---------------------------------------------------------------------------------------------------------
def test_entry_points_declared_exported_and_bound(cplib):
    for name in ("cp_preprocess_remap", "cp_preprocess_frame_table_maps"):
        assert name in _declared_symbols() and name in _lib.EXPORTS and hasattr(cplib, name), name
    with open(__file__.replace("tests/test_undistort_cpu.py", "include/centerpose_b200.h")) as fp:
        assert "CP_PIX_REMAP = %d" % _lib.CP_PIX_REMAP in fp.read()
    codes = list(_lib.PIXEL_FORMAT_CODES.values()) + [_lib.CP_PIX_PER_FRAME]
    assert all(c & _lib.CP_PIX_REMAP == 0 for c in codes)


def _args(hw, fmts, maps):
    hw = np.ascontiguousarray(hw, np.int32).reshape(-1, 2)
    offs = np.ascontiguousarray(np.arange(len(hw)) * 4096, np.int64)
    codes = np.ascontiguousarray(fmts, np.int32)
    ptrs = (ctypes.c_void_p * len(hw))(*maps)
    return hw, offs, codes, ptrs


def _remap(cplib, hw, fmts, maps, null=(), B=None, nbytes=1 << 20):
    hw, offs, codes, ptrs = _args(hw, fmts, maps)
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    return cplib.cp_preprocess_remap(
        None if "frames" in null else ctypes.c_void_p(8), nbytes,
        None if "offsets" in null else offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
        None if "src_hw" in null else hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
        None if "formats" in null else codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
        None if "maps" in null else ptrs, None if "out" in null else ctypes.c_void_p(8),
        len(offs) if B is None else B, 64, 64, None, m, m, None)


def _table(cplib, hw, fmt, fmts, maps, null=(), B=None, nbytes=1 << 20):
    hw, offs, codes, ptrs = _args(hw, fmts if fmts is not None else [0] * len(hw), maps)
    return cplib.cp_preprocess_frame_table_maps(
        nbytes, None if "offsets" in null else offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
        None if "src_hw" in null else hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), fmt,
        None if fmts is None else codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
        None if "maps" in null else ptrs, len(offs) if B is None else B, 64, 64, None,
        None if "table" in null else ctypes.c_void_p(8), None)


def test_remap_entry_points_validate_their_arguments(cplib):
    P, err = _lib, cplib.cp_last_error
    hw, fmts, maps = [(10, 10), (12, 12)], [P.CP_PIX_BGR, P.CP_PIX_NV12], [16, None]
    for what in ("frames", "offsets", "src_hw", "formats", "maps", "out"):
        assert _remap(cplib, hw, fmts, maps, null=(what,)) == INVALID and b"null argument" in err(), what
    for what in ("offsets", "src_hw", "maps", "table"):
        assert _table(cplib, hw, P.CP_PIX_PER_FRAME, fmts, maps, null=(what,)) == INVALID, what
        assert b"cp_preprocess_frame_table_maps: null argument" in err()
    for B in (0, -1):
        assert _remap(cplib, hw, fmts, maps, B=B) == INVALID and b"cp_preprocess_remap: bad shape" in err()
        assert _table(cplib, hw, P.CP_PIX_BGR, None, maps, B=B) == INVALID and b"bad shape" in err()
    # a misaligned map, an unknown per-frame format and a frame outside the buffer: before any work
    assert _remap(cplib, hw, fmts, [12, None]) == INVALID and b"map of frame 0 is not 8-byte aligned" in err()
    assert _remap(cplib, hw, [P.CP_PIX_BGR, 5], maps) == INVALID and b"frame 1 has unknown pixel format 5" in err()
    assert _remap(cplib, hw, fmts, maps, nbytes=4096 + 100) == INVALID and b"outside" in err()
    assert _table(cplib, [(10, 10), (9, 12)], P.CP_PIX_PER_FRAME, [P.CP_PIX_BGR, P.CP_PIX_I420], maps) == INVALID
    assert b"(YUV 4:2:0 needs even sizes)" in err()
    # format / formats pairs: a cp_pixel_format alone, or CP_PIX_PER_FRAME with formats
    for fmt, fm in ((P.CP_PIX_PER_FRAME, None), (P.CP_PIX_BGR, fmts), (5, None), (P.CP_PIX_BGR | P.CP_PIX_REMAP, None),
                    (P.CP_PIX_PER_FRAME | P.CP_PIX_REMAP, fmts)):
        assert _table(cplib, hw, fmt, fm, maps) == INVALID and b"cp_preprocess_frame_table_maps: format" in err(), fmt


def test_launch_codes(cplib):
    """The graph-safe table launches take every table code with CP_PIX_REMAP (they pass the code check and stop at the
    shape); the uniform launch and unknown codes are refused."""
    P, err = _lib, cplib.cp_last_error
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    v = ctypes.c_void_p(8)
    for code in list(P.PIXEL_FORMAT_CODES.values()) + [P.CP_PIX_PER_FRAME]:
        rc = cplib.cp_preprocess_slots_ragged_dev(v, v, code | P.CP_PIX_REMAP, 0, 32, 32, m, m, None, v, None, None)
        assert rc == INVALID and b"cp_preprocess_slots_ragged_dev: bad shape" in err(), code
        rc = cplib.cp_preprocess_slots_rows_dev(v, v, code | P.CP_PIX_REMAP, v, 0, 32, 32, m, m, None, None, v, None,
                                                None)
        assert rc == INVALID and b"cp_preprocess_slots_rows_dev: bad shape" in err(), code
        rc = cplib.cp_preprocess_slots_dev(v, code | P.CP_PIX_REMAP, 2, 64, 64, 32, 32, None, m, m, None, v, None, None)
        assert rc == INVALID and b"unknown pixel format %d" % (code | P.CP_PIX_REMAP) in err(), code
    for bad in (P.CP_PIX_REMAP | 5, P.CP_PIX_REMAP | 200, P.CP_PIX_REMAP * 2, -P.CP_PIX_REMAP):
        rc = cplib.cp_preprocess_slots_ragged_dev(v, v, bad, 2, 32, 32, m, m, None, v, None, None)
        assert rc == INVALID and b"unknown pixel format %d" % bad in err(), bad
        rc = cplib.cp_preprocess_slots_rows_dev(v, v, bad, v, 2, 32, 32, m, m, None, None, v, None, None)
        assert rc == INVALID and b"unknown pixel format %d" % bad in err(), bad
