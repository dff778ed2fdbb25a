"""YUV 4:2:0 input without a GPU: the numpy restatement of cv2's NV12 / I420 -> BGR conversion against cv2 itself on a
frame holding every (Y, U, V) triple, and through the warp against cv2.warpAffine; cp_preprocess_yuv420's argument
checks (CP_ERR_INVALID before any device work); and the pixel_format checks of run_batch and the pipelines."""
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.detector import ObjectPoseDetector, check_frames
from centerpose_b200.engine import frame_shape, image_size
from oracle import preprocess_ref
from tests import yuv_ref
from tests.test_abi import _declared_symbols

CODES = {"nv12": "COLOR_YUV2BGR_NV12", "i420": "COLOR_YUV2BGR_I420"}


def _cv2_bgr(f, fmt):
    import cv2
    return cv2.cvtColor(f, getattr(cv2, CODES[fmt]))


def random_yuv(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)


@pytest.mark.parametrize("fmt", ("nv12", "i420"))
def test_oracle_is_cv2_on_every_yuv_triple(fmt):
    f = yuv_ref.exhaustive_yuv420(fmt)
    assert f.shape == (6144, 4096)
    # the frame holds each of the 2^24 (Y, U, V) triples
    H = 4096
    Y = f[:H].astype(np.int64)
    if fmt == "nv12":
        U, V = f[H:, 0::2], f[H:, 1::2]
    else:
        c = f[H:].reshape(-1)
        U, V = c[:H * H // 4].reshape(H // 2, H // 2), c[H * H // 4:].reshape(H // 2, H // 2)
    up = lambda p: np.repeat(np.repeat(p.astype(np.int64), 2, 0), 2, 1)       # noqa: E731
    assert np.unique((Y << 16) | (up(U) << 8) | up(V)).size == 1 << 24
    assert np.array_equal(yuv_ref.yuv420_to_bgr(f, fmt), _cv2_bgr(f, fmt))


def _rotated(h, w, inp):
    import cv2
    M = cv2.getRotationMatrix2D((w * 0.4, h * 0.55), 30.0, inp / (0.6 * max(h, w)))
    M[:, 2] += np.array([inp / 2. - w * 0.4, inp / 2. - h * 0.55])
    return M


@pytest.mark.parametrize("fmt", ("nv12", "i420"))
@pytest.mark.parametrize("h, w, kind", [(48, 64, "fix_res"), (60, 80, "rotated"), (30, 46, "upscale")])
def test_oracle_warp_is_cv2_warp_of_cvtcolor(fmt, h, w, kind):
    import cv2
    f = random_yuv(h, w, seed=h * w)
    inp = 64
    if kind == "fix_res":
        M = preprocess_ref.fix_res_affine(h, w, inp, inp)
    elif kind == "rotated":
        M = _rotated(h, w, inp)
    else:                                  # 3x up-scaling about a point near the border: taps straddle chroma blocks
        M = np.array([[3.1, 0.0, -3.1 * (w - 9.3)], [0.0, 2.9, -2.9 * 1.7]])
    bgr = _cv2_bgr(f, fmt)
    want = cv2.warpAffine(bgr, M, (inp, inp), flags=cv2.INTER_LINEAR)
    got = preprocess_ref.warp_affine_u8(yuv_ref.yuv420_to_bgr(f, fmt), M, inp, inp)
    assert np.array_equal(got, want)
    assert (want == 0).all(axis=-1).any(), "the affine keeps part of the output outside the frame"


def test_oracle_refuses_bad_frames():
    with pytest.raises(ValueError, match="even"):
        yuv_ref.yuv420_to_bgr(np.zeros((10, 6), np.uint8), "nv12")       # 10 rows are not 3H/2
    with pytest.raises(ValueError, match="even"):
        yuv_ref.yuv420_to_bgr(np.zeros((6, 5), np.uint8), "i420")
    with pytest.raises(ValueError, match="unknown format"):
        yuv_ref.yuv420_to_bgr(np.zeros((6, 4), np.uint8), "nv21")


# ---- the C ABI -----------------------------------------------------------------------------------------------------------
def test_entry_point_declared_exported_and_bound(cplib):
    assert "cp_preprocess_yuv420" in _declared_symbols() and "cp_preprocess_yuv420" in _lib.EXPORTS
    assert hasattr(cplib, "cp_preprocess_yuv420") and cplib.cp_version() == 1
    assert (_lib.CP_PIX_NV12, _lib.CP_PIX_I420) == (0, 1)


def _yuv(cplib, offsets, hw, nbytes, fmt=_lib.CP_PIX_NV12, frames=1, out=1, offs_ptr=True, hw_ptr=True, mean=True):
    offs = np.asarray(offsets, np.int64)
    hw = np.asarray(hw, np.int32).reshape(-1, 2)
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4) if mean else None
    s = (ctypes.c_float * 3)(0.3, 0.3, 0.3)
    return cplib.cp_preprocess_yuv420(
        ctypes.c_void_p(frames), nbytes, offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)) if offs_ptr else None,
        hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)) if hw_ptr else None, fmt, ctypes.c_void_p(out), len(offs), 64,
        64, None, m, s, None)


def _err(cplib):
    return cplib.cp_last_error()


def test_yuv_preprocess_validates_its_arguments(cplib):
    # null pointers
    for kw in ({"frames": 0}, {"out": 0}, {"offs_ptr": False}, {"hw_ptr": False}, {"mean": False}):
        assert _yuv(cplib, [0], [[10, 10]], 150, **kw) == -1 and b"null argument" in _err(cplib), kw
    # unknown formats
    for fmt in (-1, 2, 7):
        assert _yuv(cplib, [0], [[10, 10]], 150, fmt=fmt) == -1
        assert b"unknown pixel format %d" % fmt in _err(cplib)
    # odd and empty image sizes, in either layout
    for fmt in (_lib.CP_PIX_NV12, _lib.CP_PIX_I420):
        assert _yuv(cplib, [0, 150], [[10, 10], [9, 10]], 1000, fmt=fmt) == -1
        assert b"frame 1 has size 9 x 10 (YUV 4:2:0 needs even sizes)" in _err(cplib)
        assert _yuv(cplib, [0], [[10, 7]], 1000, fmt=fmt) == -1 and b"needs even sizes" in _err(cplib)
        assert _yuv(cplib, [0], [[0, 4]], 1000, fmt=fmt) == -1 and b"frame 0 has size 0 x 4" in _err(cplib)
    # a frame is H * W * 3 / 2 bytes: 150 for 10 x 10
    assert _yuv(cplib, [0, 150], [[10, 10], [10, 10]], 299) == -1
    assert b"frame 1 (10 x 10 at byte 150) lies outside the 299-byte buffer" in _err(cplib)
    assert _yuv(cplib, [3], [[10, 10]], 152) == -1 and b"outside" in _err(cplib)
    assert _yuv(cplib, [-1], [[10, 10]], 300) == -1 and b"outside" in _err(cplib)
    assert _yuv(cplib, [301], [[2, 2]], 300) == -1 and b"outside" in _err(cplib)
    assert _yuv(cplib, [0], [[10, 10]], 0) == -1 and b"bad shape" in _err(cplib)
    assert b"cp_preprocess_yuv420" in _err(cplib)


# ---- pixel_format in the Python layer --------------------------------------------------------------------------------
def test_frame_shapes():
    assert frame_shape(480, 640, "bgr") == (480, 640, 3)
    assert frame_shape(480, 640, "nv12") == frame_shape(480, 640, "i420") == (720, 640)
    assert image_size((720, 640), "nv12") == (480, 640) and image_size((480, 640, 3), "bgr") == (480, 640)
    with pytest.raises(ValueError, match="even"):
        frame_shape(481, 640, "nv12")
    with pytest.raises(ValueError, match="pixel_format must be one of bgr, nv12, i420"):
        frame_shape(480, 640, "yuyv")
    for bad in ((721, 640), (720, 641), (5, 4), (720, 640, 1), (0, 4)):
        with pytest.raises(ValueError, match=r"expected a i420 frame \[3H/2,W\] with H and W even"):
            image_size(bad, "i420")


def test_check_frames_per_format():
    nv = np.zeros((6, 4), np.uint8)
    check_frames([nv, torch.zeros((12, 8), dtype=torch.uint8), None], allow_idle=True, pixel_format="nv12")
    with pytest.raises(ValueError, match=r"frame 1 has shape \(4, 6, 3\), expected a nv12 frame \[3H/2,W\]"):
        check_frames([nv, np.zeros((4, 6, 3), np.uint8)], allow_idle=False, pixel_format="nv12")
    with pytest.raises(ValueError, match=r"frame 0 has shape \(10, 4\)"):
        check_frames([np.zeros((10, 4), np.uint8)], allow_idle=False, pixel_format="i420")
    with pytest.raises(TypeError, match=r"uint8 \[3H/2,W\]"):
        check_frames([nv.astype(np.float32)], allow_idle=False, pixel_format="i420")
    with pytest.raises(ValueError, match=r"expected \[H,W,3\]"):
        check_frames([nv], allow_idle=False)                      # the default stays BGR
    with pytest.raises(ValueError, match="pixel_format must be one of"):
        check_frames([nv], allow_idle=False, pixel_format="NV12")


def _host_detector(tracking=False):
    """An ObjectPoseDetector that only gets as far as its argument checks (no model, no device work)."""
    opt = cpb.default_opt("dla_34", tracking_task=tracking)
    opt.device = torch.device("cuda")
    det = ObjectPoseDetector.__new__(ObjectPoseDetector)
    det.opt, det.scales, det._slots = opt, opt.test_scales, None
    return det


@pytest.mark.parametrize("fmt", ("nv12", "i420"))
def test_run_batch_refuses_shapes_of_another_format(fmt):
    det = _host_detector()
    cam = np.eye(3)
    with pytest.raises(ValueError, match=r"%s frames are uint8 \[B,3H/2,W\], got torch.uint8 \(2, 480, 640, 3\)" % fmt):
        det.run_batch(np.zeros((2, 480, 640, 3), np.uint8), cam, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"each frame has shape \(721, 640\), expected a %s frame \[3H/2,W\]" % fmt):
        det.run_batch(np.zeros((2, 721, 640), np.uint8), cam, pixel_format=fmt)
    with pytest.raises(ValueError, match="got torch.float32"):
        det.run_batch(torch.zeros((2, 3, 64, 64)), cam, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"frame 1 has shape \(480, 640, 3\)"):
        det.run_batch([np.zeros((720, 640), np.uint8), np.zeros((480, 640, 3), np.uint8)], cam, pixel_format=fmt)
    with pytest.raises(ValueError, match="pixel_format must be one of"):
        det.run_batch([np.zeros((720, 640), np.uint8)], cam, pixel_format="yuv420")
    trk = _host_detector(tracking=True)
    with pytest.raises(ValueError, match=r"frame 0 has shape \(720, 642, 3\)"):
        trk.run_batch([np.zeros((720, 642, 3), np.uint8), None], cam, track=True, pixel_format=fmt)


def test_pipelines_refuse_bad_formats_before_device_work():
    det = _host_detector()
    with pytest.raises(ValueError, match="even"):
        cpb.BatchPipeline(det, batch=2, height=481, width=640, camera_matrix=np.eye(3), pixel_format="nv12")
    with pytest.raises(ValueError, match="pixel_format must be one of"):
        cpb.BatchPipeline(det, batch=2, height=480, width=640, camera_matrix=np.eye(3), pixel_format="rgb")
    with pytest.raises(ValueError, match="pixel_format must be one of"):
        cpb.TrackPipeline(_host_detector(tracking=True), slots=2, camera_matrix=np.eye(3), pixel_format="p010")
