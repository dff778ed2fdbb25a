"""Camera pixel formats without a GPU: the numpy restatements of cv2's RGB24 / RGBA / BGRA / YUYV / UYVY -> BGR
conversions against cv2 itself (packed 4:2:2 on a frame holding every (Y, U, V) triple) and through the warp against
cv2.warpAffine; the argument checks of cp_preprocess_formats, cp_preprocess_frame_table_formats and the new format
values of the graph-safe launches (CP_ERR_INVALID before any device work); and the pixel_format checks of run_batch,
the pipelines and the graphs, names and lists of names, all before any device work."""
import ctypes
import os

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.detector import ObjectPoseDetector, check_frames
from centerpose_b200.engine import frame_shape, image_size, slot_formats
from oracle import preprocess_ref
from tests import yuv422_ref
from tests.test_abi import ROOT, _declared_symbols

NEW = ("rgb24", "rgba", "bgra", "yuyv422", "uyvy422")
INVALID = -1


def _cv2_bgr(f, fmt):
    import cv2
    return cv2.cvtColor(f, getattr(cv2, yuv422_ref.CV2_CODES[fmt]))


def random_frame(h, w, fmt, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, yuv422_ref.CHANNELS[fmt]), dtype=np.uint8)


@pytest.mark.parametrize("fmt", ("yuyv422", "uyvy422"))
def test_oracle_is_cv2_on_every_yuv422_triple(fmt):
    f = yuv422_ref.exhaustive_yuv422(fmt)
    assert f.shape == (4096, 4096, 2)
    pairs = f.reshape(4096, 2048, 4).astype(np.int64)
    Y, U, V = ((pairs[..., [0, 2]], pairs[..., 1], pairs[..., 3]) if fmt == "yuyv422"
               else (pairs[..., [1, 3]], pairs[..., 0], pairs[..., 2]))
    # the frame holds each of the 2^24 (Y, U, V) triples, each pixel with its pair's chroma
    assert np.unique((Y << 16) | (U[..., None] << 8) | V[..., None]).size == 1 << 24
    assert np.array_equal(yuv422_ref.yuv422_to_bgr(f, fmt), _cv2_bgr(f, fmt))


@pytest.mark.parametrize("fmt", ("rgb24", "rgba", "bgra"))
@pytest.mark.parametrize("h, w", [(480, 640), (61, 77), (1, 5)])
def test_oracle_is_cv2_on_random_packed_rgb(fmt, h, w):
    f = random_frame(h, w, fmt, seed=h * w)
    assert np.array_equal(yuv422_ref.packed_to_bgr(f, fmt), _cv2_bgr(f, fmt))


def _rotated(h, w, inp):
    import cv2
    M = cv2.getRotationMatrix2D((w * 0.4, h * 0.55), 30.0, inp / (0.6 * max(h, w)))
    M[:, 2] += np.array([inp / 2. - w * 0.4, inp / 2. - h * 0.55])
    return M


@pytest.mark.parametrize("fmt", NEW)
@pytest.mark.parametrize("h, w, kind", [(48, 64, "fix_res"), (61, 80, "rotated"), (31, 46, "upscale")])
def test_oracle_warp_is_cv2_warp_of_cvtcolor(fmt, h, w, kind):
    import cv2
    f = random_frame(h, w, fmt, seed=h * w + len(fmt))
    inp = 64
    if kind == "fix_res":
        M = preprocess_ref.fix_res_affine(h, w, inp, inp)
    elif kind == "rotated":
        M = _rotated(h, w, inp)
    else:                                  # 3x up-scaling about a point near the border: taps straddle pixel pairs
        M = np.array([[3.1, 0.0, -3.1 * (w - 9.3)], [0.0, 2.9, -2.9 * 1.7]])
    want = cv2.warpAffine(_cv2_bgr(f, fmt), M, (inp, inp), flags=cv2.INTER_LINEAR)
    got = preprocess_ref.warp_affine_u8(yuv422_ref.to_bgr(f, fmt), M, inp, inp)
    assert np.array_equal(got, want)
    assert (want == 0).all(axis=-1).any(), "the affine keeps part of the output outside the frame"


def test_oracle_refuses_bad_frames():
    with pytest.raises(ValueError, match="W even"):
        yuv422_ref.yuv422_to_bgr(np.zeros((4, 5, 2), np.uint8), "yuyv422")
    with pytest.raises(ValueError, match="unknown format"):
        yuv422_ref.yuv422_to_bgr(np.zeros((4, 4, 2), np.uint8), "yuyv")
    with pytest.raises(ValueError, match=r"uint8 \[H, W, 4\]"):
        yuv422_ref.packed_to_bgr(np.zeros((4, 4, 3), np.uint8), "rgba")


# ---- the C ABI -----------------------------------------------------------------------------------------------------------
def test_entry_points_declared_exported_and_bound(cplib):
    for name in ("cp_preprocess_formats", "cp_preprocess_frame_table_formats"):
        assert name in _declared_symbols() and name in _lib.EXPORTS and hasattr(cplib, name), name
    assert (_lib.CP_PIX_NV12, _lib.CP_PIX_I420, _lib.CP_PIX_BGR) == (0, 1, 2)
    codes = [_lib.PIXEL_FORMAT_CODES[f] for f in _lib.PIXEL_FORMATS]
    assert len(set(codes)) == len(codes) == 8 and _lib.CP_PIX_PER_FRAME not in codes
    assert _lib.PIXEL_FORMATS[:3] == ("bgr", "nv12", "i420") and _lib.PIXEL_FORMATS[3:] == NEW
    with open(os.path.join(ROOT, "include", "centerpose_b200.h")) as fp:
        hdr = fp.read()
    for name in NEW + ("per_frame",):
        value = getattr(_lib, "CP_PIX_" + name.upper())
        assert "CP_PIX_%s = %d" % (name.upper(), value) in hdr, name


def _bytes(fmt, h, w):
    return h * w * 3 // 2 if fmt in (_lib.CP_PIX_NV12, _lib.CP_PIX_I420) else h * w * {
        _lib.CP_PIX_BGR: 3, _lib.CP_PIX_RGB24: 3, _lib.CP_PIX_RGBA: 4, _lib.CP_PIX_BGRA: 4, _lib.CP_PIX_YUYV422: 2,
        _lib.CP_PIX_UYVY422: 2}[fmt]


def _formats(cplib, hw, fmts, offsets=None, nbytes=None, frames=8, out=8, null=()):
    hw = np.ascontiguousarray(hw, np.int32).reshape(-1, 2)
    codes = np.ascontiguousarray(fmts, np.int32)
    per = [_bytes(f, h, w) if f in _lib.PIXEL_FORMAT_CODES.values() else 4 * h * w for f, (h, w) in zip(fmts, hw)]
    offs = np.ascontiguousarray(offsets if offsets is not None else np.concatenate([[0], np.cumsum(per)[:-1]]), np.int64)
    nbytes = int(sum(per)) if nbytes is None else nbytes
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    s = (ctypes.c_float * 3)(0.3, 0.3, 0.3)
    return cplib.cp_preprocess_formats(
        ctypes.c_void_p(frames), nbytes, None if "offsets" in null else offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
        None if "src_hw" in null else hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
        None if "formats" in null else codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), ctypes.c_void_p(out),
        len(offs), 64, 64, None, m, s, None)


def _table(cplib, hw, fmts, offsets=None, nbytes=None, null=()):
    hw = np.ascontiguousarray(hw, np.int32).reshape(-1, 2)
    codes = np.ascontiguousarray(fmts, np.int32)
    per = [_bytes(f, h, w) if f in _lib.PIXEL_FORMAT_CODES.values() else 4 * h * w for f, (h, w) in zip(fmts, hw)]
    offs = np.ascontiguousarray(offsets if offsets is not None else np.concatenate([[0], np.cumsum(per)[:-1]]), np.int64)
    nbytes = int(sum(per)) if nbytes is None else nbytes
    return cplib.cp_preprocess_frame_table_formats(
        nbytes, None if "offsets" in null else offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
        None if "src_hw" in null else hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
        None if "formats" in null else codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), len(offs), 64, 64, None,
        None if "table" in null else ctypes.c_void_p(8), None)


def _err(cplib):
    return cplib.cp_last_error()


@pytest.mark.parametrize("who, call", [("cp_preprocess_formats", _formats),
                                       ("cp_preprocess_frame_table_formats", _table)])
def test_per_frame_entry_points_validate_their_arguments(who, call, cplib):
    P = _lib
    hw, fmts = [(10, 10), (9, 12)], [P.CP_PIX_NV12, P.CP_PIX_RGBA]
    for what in (("offsets", "src_hw", "formats") + (("table",) if call is _table else ())):
        assert call(cplib, hw, fmts, null=(what,)) == INVALID and b"null argument" in _err(cplib), what
    if call is _formats:
        for kw in ({"frames": 0}, {"out": 0}):
            assert call(cplib, hw, fmts, **kw) == INVALID and b"null argument" in _err(cplib), kw
    assert call(cplib, hw, fmts, nbytes=0) == INVALID and b"bad shape" in _err(cplib)
    # unknown format values, the per-frame launch value among them
    for bad in (-1, 3, 7, 19, 34, P.CP_PIX_PER_FRAME):
        assert call(cplib, hw, [P.CP_PIX_BGR, bad]) == INVALID
        assert b"frame 1 has unknown pixel format %d" % bad in _err(cplib), bad
    # an odd width in 4:2:2 (an odd height is fine), an odd size in 4:2:0
    for f in (P.CP_PIX_YUYV422, P.CP_PIX_UYVY422):
        assert call(cplib, [(10, 10), (8, 7)], [P.CP_PIX_BGR, f]) == INVALID
        assert b"frame 1 has size 8 x 7 (YUV 4:2:2 needs an even width)" in _err(cplib)
    assert call(cplib, [(9, 10)], [P.CP_PIX_I420]) == INVALID and b"(YUV 4:2:0 needs even sizes)" in _err(cplib)
    assert call(cplib, [(10, 10), (0, 4)], fmts) == INVALID and b"frame 1 has size 0 x 4" in _err(cplib)
    # a frame overrunning the buffer at its own format's size: 10 x 10 is 150 bytes in NV12, 400 in RGBA
    assert call(cplib, hw, fmts, nbytes=150 + 9 * 12 * 4 - 1) == INVALID
    assert b"frame 1 (9 x 12 at byte 150) lies outside the 581-byte buffer" in _err(cplib)
    assert call(cplib, [(10, 10), (10, 10)], [P.CP_PIX_RGBA, P.CP_PIX_YUYV422], nbytes=599) == INVALID
    assert b"outside" in _err(cplib)
    assert call(cplib, hw, fmts, offsets=[-1, 150]) == INVALID and b"outside" in _err(cplib)
    assert who.encode() in _err(cplib)


def test_single_format_launches_take_the_new_values(cplib):
    """cp_preprocess_slots_dev / _frame_table / _slots_ragged_dev / _slots_rows_dev accept the five values (their
    argument checks pass up to the first device-side step, which a null pointer then stops) and check 4:2:2 widths."""
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    s = (ctypes.c_float * 3)(0.3, 0.3, 0.3)
    for f in NEW:
        code = _lib.PIXEL_FORMAT_CODES[f]
        assert cplib.cp_preprocess_slots_dev(ctypes.c_void_p(8), code, 2, 64, 64, 32, 32, None, None, s, None,
                                             ctypes.c_void_p(8), None, None) == INVALID
        assert b"null argument" in _err(cplib)                  # past nothing: mean is null; the format is not named
        hw = np.array([[10, 10]], np.int32)
        offs = np.zeros(1, np.int64)
        rc = cplib.cp_preprocess_frame_table(_bytes(code, 10, 10), offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                             hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), code, 1, 32, 32, None,
                                             None, None)
        assert rc == INVALID and b"null argument" in _err(cplib)
        assert cplib.cp_preprocess_slots_ragged_dev(ctypes.c_void_p(8), ctypes.c_void_p(8), code, 0, 32, 32, m, s,
                                                    None, ctypes.c_void_p(8), None, None) == INVALID
        assert b"cp_preprocess_slots_ragged_dev: bad shape" in _err(cplib), f        # the format passed its check
        assert cplib.cp_preprocess_slots_rows_dev(ctypes.c_void_p(8), ctypes.c_void_p(8), code, ctypes.c_void_p(8), 0,
                                                  32, 32, m, s, None, None, ctypes.c_void_p(8), None, None) == INVALID
        assert b"cp_preprocess_slots_rows_dev: bad shape" in _err(cplib), f
        assert cplib.cp_preprocess_slots_dev(ctypes.c_void_p(8), code, 0, 64, 64, 32, 32, None, m, s, None,
                                             ctypes.c_void_p(8), None, None) == INVALID
        assert b"cp_preprocess_slots_dev: bad shape" in _err(cplib), f
    for code in (_lib.CP_PIX_YUYV422, _lib.CP_PIX_UYVY422):
        assert cplib.cp_preprocess_slots_dev(ctypes.c_void_p(8), code, 2, 63, 65, 32, 32, None, m, s, None,
                                             ctypes.c_void_p(8), None, None) == INVALID
        assert b"YUV 4:2:2 frames need an even width, got 63 x 65" in _err(cplib)
        hw = np.array([[10, 9]], np.int32)
        offs = np.zeros(1, np.int64)
        assert cplib.cp_preprocess_frame_table(180, offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                               hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), code, 1, 32, 32, None,
                                               ctypes.c_void_p(8), None) == INVALID
        assert b"frame 0 has size 10 x 9 (YUV 4:2:2 needs an even width)" in _err(cplib)
    # the per-frame launch value is a table launch only
    P = _lib.CP_PIX_PER_FRAME
    assert cplib.cp_preprocess_slots_dev(ctypes.c_void_p(8), P, 2, 64, 64, 32, 32, None, m, s, None,
                                         ctypes.c_void_p(8), None, None) == INVALID
    assert b"unknown pixel format %d" % P in _err(cplib)
    hw, offs = np.array([[10, 10]], np.int32), np.zeros(1, np.int64)
    assert cplib.cp_preprocess_frame_table(300, offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                           hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), P, 1, 32, 32, None,
                                           ctypes.c_void_p(8), None) == INVALID
    assert b"unknown pixel format %d" % P in _err(cplib)
    assert cplib.cp_preprocess_slots_ragged_dev(ctypes.c_void_p(8), ctypes.c_void_p(8), P, 0, 32, 32, m, s, None,
                                                ctypes.c_void_p(8), None, None) == INVALID
    assert b"bad shape" in _err(cplib)


# ---- pixel_format in the Python layer --------------------------------------------------------------------------------
def test_frame_shapes_of_the_camera_formats():
    assert frame_shape(480, 640, "rgb24") == (480, 640, 3)
    assert frame_shape(480, 640, "rgba") == frame_shape(480, 640, "bgra") == (480, 640, 4)
    assert frame_shape(481, 640, "yuyv422") == frame_shape(481, 640, "uyvy422") == (481, 640, 2)
    with pytest.raises(ValueError, match="yuyv422 frames need an even, positive width; got 480 x 641"):
        frame_shape(480, 641, "yuyv422")
    assert image_size((481, 640, 2), "uyvy422") == (481, 640) and image_size((5, 7, 4), "bgra") == (5, 7)
    assert image_size((5, 7, 3), "rgb24") == (5, 7)
    with pytest.raises(ValueError, match=r"expected a uyvy422 frame \[H,W,2\] with W even"):
        image_size((480, 641, 2), "uyvy422")
    with pytest.raises(ValueError, match=r"expected a rgba frame \[H,W,4\]"):
        image_size((480, 640, 3), "rgba")
    with pytest.raises(ValueError, match=r"expected \[H,W,3\]"):
        image_size((480, 640, 4), "rgb24")
    # the names are ffmpeg's; others (and a case change) are refused, the message listing bgr, nv12, i420 first
    for bad in ("yuyv", "rgb", "RGB24", "yuv422", "uyvy", "bgrx", "p010"):
        with pytest.raises(ValueError, match="pixel_format must be one of bgr, nv12, i420, rgb24, rgba, bgra, yuyv422, "
                                             "uyvy422"):
            frame_shape(480, 640, bad)


def test_lists_of_names():
    assert slot_formats("rgb24", 3) == ["rgb24"] * 3
    assert slot_formats(["nv12", "yuyv422"], 2) == ["nv12", "yuyv422"]
    with pytest.raises(ValueError, match="one name or one per frame, got 3 names for 2 frames"):
        slot_formats(["bgr"] * 3, 2)
    with pytest.raises(ValueError, match=r"pixel_format must be one of .*got 'yuyv' in \['bgr', 'yuyv'\]"):
        slot_formats(["bgr", "yuyv"], 2)
    with pytest.raises(ValueError, match="pixel_format must be one name here, got a list"):
        frame_shape(480, 640, ["bgr"])


def test_check_frames_per_format_and_per_frame():
    check_frames([np.zeros((5, 6, 2), np.uint8), torch.zeros((4, 4, 4), dtype=torch.uint8), None], allow_idle=True,
                 pixel_format=["yuyv422", "rgba", "nv12"])
    check_frames([np.zeros((5, 6, 3), np.uint8)] * 2, allow_idle=False, pixel_format=["rgb24", "bgr"])
    with pytest.raises(ValueError, match=r"frame 1 has shape \(4, 6, 3\), expected a uyvy422 frame \[H,W,2\]"):
        check_frames([np.zeros((6, 4), np.uint8), np.zeros((4, 6, 3), np.uint8)], allow_idle=False,
                     pixel_format=["nv12", "uyvy422"])
    with pytest.raises(ValueError, match=r"frame 0 has shape \(4, 5, 2\), expected a yuyv422 frame \[H,W,2\] with W"):
        check_frames([np.zeros((4, 5, 2), np.uint8)], allow_idle=False, pixel_format="yuyv422")
    with pytest.raises(TypeError, match=r"uint8 \[H,W,4\]"):
        check_frames([np.zeros((4, 4, 4), np.float32)], allow_idle=False, pixel_format="bgra")
    with pytest.raises(ValueError, match="2 names for 3 frames"):
        check_frames([np.zeros((4, 4, 3), np.uint8)] * 3, allow_idle=False, pixel_format=["bgr", "rgb24"])


def _host_detector(tracking=False):
    """An ObjectPoseDetector that only gets as far as its argument checks (no model, no device work)."""
    opt = cpb.default_opt("dla_34", tracking_task=tracking)
    opt.device = torch.device("cuda")
    det = ObjectPoseDetector.__new__(ObjectPoseDetector)
    det.opt, det.scales, det._slots = opt, opt.test_scales, None
    return det


@pytest.mark.parametrize("fmt", NEW)
def test_run_batch_refuses_shapes_of_another_format(fmt):
    det = _host_detector()
    cam = np.eye(3)
    c = yuv422_ref.CHANNELS[fmt]
    with pytest.raises(ValueError, match=r"%s frames are uint8 \[B,H,W,%d\], got torch.uint8 \(2, 720, 640\)" % (fmt, c)):
        det.run_batch(np.zeros((2, 720, 640), np.uint8), cam, pixel_format=fmt)
    other = 3 if c != 3 else 4
    with pytest.raises(ValueError, match=r"each frame has shape \(480, 640, %d\)" % other):
        det.run_batch(np.zeros((2, 480, 640, other), np.uint8), cam, pixel_format=fmt)
    with pytest.raises(ValueError, match="got torch.float32"):
        det.run_batch(torch.zeros((2, 3, 64, 64)), cam, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"frame 1 has shape \(720, 640\)"):
        det.run_batch([np.zeros((480, 640, c), np.uint8), np.zeros((720, 640), np.uint8)], cam, pixel_format=fmt)
    trk = _host_detector(tracking=True)
    with pytest.raises(ValueError, match=r"frame 0 has shape \(720, 642\)"):
        trk.run_batch([np.zeros((720, 642), np.uint8), None], cam, track=True, pixel_format=fmt)


def test_lists_go_with_lists_of_frames_only():
    det, trk, cam = _host_detector(), _host_detector(tracking=True), np.eye(3)
    one = r"pixel_format must be one name here, got a list \['bgr', 'rgb24'\]"
    with pytest.raises(ValueError, match=one):
        det.run_batch(np.zeros((2, 480, 640, 3), np.uint8), cam, pixel_format=["bgr", "rgb24"])
    with pytest.raises(ValueError, match=one):
        trk.run_batch(np.zeros((2, 480, 640, 3), np.uint8), cam, track=True, pixel_format=["bgr", "rgb24"])
    with pytest.raises(ValueError, match="got 1 names for 2 frames"):
        det.run_batch([np.zeros((480, 640, 3), np.uint8)] * 2, cam, pixel_format=["bgr"])
    with pytest.raises(ValueError, match="got 2 names for 3 frames"):
        trk.run_batch([np.zeros((480, 640, 3), np.uint8), None, None], cam, track=True, pixel_format=["bgr", "bgr"])
    with pytest.raises(ValueError, match=r"frame 1 has shape \(480, 640, 3\), expected a bgra frame"):
        trk.run_batch([np.zeros((480, 640, 3), np.uint8), np.zeros((480, 640, 3), np.uint8)], cam, track=True,
                      pixel_format=["rgb24", "bgra"])
    with pytest.raises(ValueError, match=one):
        cpb.BatchPipeline(det, batch=2, height=480, width=640, camera_matrix=cam, pixel_format=["bgr", "rgb24"])
    with pytest.raises(ValueError, match=one):
        cpb.TrackPipeline(trk, slots=2, camera_matrix=cam, pixel_format=["bgr", "rgb24"])
    with pytest.raises(ValueError, match="yuyv422 frames need an even, positive width; got 480 x 641"):
        cpb.BatchPipeline(det, batch=2, height=480, width=641, camera_matrix=cam, pixel_format="yuyv422")


def _multi_shell(cls):
    det = cls.__new__(cls)
    det.opt = cpb.default_opt("dla_34", tracking_task=cls in (cpb.MultiCategoryTracker,))
    det.categories = ["chair", "cup"]
    return det


def _det_shell(tracking):
    det = ObjectPoseDetector.__new__(ObjectPoseDetector)
    det.opt = cpb.default_opt("dla_34", tracking_task=tracking)
    return det


@pytest.mark.parametrize("cls, make", [
    (cpb.TrackGraph, lambda: _det_shell(True)), (cpb.DetectGraph, lambda: _det_shell(False)),
    (cpb.MultiCategoryTrackGraph, lambda: _multi_shell(cpb.MultiCategoryTracker)),
    (cpb.MultiCategoryDetectGraph, lambda: _multi_shell(cpb.MultiCategoryDetector))])
def test_graphs_check_formats_before_device_work(cls, make, monkeypatch):
    # nothing below may reach the library
    monkeypatch.setattr(_lib, "load", lambda: (_ for _ in ()).throw(AssertionError("the library was loaded")))
    name = cls.__name__
    with pytest.raises(ValueError, match="%s: one pixel_format per slot goes with one frame_hw per slot" % name):
        cls(make(), slots=2, frame_hw=(480, 640), camera_matrix=np.eye(3), pixel_format=["bgr", "rgb24"])
    with pytest.raises(ValueError, match="%s: pixel_format is one name or one per frame, got 3 names for 2" % name):
        cls(make(), slots=2, frame_hw=[(480, 640), (720, 1280)], camera_matrix=np.eye(3),
            pixel_format=["bgr", "rgb24", "bgr"])
    with pytest.raises(ValueError, match="pixel_format must be one of .* got 'yuyv' in"):
        cls(make(), slots=2, frame_hw=[(480, 640), (720, 1280)], camera_matrix=np.eye(3), pixel_format=["bgr", "yuyv"])
    with pytest.raises(ValueError, match="uyvy422 frames need an even, positive width; got 720 x 1279"):
        cls(make(), slots=2, frame_hw=[(480, 640), (720, 1279)], camera_matrix=np.eye(3),
            pixel_format=["nv12", "uyvy422"])
    with pytest.raises(ValueError, match="yuyv422 frames need an even, positive width; got 480 x 641"):
        cls(make(), slots=2, frame_hw=(480, 641), camera_matrix=np.eye(3), pixel_format="yuyv422")
    with pytest.raises(ValueError, match="pixel_format must be one of bgr, nv12, i420"):
        cls(make(), slots=2, frame_hw=(480, 640), camera_matrix=np.eye(3), pixel_format="rgb")
