"""Sensor formats ("gray" and the Bayer mosaics) without a GPU: the numpy restatement of cv2's conversions to BGR
(tests/bayer_ref.py) against cv2 itself, on random frames down to 3 x 3 and on 0 / 255 frames that put every rounding
case on every site, and through the warp against cv2.warpAffine; the header / _lib agreement of the five codes; the
CP_ERR_INVALID refusals before any device work; and the shape, name and list checks of the Python layer."""
import ctypes
import os

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.detector import check_frames
from centerpose_b200.engine import frame_layout, frame_shape, image_size, slot_formats
from oracle import preprocess_ref
from tests import bayer_ref
from tests.test_abi import ROOT
from tests.test_pixel_formats_cpu import _det_shell, _host_detector, _multi_shell

INVALID = -1
SENSOR = bayer_ref.FORMATS
SIZES = [(3, 3), (3, 4), (3, 8), (4, 4), (5, 3), (6, 8), (7, 5), (33, 47), (64, 96)]


def _cv2_bgr(f, fmt):
    import cv2
    return cv2.cvtColor(f, getattr(cv2, bayer_ref.CV2_CODES[fmt]))


@pytest.mark.parametrize("fmt", SENSOR)
@pytest.mark.parametrize("h, w", SIZES)
def test_oracle_is_cv2_on_random_frames(fmt, h, w):
    f = np.random.default_rng(h * 100 + w).integers(0, 256, (h, w), dtype=np.uint8)
    assert np.array_equal(bayer_ref.to_bgr(f, fmt), _cv2_bgr(f, fmt))


@pytest.mark.parametrize("fmt", bayer_ref.BAYER)
@pytest.mark.parametrize("h, w", [(3, 3), (4, 5), (8, 8), (9, 11)])
def test_oracle_is_cv2_on_every_rounding_case(fmt, h, w):
    frames = bayer_ref.rounding_frames(h, w)
    for k, f in enumerate(frames):
        assert np.array_equal(bayer_ref.bayer_to_bgr(f, fmt), _cv2_bgr(f, fmt)), k
    if min(h, w) >= 8:                     # room for every case: the averages of one to four 255s come out
        conv = np.stack([bayer_ref.bayer_to_bgr(f, fmt) for f in frames])
        assert {int(v) for v in np.unique(conv)} == {0, 64, 128, 191, 255}


def test_oracle_phases_and_refusals():
    # the patterns are one mosaic shifted: rggb by one column is grbg, by one row gbrg, by both bggr
    f = np.random.default_rng(3).integers(0, 256, (12, 14), dtype=np.uint8)
    rggb = bayer_ref.bayer_to_bgr(f, "bayer_rggb8")
    for fmt, (dy, dx) in (("bayer_grbg8", (0, 1)), ("bayer_gbrg8", (1, 0)), ("bayer_bggr8", (1, 1))):
        shifted = bayer_ref.bayer_to_bgr(f[dy:, dx:], fmt)
        assert np.array_equal(shifted[1:-1, 1:-1], rggb[dy + 1:-1, dx + 1:-1]), fmt
    # the mosaics from_bgr makes carry each site's own channel
    bgr = np.random.default_rng(4).integers(0, 256, (6, 8, 3), dtype=np.uint8)
    raw = bayer_ref.from_bgr(bgr, "bayer_rggb8")
    assert raw[0, 0] == bgr[0, 0, 2] and raw[0, 1] == bgr[0, 1, 1] and raw[1, 1] == bgr[1, 1, 0]
    with pytest.raises(ValueError, match="at least 3"):
        bayer_ref.bayer_to_bgr(np.zeros((2, 5), np.uint8), "bayer_rggb8")
    with pytest.raises(ValueError, match="unknown format"):
        bayer_ref.bayer_to_bgr(np.zeros((4, 4), np.uint8), "bayer_rgbg8")


def _rotated(h, w, inp):
    import cv2
    M = cv2.getRotationMatrix2D((w * 0.4, h * 0.55), 30.0, inp / (0.6 * max(h, w)))
    M[:, 2] += np.array([inp / 2. - w * 0.4, inp / 2. - h * 0.55])
    return M


@pytest.mark.parametrize("fmt", SENSOR)
@pytest.mark.parametrize("h, w, kind", [(48, 64, "fix_res"), (61, 80, "rotated"), (31, 46, "upscale"),
                                        (5, 7, "fix_res"), (150, 97, "downscale")])
def test_oracle_warp_is_cv2_warp_of_cvtcolor(fmt, h, w, kind):
    import cv2
    f = np.random.default_rng(h * w + len(fmt)).integers(0, 256, (h, w), dtype=np.uint8)
    inp = 64
    if kind == "fix_res":
        M = preprocess_ref.fix_res_affine(h, w, inp, inp)
    elif kind == "rotated":
        M = _rotated(h, w, inp)
    elif kind == "upscale":                # 3x about a point near the border: taps straddle the border pixels
        M = np.array([[3.1, 0.0, -3.1 * (w - 9.3)], [0.0, 2.9, -2.9 * 1.7]])
    else:                                  # shrink and shift: the frame ends inside the output on two sides
        M = np.array([[0.37, 0.0, 9.5], [0.0, 0.31, 7.25]])
    want = cv2.warpAffine(_cv2_bgr(f, fmt), M, (inp, inp), flags=cv2.INTER_LINEAR)
    got = preprocess_ref.warp_affine_u8(bayer_ref.to_bgr(f, fmt), M, inp, inp)
    assert np.array_equal(got, want)
    assert (want == 0).all(axis=-1).any(), "the affine keeps part of the output outside the frame"


# ---- the C ABI -----------------------------------------------------------------------------------------------------------
def test_codes_agree_with_the_header():
    with open(os.path.join(ROOT, "include", "centerpose_b200.h")) as fp:
        hdr = fp.read()
    assert _lib.SENSOR_FORMATS == SENSOR
    codes = [_lib.PIXEL_FORMAT_CODES[f] for f in SENSOR]
    assert codes == [48, 49, 50, 51, 52]
    for f in SENSOR:
        assert "CP_PIX_%s = %d" % (f.upper(), _lib.PIXEL_FORMAT_CODES[f]) in hdr, f
    colour = [_lib.PIXEL_FORMAT_CODES[f] for f in _lib.PIXEL_FORMATS]
    assert not set(codes) & set(colour + [_lib.CP_PIX_PER_FRAME, _lib.CP_PIX_REMAP])
    assert all(c < 64 and not c & (1 << 6) for c in codes)                     # bit 6 is a table entry's mapped flag
    assert all(c | _lib.CP_PIX_REMAP != c and (c | _lib.CP_PIX_REMAP) & ~_lib.CP_PIX_REMAP == c for c in codes)


def _err(cplib):
    return cplib.cp_last_error()


def _args(hw, fmts, offsets, null):
    hw = np.ascontiguousarray(hw, np.int32).reshape(-1, 2)
    codes = np.ascontiguousarray(fmts, np.int32)
    offs = np.ascontiguousarray(offsets, np.int64)
    return (None if "offsets" in null else offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
            None if "src_hw" in null else hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
            codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), len(offs)), (hw, codes, offs)


def _formats(cplib, hw, fmts, offsets, nbytes, null=()):
    (offs, hws, codes, B), keep = _args(hw, fmts, offsets, null)
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    return cplib.cp_preprocess_formats(ctypes.c_void_p(8), nbytes, offs, hws, codes, ctypes.c_void_p(8), B, 64, 64,
                                       None, m, m, None)


def _table(cplib, hw, fmts, offsets, nbytes, null=()):
    (offs, hws, codes, B), keep = _args(hw, fmts, offsets, null)
    return cplib.cp_preprocess_frame_table_formats(nbytes, offs, hws, codes, B, 64, 64, None, ctypes.c_void_p(8), None)


@pytest.mark.parametrize("who, call", [("cp_preprocess_formats", _formats),
                                       ("cp_preprocess_frame_table_formats", _table)])
def test_per_frame_entry_points_refuse_bad_sensor_frames(who, call, cplib):
    P = _lib
    for code in (P.CP_PIX_BAYER_RGGB8, P.CP_PIX_BAYER_BGGR8, P.CP_PIX_BAYER_GBRG8, P.CP_PIX_BAYER_GRBG8):
        for h, w in ((2, 5), (5, 2), (2, 2), (1, 1)):
            assert call(cplib, [(10, 10), (h, w)], [P.CP_PIX_BGR, code], [0, 300], 1000) == INVALID
            assert b"frame 1 has size %d x %d (a Bayer mosaic needs at least 3 x 3)" % (h, w) in _err(cplib)
            assert who.encode() in _err(cplib)
    # a frame overrunning the buffer at H * W bytes: 10 x 10 BGR is 300 bytes, a 9 x 12 mosaic or gray frame 108
    for code in (P.CP_PIX_GRAY, P.CP_PIX_BAYER_GBRG8):
        assert call(cplib, [(10, 10), (9, 12)], [P.CP_PIX_BGR, code], [0, 300], 300 + 108 - 1) == INVALID
        assert b"frame 1 (9 x 12 at byte 300) lies outside the 407-byte buffer" in _err(cplib)
        assert call(cplib, [(9, 12)], [code], [-1], 1000) == INVALID and b"outside" in _err(cplib)
    assert call(cplib, [(1, 1)], [P.CP_PIX_GRAY], [0], 0) == INVALID and b"bad shape" in _err(cplib)
    assert call(cplib, [(10, 10)], [P.CP_PIX_GRAY], [0], 100, null=("offsets",)) == INVALID
    assert b"null argument" in _err(cplib)


def test_single_format_launches_take_the_sensor_codes(cplib):
    """cp_preprocess_slots_dev / _frame_table / _slots_ragged_dev / _slots_rows_dev / _remap / _frame_table_maps accept
    the five values (their checks pass up to a later one) and check a mosaic's size; cp_preprocess_yuv420 refuses them."""
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    v = ctypes.c_void_p(8)
    hw, offs = np.array([[10, 10]], np.int32), np.zeros(1, np.int64)
    HW, OFFS = hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
    for f in SENSOR:
        code = _lib.PIXEL_FORMAT_CODES[f]
        assert cplib.cp_preprocess_slots_dev(v, code, 0, 64, 64, 32, 32, None, m, m, None, v, None, None) == INVALID
        assert b"cp_preprocess_slots_dev: bad shape" in _err(cplib), f              # the format passed its check
        assert cplib.cp_preprocess_frame_table(100, OFFS, HW, code, 1, 32, 32, None, None, None) == INVALID
        assert b"null argument" in _err(cplib)
        assert cplib.cp_preprocess_frame_table(99, OFFS, HW, code, 1, 32, 32, None, v, None) == INVALID
        assert b"frame 0 (10 x 10 at byte 0) lies outside the 99-byte buffer" in _err(cplib), f
        for launch in (code, code | _lib.CP_PIX_REMAP):
            assert cplib.cp_preprocess_slots_ragged_dev(v, v, launch, 0, 32, 32, m, m, None, v, None, None) == INVALID
            assert b"cp_preprocess_slots_ragged_dev: bad shape" in _err(cplib), launch
            assert cplib.cp_preprocess_slots_rows_dev(v, v, launch, v, 0, 32, 32, m, m, None, None, v, None,
                                                      None) == INVALID
            assert b"cp_preprocess_slots_rows_dev: bad shape" in _err(cplib), launch
        codes = np.array([code], np.int32)
        maps = (ctypes.c_void_p * 1)(12)                                          # misaligned: the last check
        rc = cplib.cp_preprocess_remap(v, 100, OFFS, HW, codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), maps, v,
                                       1, 32, 32, None, m, m, None)
        assert rc == INVALID and b"map of frame 0 is not 8-byte aligned" in _err(cplib), f
        rc = cplib.cp_preprocess_frame_table_maps(100, OFFS, HW, code, None, maps, 1, 32, 32, None, v, None)
        assert rc == INVALID and b"map of frame 0 is not 8-byte aligned" in _err(cplib), f
        rc = cplib.cp_preprocess_yuv420(v, 100, OFFS, HW, code, v, 1, 32, 32, None, m, m, None)
        assert rc == INVALID and b"cp_preprocess_yuv420: unknown pixel format %d" % code in _err(cplib), f
    for f in bayer_ref.BAYER:
        code = _lib.PIXEL_FORMAT_CODES[f]
        for h, w in ((2, 64), (64, 2)):
            assert cplib.cp_preprocess_slots_dev(v, code, 2, h, w, 32, 32, None, m, m, None, v, None, None) == INVALID
            assert b"Bayer mosaics need at least 3 x 3, got %d x %d" % (h, w) in _err(cplib)
    # a gray frame may be any positive size
    assert cplib.cp_preprocess_slots_dev(v, _lib.CP_PIX_GRAY, 0, 1, 1, 32, 32, None, m, m, None, v, None,
                                         None) == INVALID
    assert b"bad shape" in _err(cplib)


# ---- pixel_format in the Python layer --------------------------------------------------------------------------------
def test_shapes_of_the_sensor_formats():
    for f in SENSOR:
        assert frame_shape(1200, 1920, f) == (1200, 1920) and frame_layout(f) == "[H,W]"
        assert image_size((1201, 1921), f) == (1201, 1921)
        with pytest.raises(ValueError, match=r"expected a %s frame \[H,W\]" % f):
            image_size((1200, 1920, 1), f)
    assert frame_shape(1, 1, "gray") == (1, 1) and image_size((1, 2), "gray") == (1, 2)
    for f in bayer_ref.BAYER:
        assert frame_shape(3, 3, f) == (3, 3)
        with pytest.raises(ValueError, match="%s frames need at least 3 x 3 pixels; got 2 x 640" % f):
            frame_shape(2, 640, f)
        with pytest.raises(ValueError, match=r"expected a %s frame \[H,W\] with H and W at least 3" % f):
            image_size((640, 2), f)
    # a 2-D shape is 4:2:0 only in a 4:2:0 format
    assert image_size((720, 640), "nv12") == (480, 640) and image_size((720, 640), "gray") == (720, 640)
    # the refusal lists the colour formats first, then the sensor formats
    for bad in ("mono8", "bayer_rggb", "BAYER_RGGB8", "grey", "bayer_rggb16"):
        with pytest.raises(ValueError, match="pixel_format must be one of bgr, nv12, i420, rgb24, rgba, bgra, yuyv422, "
                                             "uyvy422, gray, bayer_rggb8, bayer_bggr8, bayer_gbrg8, bayer_grbg8, got"):
            frame_shape(480, 640, bad)


def test_lists_and_check_frames():
    assert slot_formats(["bayer_rggb8", "nv12", "gray", "bgr"], 4) == ["bayer_rggb8", "nv12", "gray", "bgr"]
    with pytest.raises(ValueError, match=r"got 'mono8' in \['gray', 'mono8'\]"):
        slot_formats(["gray", "mono8"], 2)
    check_frames([np.zeros((5, 6), np.uint8), torch.zeros((4, 4, 3), dtype=torch.uint8), None, np.zeros((3, 3), np.uint8)],
                 allow_idle=True, pixel_format=["gray", "bgr", "nv12", "bayer_bggr8"])
    with pytest.raises(ValueError, match=r"frame 1 has shape \(480, 640, 3\), expected a bayer_rggb8 frame \[H,W\]"):
        check_frames([np.zeros((6, 4), np.uint8), np.zeros((480, 640, 3), np.uint8)], allow_idle=False,
                     pixel_format=["nv12", "bayer_rggb8"])
    with pytest.raises(ValueError, match=r"frame 0 has shape \(2, 9\), expected a bayer_grbg8 frame \[H,W\] with H"):
        check_frames([np.zeros((2, 9), np.uint8)], allow_idle=False, pixel_format="bayer_grbg8")
    with pytest.raises(TypeError, match=r"uint8 \[H,W\]"):
        check_frames([np.zeros((4, 4), np.float32)], allow_idle=False, pixel_format="gray")


@pytest.mark.parametrize("fmt", SENSOR)
def test_run_batch_refuses_shapes_of_another_format(fmt):
    det, trk, cam = _host_detector(), _host_detector(tracking=True), np.eye(3)
    with pytest.raises(ValueError, match=r"%s frames are uint8 \[B,H,W\], got torch.uint8 \(2, 480, 640, 3\)" % fmt):
        det.run_batch(np.zeros((2, 480, 640, 3), np.uint8), cam, pixel_format=fmt)
    with pytest.raises(ValueError, match="got torch.float32"):
        det.run_batch(torch.zeros((2, 3, 64, 64)), cam, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"frame 1 has shape \(480, 640, 1\)"):
        det.run_batch([np.zeros((480, 640), np.uint8), np.zeros((480, 640, 1), np.uint8)], cam, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"frame 0 has shape \(720, 642, 3\)"):
        trk.run_batch([np.zeros((720, 642, 3), np.uint8), None], cam, track=True, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"pixel_format must be one name here, got a list"):
        det.run_batch(np.zeros((2, 480, 640), np.uint8), cam, pixel_format=[fmt, "bgr"])
    with pytest.raises(ValueError, match="got 1 names for 2 frames"):
        trk.run_batch([np.zeros((480, 640), np.uint8)] * 2, cam, track=True, pixel_format=[fmt])


def test_pipelines_check_sensor_sizes():
    det, cam = _host_detector(), np.eye(3)
    with pytest.raises(ValueError, match="bayer_rggb8 frames need at least 3 x 3 pixels; got 2 x 640"):
        cpb.BatchPipeline(det, batch=2, height=2, width=640, camera_matrix=cam, pixel_format="bayer_rggb8")
    with pytest.raises(ValueError, match=r"pixel_format must be one name here, got a list \['gray', 'bgr'\]"):
        cpb.TrackPipeline(_host_detector(tracking=True), slots=2, camera_matrix=cam, pixel_format=["gray", "bgr"])


@pytest.mark.parametrize("cls, make", [
    (cpb.TrackGraph, lambda: _det_shell(True)), (cpb.DetectGraph, lambda: _det_shell(False)),
    (cpb.MultiCategoryTrackGraph, lambda: _multi_shell(cpb.MultiCategoryTracker)),
    (cpb.MultiCategoryDetectGraph, lambda: _multi_shell(cpb.MultiCategoryDetector))])
def test_graphs_check_sensor_formats_before_device_work(cls, make, monkeypatch):
    monkeypatch.setattr(_lib, "load", lambda: (_ for _ in ()).throw(AssertionError("the library was loaded")))
    name = cls.__name__
    with pytest.raises(ValueError, match="bayer_gbrg8 frames need at least 3 x 3 pixels; got 2 x 1279"):
        cls(make(), slots=2, frame_hw=[(480, 640), (2, 1279)], camera_matrix=np.eye(3),
            pixel_format=["gray", "bayer_gbrg8"])
    with pytest.raises(ValueError, match="bayer_bggr8 frames need at least 3 x 3 pixels; got 480 x 2"):
        cls(make(), slots=2, frame_hw=(480, 2), camera_matrix=np.eye(3), pixel_format="bayer_bggr8")
    with pytest.raises(ValueError, match="%s: one pixel_format per slot goes with one frame_hw per slot" % name):
        cls(make(), slots=2, frame_hw=(480, 640), camera_matrix=np.eye(3), pixel_format=["gray", "bayer_rggb8"])
    with pytest.raises(ValueError, match="pixel_format must be one of .* got 'mono8' in"):
        cls(make(), slots=2, frame_hw=[(480, 640), (720, 1280)], camera_matrix=np.eye(3), pixel_format=["gray", "mono8"])
