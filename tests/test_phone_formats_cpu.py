"""Phone camera formats without a GPU: the full-range rule of tests/phone_ref.py against cv2 on every (Y, Cr, Cb), and
the numpy restatement of all six formats against cv2 on random frames down to 2 x 2; the header / _lib agreement of the
codes; the CP_ERR_INVALID refusals before any device work; the Python shape, name and list checks; and the checks of a
per-step camera_matrix in the live-video graphs."""
import ctypes
import os

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.detector import check_frames
from centerpose_b200.engine import frame_layout, frame_shape, image_size, slot_formats
from centerpose_b200.graph import _SlotGraph
from tests import phone_ref
from tests.test_abi import ROOT
from tests.test_pixel_formats_cpu import _det_shell, _host_detector, _multi_shell

INVALID = -1
PHONE = phone_ref.FORMATS
SIZES = [(2, 2), (2, 8), (6, 2), (4, 6), (10, 14), (34, 46), (64, 96)]


def test_full_range_rule_is_cv2_on_every_triple():
    import cv2
    ycc = phone_ref.exhaustive_triples()
    want = cv2.cvtColor(ycc, cv2.COLOR_YCrCb2BGR)
    got = phone_ref.full_range_to_bgr(ycc[..., 0], ycc[..., 2], ycc[..., 1])
    assert np.array_equal(got, want)


@pytest.mark.parametrize("fmt", PHONE + ("nv12", "i420"))
@pytest.mark.parametrize("h, w", SIZES)
def test_oracle_is_cv2_on_random_frames(fmt, h, w):
    f = np.random.default_rng(h * 100 + w + len(fmt)).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    assert np.array_equal(phone_ref.to_bgr(f, fmt), phone_ref.cv2_bgr(f, fmt))


@pytest.mark.parametrize("h, w", SIZES)
def test_swapped_chroma_is_cv2s_nv12_and_i420(h, w):
    """COLOR_YUV2BGR_NV21 / _YV12 are NV12 / I420 on the frame with its chroma swapped, and a full-range frame's layout
    carries the same planes whichever of the four it is."""
    import cv2
    f = np.random.default_rng(7 * h + w).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    for swapped, base in (("nv21", "nv12"), ("yv12", "i420")):
        Y, U, V = phone_ref.planes(f, swapped)
        assert np.array_equal(cv2.cvtColor(f, getattr(cv2, phone_ref.CV2_CODES[swapped])),
                              cv2.cvtColor(phone_ref.pack(Y, U, V, base), getattr(cv2, phone_ref.CV2_CODES[base])))
        assert np.array_equal(phone_ref.pack(Y, U, V, swapped), f)
    Y, U, V = phone_ref.planes(f, "nv12_full")
    want = phone_ref.to_bgr(f, "nv12_full")
    for fmt in ("nv21_full", "i420_full", "yv12_full"):
        assert np.array_equal(phone_ref.to_bgr(phone_ref.pack(Y, U, V, fmt), fmt), want), fmt


def test_from_bgr_is_a_camera_frame():
    yy, xx = np.mgrid[0:48, 0:64]
    bgr = np.dstack([4 * xx, 40 + 3 * yy, 200 - 2 * xx - yy]).astype(np.uint8)       # smooth: chroma survives 4:2:0
    for fmt in PHONE:
        f = phone_ref.from_bgr(bgr, fmt)
        assert f.shape == (72, 64) and f.dtype == np.uint8
        # the conversion back is the image up to subsampling and rounding
        assert np.abs(phone_ref.to_bgr(f, fmt).astype(int) - bgr).max() <= 6, fmt
    with pytest.raises(ValueError, match="unknown format"):
        phone_ref.layout("nv16")
    with pytest.raises(ValueError, match="even H and W"):
        phone_ref.planes(np.zeros((4, 5), np.uint8), "nv21")


# ---- the C ABI -----------------------------------------------------------------------------------------------------------
def test_codes_agree_with_the_header():
    with open(os.path.join(ROOT, "include", "centerpose_b200.h")) as fp:
        hdr = fp.read()
    assert _lib.PHONE_FORMATS == PHONE
    codes = [_lib.PIXEL_FORMAT_CODES[f] for f in PHONE]
    assert codes == [10, 11, 12, 14, 13, 15]
    for f in PHONE:
        assert "CP_PIX_%s = %d" % (f.upper(), _lib.PIXEL_FORMAT_CODES[f]) in hdr, f
    # 8 plus the bits 1 (planar), 2 (V first), 4 (full range)
    for f, c in zip(PHONE, codes):
        lay = phone_ref.layout(f)
        assert c == 8 | (lay in ("i420", "yv12")) | 2 * (lay in ("nv21", "yv12")) | 4 * phone_ref.is_full(f), f
    others = [_lib.PIXEL_FORMAT_CODES[f] for f in _lib.PIXEL_FORMATS + _lib.SENSOR_FORMATS]
    assert not set(codes) & set(others + [_lib.CP_PIX_PER_FRAME, _lib.CP_PIX_REMAP])
    assert all(c < 64 and not c & (1 << 6) and not c & _lib.CP_PIX_REMAP for c in codes)
    assert _lib.YUV420_FORMATS == ("nv12", "i420") + PHONE
    assert "CP_PIX_NV21" in hdr and "cp_preprocess_yuv420" in _lib.EXPORTS


def _err(cplib):
    return cplib.cp_last_error()


def _ptrs(hw, fmts, offsets):
    hw = np.ascontiguousarray(hw, np.int32).reshape(-1, 2)
    codes = np.ascontiguousarray(fmts, np.int32)
    offs = np.ascontiguousarray(offsets, np.int64)
    return (offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
            codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), len(offs)), (hw, codes, offs)


def _formats(cplib, hw, fmts, offsets, nbytes):
    (offs, hws, codes, B), keep = _ptrs(hw, fmts, offsets)
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    return cplib.cp_preprocess_formats(ctypes.c_void_p(8), nbytes, offs, hws, codes, ctypes.c_void_p(8), B, 64, 64,
                                       None, m, m, None)


def _table(cplib, hw, fmts, offsets, nbytes):
    (offs, hws, codes, B), keep = _ptrs(hw, fmts, offsets)
    return cplib.cp_preprocess_frame_table_formats(nbytes, offs, hws, codes, B, 64, 64, None, ctypes.c_void_p(8), None)


def _yuv(cplib, hw, fmts, offsets, nbytes):
    (offs, hws, codes, B), keep = _ptrs(hw, fmts, offsets)
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    return cplib.cp_preprocess_yuv420(ctypes.c_void_p(8), nbytes, offs, hws, int(fmts[0]), ctypes.c_void_p(8), B, 64,
                                      64, None, m, m, None)


@pytest.mark.parametrize("who, call", [("cp_preprocess_formats", _formats),
                                       ("cp_preprocess_frame_table_formats", _table),
                                       ("cp_preprocess_yuv420", _yuv)])
def test_entry_points_refuse_bad_phone_frames(who, call, cplib):
    for f in PHONE:
        code = _lib.PIXEL_FORMAT_CODES[f]
        for h, w in ((9, 10), (10, 9), (1, 2), (2, 1)):
            assert call(cplib, [(10, 10), (h, w)], [code, code], [0, 200], 1000) == INVALID
            assert b"frame 1 has size %d x %d (YUV 4:2:0 needs even sizes)" % (h, w) in _err(cplib), f
            assert who.encode() in _err(cplib)
        # a frame overrunning the buffer at 1.5 bytes per pixel: 10 x 10 is 150 bytes, 8 x 12 is 144
        assert call(cplib, [(10, 10), (8, 12)], [code, code], [0, 150], 150 + 144 - 1) == INVALID
        assert b"frame 1 (8 x 12 at byte 150) lies outside the 293-byte buffer" in _err(cplib), f
        assert call(cplib, [(8, 12)], [code], [-1], 1000) == INVALID and b"outside" in _err(cplib)
    # 8 and 9 would be NV12 and I420 again: not formats
    for bad in (8, 9):
        if call is _yuv:
            assert call(cplib, [(10, 10)], [bad], [0], 1000) == INVALID
            assert b"cp_preprocess_yuv420: unknown pixel format %d" % bad in _err(cplib)
        else:
            assert call(cplib, [(10, 10), (10, 10)], [_lib.CP_PIX_NV21, bad], [0, 150], 1000) == INVALID
            assert b"frame 1 has unknown pixel format %d" % bad in _err(cplib)


def test_single_format_launches_take_the_phone_codes(cplib):
    """cp_preprocess_slots_dev / _frame_table / _slots_ragged_dev / _slots_rows_dev / _remap / _frame_table_maps accept
    the six values (their checks pass up to a later one) and check 4:2:0 sizes."""
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    v = ctypes.c_void_p(8)
    hw, offs = np.array([[10, 10]], np.int32), np.zeros(1, np.int64)
    HW, OFFS = hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
    for f in PHONE:
        code = _lib.PIXEL_FORMAT_CODES[f]
        assert cplib.cp_preprocess_slots_dev(v, code, 0, 64, 64, 32, 32, None, m, m, None, v, None, None) == INVALID
        assert b"cp_preprocess_slots_dev: bad shape" in _err(cplib), f
        for h, w in ((63, 64), (64, 9)):
            assert cplib.cp_preprocess_slots_dev(v, code, 2, h, w, 32, 32, None, m, m, None, v, None, None) == INVALID
            assert b"YUV 4:2:0 frames need an even size, got %d x %d" % (h, w) in _err(cplib), f
        assert cplib.cp_preprocess_frame_table(149, OFFS, HW, code, 1, 32, 32, None, v, None) == INVALID
        assert b"frame 0 (10 x 10 at byte 0) lies outside the 149-byte buffer" in _err(cplib), f
        for launch in (code, code | _lib.CP_PIX_REMAP):
            assert cplib.cp_preprocess_slots_ragged_dev(v, v, launch, 0, 32, 32, m, m, None, v, None, None) == INVALID
            assert b"cp_preprocess_slots_ragged_dev: bad shape" in _err(cplib), launch
            assert cplib.cp_preprocess_slots_rows_dev(v, v, launch, v, 0, 32, 32, m, m, None, None, v, None,
                                                      None) == INVALID
            assert b"cp_preprocess_slots_rows_dev: bad shape" in _err(cplib), launch
        codes = np.array([code], np.int32)
        maps = (ctypes.c_void_p * 1)(12)                                          # misaligned: the last check
        rc = cplib.cp_preprocess_remap(v, 150, OFFS, HW, codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), maps, v,
                                       1, 32, 32, None, m, m, None)
        assert rc == INVALID and b"map of frame 0 is not 8-byte aligned" in _err(cplib), f
        rc = cplib.cp_preprocess_frame_table_maps(150, OFFS, HW, code, None, maps, 1, 32, 32, None, v, None)
        assert rc == INVALID and b"map of frame 0 is not 8-byte aligned" in _err(cplib), f
    for bad in (8, 9):
        assert cplib.cp_preprocess_slots_dev(v, bad, 2, 64, 64, 32, 32, None, m, m, None, v, None, None) == INVALID
        assert b"unknown pixel format %d" % bad in _err(cplib)
        assert cplib.cp_preprocess_slots_ragged_dev(v, v, bad, 2, 32, 32, m, m, None, v, None, None) == INVALID
        assert b"unknown pixel format %d" % bad in _err(cplib)


# ---- pixel_format in the Python layer --------------------------------------------------------------------------------
def test_shapes_of_the_phone_formats():
    for f in PHONE:
        assert frame_shape(1440, 1920, f) == (2160, 1920) and frame_layout(f) == "[3H/2,W]"
        assert frame_shape(2, 2, f) == (3, 2)
        assert image_size((2160, 1920), f) == (1440, 1920) and image_size((3, 2), f) == (2, 2)
        with pytest.raises(ValueError, match="%s frames need an even, positive image size; got 1441 x 1920" % f):
            frame_shape(1441, 1920, f)
        with pytest.raises(ValueError, match=r"expected a %s frame \[3H/2,W\] with H and W even" % f):
            image_size((1440, 1920, 3), f)
        with pytest.raises(ValueError, match=r"expected a %s frame \[3H/2,W\]" % f):
            image_size((2160, 1921), f)
    # unknown names: the message lists the colour and sensor formats, then the phone formats
    for bad in ("NV21", "yvu420p", "nv12full", "nv21_limited", "p010"):
        with pytest.raises(ValueError, match="pixel_format must be one of bgr, nv12, i420, .* got %r; phone cameras also "
                                             "give nv21, yv12, nv12_full, nv21_full, i420_full, yv12_full" % bad):
            frame_shape(480, 640, bad)


def test_lists_and_check_frames(cplib):
    from centerpose_b200.engine import preprocess_yuv420
    with pytest.raises(ValueError, match=r"'nv12' or 'i420', or a phone format \(nv21, yv12, nv12_full, .* got 'bgr'"):
        preprocess_yuv420(None, [0], [(10, 10)], "bgr", 64, 64, (0.4,) * 3, (0.3,) * 3)
    mix = ["nv21_full", "nv12", "bayer_rggb8", "yv12"]
    assert slot_formats(mix, 4) == mix
    with pytest.raises(ValueError, match=r"got 'nv61' in \['nv21', 'nv61'\]; phone cameras also give"):
        slot_formats(["nv21", "nv61"], 2)
    check_frames([np.zeros((6, 4), np.uint8), np.zeros((5, 6), np.uint8), None, torch.zeros((3, 2), dtype=torch.uint8)],
                 allow_idle=True, pixel_format=["i420_full", "gray", "nv21", "yv12_full"])
    with pytest.raises(ValueError, match=r"frame 1 has shape \(480, 640, 3\), expected a nv21_full frame \[3H/2,W\]"):
        check_frames([np.zeros((6, 4), np.uint8), np.zeros((480, 640, 3), np.uint8)], allow_idle=False,
                     pixel_format=["nv12", "nv21_full"])
    with pytest.raises(ValueError, match=r"frame 0 has shape \(8, 10\), expected a yv12 frame \[3H/2,W\] with H and W"):
        check_frames([np.zeros((8, 10), np.uint8)], allow_idle=False, pixel_format="yv12")


@pytest.mark.parametrize("fmt", PHONE)
def test_run_batch_refuses_shapes_of_another_format(fmt):
    det, trk, cam = _host_detector(), _host_detector(tracking=True), np.eye(3)
    with pytest.raises(ValueError, match=r"%s frames are uint8 \[B,3H/2,W\], got torch.uint8 \(2, 480, 640, 3\)" % fmt):
        det.run_batch(np.zeros((2, 480, 640, 3), np.uint8), cam, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"each frame has shape \(721, 640\)"):
        det.run_batch(np.zeros((2, 721, 640), np.uint8), cam, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"frame 1 has shape \(480, 640, 1\)"):
        det.run_batch([np.zeros((720, 640), np.uint8), np.zeros((480, 640, 1), np.uint8)], cam, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"frame 0 has shape \(721, 642\)"):
        trk.run_batch([np.zeros((721, 642), np.uint8), None], cam, track=True, pixel_format=fmt)
    with pytest.raises(ValueError, match=r"pixel_format must be one name here, got a list"):
        det.run_batch(np.zeros((2, 720, 640), np.uint8), cam, pixel_format=[fmt, "nv12"])


def test_pipelines_check_phone_sizes():
    det, cam = _host_detector(), np.eye(3)
    with pytest.raises(ValueError, match="nv21_full frames need an even, positive image size; got 1441 x 1920"):
        cpb.BatchPipeline(det, batch=2, height=1441, width=1920, camera_matrix=cam, pixel_format="nv21_full")
    with pytest.raises(ValueError, match=r"pixel_format must be one name here, got a list \['yv12', 'bgr'\]"):
        cpb.TrackPipeline(_host_detector(tracking=True), slots=2, camera_matrix=cam, pixel_format=["yv12", "bgr"])


GRAPHS = [(cpb.TrackGraph, lambda: _det_shell(True)), (cpb.DetectGraph, lambda: _det_shell(False)),
          (cpb.MultiCategoryTrackGraph, lambda: _multi_shell(cpb.MultiCategoryTracker)),
          (cpb.MultiCategoryDetectGraph, lambda: _multi_shell(cpb.MultiCategoryDetector))]


@pytest.mark.parametrize("cls, make", GRAPHS)
def test_graphs_check_phone_formats_before_device_work(cls, make, monkeypatch):
    monkeypatch.setattr(_lib, "load", lambda: (_ for _ in ()).throw(AssertionError("the library was loaded")))
    with pytest.raises(ValueError, match="yv12_full frames need an even, positive image size; got 480 x 641"):
        cls(make(), slots=2, frame_hw=[(480, 640), (480, 641)], camera_matrix=np.eye(3),
            pixel_format=["nv21", "yv12_full"])
    with pytest.raises(ValueError, match="nv12_full frames need an even, positive image size; got 1441 x 1920"):
        cls(make(), slots=2, frame_hw=(1441, 1920), camera_matrix=np.eye(3), pixel_format="nv12_full")
    with pytest.raises(ValueError, match="pixel_format must be one of .* got 'nv21_jfif' in"):
        cls(make(), slots=2, frame_hw=[(480, 640), (720, 1280)], camera_matrix=np.eye(3),
            pixel_format=["nv21", "nv21_jfif"])


# ---- a per-step camera_matrix -----------------------------------------------------------------------------------------
def _graph_shell(S, distorted):
    """The state _SlotGraph._camera_rows reads: S slots of meta rows, and whether the graph undistorts."""
    g = _SlotGraph.__new__(_SlotGraph)
    g.slots, g._distorted = S, distorted
    g._meta_host = np.arange(S * _lib.CP_META_DOUBLES, dtype=np.float64).reshape(S, -1)
    return g


def test_camera_rows_replace_the_camera_fields_only():
    g = _graph_shell(3, False)
    assert g._camera_rows(None) is None
    K = np.array([[1500., 0, 960], [0, 1500, 720], [0, 0, 1]])
    for cam in (K, torch.from_numpy(K), [K.tolist()] * 3, np.stack([K, 2 * K, 3 * K])):
        rows = g._camera_rows(cam)
        want = g._meta_host.copy()
        ks = np.asarray(cam if not torch.is_tensor(cam) else cam.numpy(), np.float64)
        want[:, 5:14] = np.broadcast_to(ks.reshape(-1, 9), (3, 9))
        assert rows.dtype == np.float64 and np.array_equal(rows, want)
    assert np.array_equal(g._meta_host, np.arange(3 * _lib.CP_META_DOUBLES).reshape(3, -1))   # set by the upload only


def test_camera_rows_refusals():
    K = np.eye(3)
    with pytest.raises(ValueError, match="built with distortion=: .* takes no per-step camera_matrix"):
        _graph_shell(2, True)._camera_rows(K)
    g = _graph_shell(2, False)
    for bad in (np.eye(4), np.stack([K] * 3), np.ones(9), [[1, 2], [3]]):
        with pytest.raises(ValueError, match=r"camera_matrix must be \[3,3\] or one \[3,3\] per slot \(\[2,3,3\]\)"):
            g._camera_rows(bad)
    for v in (np.nan, np.inf, -np.inf):
        c = K.copy()
        c[0, 2] = v
        with pytest.raises(ValueError, match="camera_matrix holds a non-finite value"):
            g._camera_rows(c)
    meta = torch.zeros((3, 3), dtype=torch.float64, device="meta")
    with pytest.raises(ValueError, match="camera_matrix is read on the host: pass a numpy array or a CPU tensor"):
        g._camera_rows(meta)
