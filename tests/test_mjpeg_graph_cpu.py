"""MJPEG slots of the live-video graphs without a GPU: the slot capacity of jpeg_core.h (compiled for the host by
tests/host/jpeg_slots_host.cpp) bounds what every supported file of that decoded size needs, cp_jpeg_slots_prepare
fills its block or refuses a slot, the new entry points are exported and bound, and "mjpeg" is refused with a message
that names where it runs, before any device work: outside the graphs, with max_frame_bytes but no "mjpeg" slot, and
on a call whose frame is refused."""
import ctypes
import itertools
import os
import subprocess

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.engine import jpeg_parse
from tests import jpeg_craft as jc
from tests.test_detect_graph_cpu import _built, no_device  # noqa: F401  (a fixture)
from tests.test_jpeg_cpu import _frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("cp_jpeg_slots_workspace_bytes", "cp_jpeg_slots_block_bytes", "cp_jpeg_slots_prepare",
       "cp_jpeg_decode_slots_dev", "cp_jpeg_mask_counts_dev")
FIELDS = ("comp", "nseg", "nsub", "nblocks", "nplane")


@pytest.fixture(scope="module")
def js():
    src = os.path.join(ROOT, "tests", "host", "jpeg_slots_host.cpp")
    hdr = os.path.join(ROOT, "centerpose_b200", "csrc", "jpeg_core.h")
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    so = os.path.join(out_dir, "libjpeg_slots_host.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, src])
    return ctypes.CDLL(so)


def _capacity(js, h, w, max_bytes, words):
    out = np.zeros(5, np.int64)
    js.js_capacity(int(h), int(w), ctypes.c_int64(max_bytes), words, out.ctypes.data_as(ctypes.c_void_p))
    return out


def _need(js, data, words):
    a = np.frombuffer(data, np.uint8)
    out, hw = np.zeros(5, np.int64), np.zeros(2, np.int32)
    assert js.js_need(a.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(len(a)), words,
                      hw.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p)) == 0
    return tuple(hw), out


def test_new_symbols_are_exported_and_bound(cplib):
    for name in NEW:
        assert name in _lib.EXPORTS and hasattr(cplib, name) and getattr(cplib, name).argtypes
    assert _lib.JPEG_ERR_SYNC == 16 and _lib.JPEG_ERR_SYNC in _lib.JPEG_ERRORS
    hdr = open(os.path.join(ROOT, "include", "centerpose_b200.h")).read()
    assert "CP_JPEG_ERR_SYNC = 16" in hdr and all(name + "(" in hdr for name in NEW)


SIZES = [(1, 1), (1, 17), (5, 3), (9, 7), (17, 33), (37, 53), (121, 97), (480, 640), (1080, 1920)]


@pytest.mark.parametrize("sampling", jc.SAMPLINGS)
def test_capacity_bounds_every_layout(js, sampling):
    """For every sampling, orientation 1..8 and restart interval 0 / 1 / 4, what a file needs fits the capacity of its
    decoded size at its own length, at several subsequence lengths."""
    exact = np.zeros(5, bool)
    for (h, w), ri in itertools.product(SIZES, (0, 1, 4)):
        base = jc.encode(_frame(h, w, h * 7 + w), sampling, 75, restart=ri)
        for o in range(1, 9):
            data = jc.with_orientation(base, o, big_endian=o % 2 == 0) if o > 1 else base
            hw, need = _need(js, data, 1)
            assert hw == ((w, h) if o >= 5 else (h, w))
            for words in (1, 2, 8):
                _, need = _need(js, data, words)
                cap = _capacity(js, hw[0], hw[1], len(data), words)
                assert (need <= cap).all(), (sampling, h, w, ri, o, words, dict(zip(FIELDS, need)),
                                             dict(zip(FIELDS, cap)))
                exact |= need == cap
    if sampling in ("444", "411"):           # the block bound is 4:4:4's for most sizes, 4:1:1's for the narrowest
        assert exact[3] and exact[4]


def _prepare(cplib, S, hw, max_bytes, headers, nbytes, out_offsets, words=0):
    hw = np.ascontiguousarray(hw, np.int32)
    mb = np.ascontiguousarray(max_bytes, np.int64)
    hs = (_lib.CpJpegHeader * S)(*headers)
    nb = np.ascontiguousarray(nbytes, np.int64)
    oo = np.ascontiguousarray(out_offsets, np.int64)
    block = np.full(cplib.cp_jpeg_slots_block_bytes(S), 0xAB, np.uint8)
    p32, p64 = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
    rc = cplib.cp_jpeg_slots_prepare(S, hw.ctypes.data_as(p32), mb.ctypes.data_as(p64), words, hs,
                                     nb.ctypes.data_as(p64), oo.ctypes.data_as(p64), block.ctypes.data_as(ctypes.c_void_p))
    return rc, block


def test_slots_prepare(cplib):
    hsz = ctypes.sizeof(_lib.CpJpegHeader)
    a, b = jc.encode(_frame(48, 64, 1), "420", 90), jc.encode(_frame(64, 48, 2), "gray", 80, restart=2)
    ha, hb = (jpeg_parse(np.frombuffer(d, np.uint8)) for d in (a, b))
    hw, mb = [(48, 64), (64, 48), (48, 64)], [len(a), 4096, 9216]
    assert cplib.cp_jpeg_slots_block_bytes(0) == 0
    assert cplib.cp_jpeg_slots_block_bytes(3) >= 3 * hsz
    rc, block = _prepare(cplib, 3, hw, mb, [ha, hb, _lib.CpJpegHeader()], [len(a), len(b), 0], [0, 9216, 18432])
    assert rc == 0
    assert block[:hsz].tobytes() == bytes(ha) and block[hsz:2 * hsz].tobytes() == bytes(hb)
    assert not block[2 * hsz:3 * hsz].any()                      # slot 2 skipped: a zero header
    p32, p64 = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
    hwa, mba = np.array(hw, np.int32), np.array(mb, np.int64)
    ws = [cplib.cp_jpeg_slots_workspace_bytes(3, hwa.ctypes.data_as(p32), mba.ctypes.data_as(p64), w) for w in (0, 1, 8)]
    assert ws[0] == ws[2] and ws[1] > ws[2] > 0
    # refusals name the slot and leave the block as it was
    prog = jpeg_parse(np.frombuffer(jc.encode(_frame(48, 64, 1), "420", 90, progressive=True), np.uint8))
    cases = [([prog, hb, ha], [len(a), len(b), len(a)], "slot 0"),                   # a refused header
             ([ha, ha, ha], [len(a), len(a), len(a)], "slot 1 decodes to 48 x 64"),   # the wrong decoded size
             ([ha, hb, ha], [len(a), 4097, len(a)], "slot 1: 4097 bytes"),            # more than max_bytes
             ([ha, hb, ha], [len(a), 10, len(a)], "slot 1: 10 bytes")]                 # a scan past the bytes
    for headers, nbytes, msg in cases:
        rc, block = _prepare(cplib, 3, hw, mb, headers, nbytes, [0, 9216, 18432])
        assert rc == -1 and msg in cplib.cp_last_error().decode() and (block == 0xAB).all(), msg
    assert cplib.cp_jpeg_slots_workspace_bytes(1, np.array([0, 5], np.int32).ctypes.data_as(p32),
                                               np.array([9], np.int64).ctypes.data_as(p64), 0) == 0
    assert _prepare(cplib, 1, [(48, 64)], [0], [ha], [0], [0])[0] == -1


# ---------------------------------------------------------------- Python refusals
def test_mjpeg_is_not_a_pixel_format():
    from centerpose_b200.engine import _ALL_FORMATS, check_pixel_format, slot_formats
    assert "mjpeg" not in _lib.PIXEL_FORMATS + _lib.SENSOR_FORMATS and "mjpeg" not in _lib.PIXEL_FORMAT_CODES
    assert "mjpeg" not in _ALL_FORMATS
    for call in (lambda: check_pixel_format("mjpeg"), lambda: slot_formats(["bgr", "mjpeg"], 2)):
        with pytest.raises(ValueError, match=r"live-video graphs .*run_batch\(list, pixel_format=\"jpeg\"\)"):
            call()


def test_pipelines_array_forms_and_run_batch_refuse_mjpeg():
    from centerpose_b200.pipeline import BatchPipeline, TrackPipeline
    from tests.test_meta_geometry import _detector
    det = _detector("fix_res")
    det.opt.device = "cpu"
    makes = [lambda: BatchPipeline(det, 2, 480, 640, np.eye(3), pixel_format="mjpeg"),
             lambda: TrackPipeline(det, 2, np.eye(3), pixel_format="mjpeg"),
             lambda: det._array_input(np.zeros((1, 8, 8, 3), np.uint8), np.eye(3), pixel_format="mjpeg"),
             lambda: det.run_batch([b"\xff\xd8\xff", b"\xff\xd8\xff"], np.eye(3), pixel_format="mjpeg"),
             lambda: det.run_batch([b"\xff\xd8\xff", np.zeros((8, 8, 3), np.uint8)], np.eye(3),
                                   pixel_format=["mjpeg", "bgr"])]
    for make in makes:
        with pytest.raises(ValueError, match=r"\"mjpeg\" is an MJPEG camera .*DetectGraph, TrackGraph"):
            make()


def test_max_frame_bytes_needs_an_mjpeg_slot(no_device):
    from tests.test_yuv_input_cpu import _host_detector
    for fmt, hw in (("bgr", (480, 640)), (["nv12", "bgr"], [(480, 640), (480, 640)])):
        with pytest.raises(ValueError, match="max_frame_bytes caps the encoded frames of \"mjpeg\" slots, and no slot"):
            cpb.DetectGraph(_host_detector(), 2, hw, np.eye(3), pixel_format=fmt, max_frame_bytes=1 << 20)
    for bad in (0, [1 << 20], 1 << 28, 1.5):
        with pytest.raises(ValueError, match="max_frame_bytes is one int or one per slot"):
            cpb.DetectGraph(_host_detector(), 2, (480, 640), np.eye(3), pixel_format="mjpeg", max_frame_bytes=bad)


def _mjpeg_shell(cls=cpb.DetectGraph, S=3, idle=False, mjpeg=(0, 1, 2), max_bytes=1 << 20):
    g = _built(cls, S=S, idle=idle, per_slot=True)
    g._mjpeg = list(mjpeg)
    g._jmax = np.full(S, max_bytes, np.int64)
    g.pixel_format = ["mjpeg" if b in mjpeg else "bgr" for b in range(S)]

    def device_work(*a, **k):
        raise AssertionError("device work before the refusal")
    g._replay = g._upload_encoded = device_work
    return g


@pytest.mark.parametrize("cls", [cpb.DetectGraph, cpb.TrackGraph])
def test_call_refusals_come_before_device_work(cls):
    ok = jc.encode(_frame(480, 640, 3), "422", 85)
    g = _mjpeg_shell(cls)
    name = cls.__name__
    with pytest.raises(ValueError, match=name + r" has \"mjpeg\" slots: frames is a list of 3 entries.*got ndarray"):
        g(np.zeros((3, 480, 640, 3), np.uint8))
    with pytest.raises(ValueError, match="frames is a list of 3 entries.*got 2 entries"):
        g([ok, ok])
    with pytest.raises(ValueError, match="slot 1 decodes to 640 x 480, its frame_hw is \\(480, 640\\)"):
        g([ok, jc.encode(_frame(640, 480, 3), "422", 85), ok])
    with pytest.raises(ValueError, match="slot 2 is a JPEG the device decoder does not take: progressive JPEG"):
        g([ok, ok, jc.encode(_frame(480, 640, 3), "420", 85, progressive=True)])
    with pytest.raises(ValueError, match="slot 0 is an \"mjpeg\" slot: its frame is the encoded bytes.*got str"):
        g(["frame.jpg", ok, ok])
    with pytest.raises(ValueError, match="slot 1 is an \"mjpeg\" slot: its frame is the encoded bytes.*got ndarray"):
        g([ok, np.zeros((480, 640, 3), np.uint8), ok])
    with pytest.raises(ValueError, match="slot 2 is idle"):
        g([ok, ok, None])
    small = _mjpeg_shell(cls, max_bytes=len(ok) - 1)
    with pytest.raises(ValueError, match="slot 0 takes encoded frames of at most max_frame_bytes = %d bytes, got %d"
                                         % (len(ok) - 1, len(ok))):
        small([ok, ok, ok])
    # an idle-capable graph takes None; the bytes of a good frame in any form pass the checks
    idle = _mjpeg_shell(cls, idle=True)
    idle._replay = lambda frames, *a: frames
    got = idle._frames([ok, None, torch.from_numpy(np.frombuffer(ok, np.uint8).copy())])
    assert got[1] is None and all(e[1].out_h == 480 and e[0].numel() == len(ok) for e in (got[0], got[2]))
