"""CPU tests of the JPEG decoder: centerpose_b200/csrc/jpeg_core.h compiled for the host (tests/host/jpeg_core_host.cpp)
restates the whole baseline decoder sequentially, and equals cv2.imdecode (libjpeg-turbo) bit for bit on cv2.imencode
frames of every sampling, quality, size and restart interval, with optimised and with absent Huffman tables, under
every EXIF orientation, and on crafted files cv2's encoder cannot write.  The host simulation of the subsequence decode
gives the sequential decoder's coefficients.  Every refusal reason comes from a crafted header, and the Python API
refuses pixel_format "jpeg" outside run_batch(list)."""
import ctypes
import itertools
import os
import struct
import subprocess

import numpy as np
import pytest

from tests import jpeg_craft as jc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(1, 1), (1, 17), (5, 3), (8, 8), (16, 16), (17, 33), (37, 53), (480, 640), (640, 480)]
QUALITIES = (10, 50, 75, 95, 100)


@pytest.fixture(scope="module")
def jh():
    src = os.path.join(ROOT, "tests", "host", "jpeg_core_host.cpp")
    hdr = os.path.join(ROOT, "centerpose_b200", "csrc", "jpeg_core.h")
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    so = os.path.join(out_dir, "libjpeg_core_host.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.jh_blocks.restype = ctypes.c_int64
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def host_decode(jh, data):
    a = np.frombuffer(data, np.uint8)
    h = parse(jh, data)
    out = np.zeros((h.out_h, h.out_w, 3), np.uint8)
    err = jh.jh_decode(_p(a), ctypes.c_int64(len(a)), _p(out))
    return err, out


def parse(jh, data):
    from centerpose_b200 import _lib
    a = np.frombuffer(data, np.uint8)
    h = _lib.CpJpegHeader()
    jh.jh_parse(_p(a), ctypes.c_int64(len(a)), ctypes.byref(h))
    return h


def coefficients(jh, data, words):
    a = np.frombuffer(data, np.uint8)
    c = np.zeros(jh.jh_blocks(_p(a), ctypes.c_int64(len(a))) * 64, np.int16)
    rounds = ctypes.c_int(0)
    err = jh.jh_coefficients(_p(a), ctypes.c_int64(len(a)), int(words), _p(c), ctypes.byref(rounds))
    return err, c, rounds.value


def _frame(h, w, seed):
    """A test frame resized to h x w with seeded noise, or pure noise for tiny sizes."""
    import cv2
    rng = np.random.default_rng(seed)
    if h * w < 64:
        return rng.integers(0, 256, (h, w, 3), np.uint8)
    base = cv2.imread(os.path.join(ROOT, "tests", "data", "frame_%d.png" % (seed % 2)))
    img = cv2.resize(base, (w, h)).astype(np.int16) + rng.integers(-8, 9, (h, w, 3)).astype(np.int16)
    return np.clip(img, 0, 255).astype(np.uint8)


def _assert_cv2(jh, data, what):
    err, got = host_decode(jh, data)
    want = jc.decode(data)
    assert err == 0 and got.shape == want.shape and np.array_equal(got, want), what


def test_header_struct_matches_the_c_abi(jh, cplib):
    from centerpose_b200 import _lib
    assert ctypes.sizeof(_lib.CpJpegHeader) == jh.jh_header_size()
    assert ctypes.sizeof(_lib.CpJpegHuff) == 512 * 2 + 18 * 4 * 2 + 256
    for name in ("cp_jpeg_parse", "cp_jpeg_workspace_bytes", "cp_jpeg_decode", "cp_jpeg_last_rounds"):
        assert name in _lib.EXPORTS and hasattr(cplib, name)


def test_standard_tables_are_cv2s(jh):
    """The K.3 tables of the writer (and, through the DHT-free decodes below, of jpeg_core.h) are those cv2 writes."""
    t = jc.dht_tables(jc.encode(_frame(16, 16, 0), "420", 75))
    for k in range(2):
        assert t[(0, k)] == (jc.STD_DC_BITS[k], bytes(range(12)))
        assert t[(1, k)][0] == jc.STD_AC_BITS[k] and len(t[(1, k)][1]) == 162


@pytest.mark.parametrize("sampling", jc.SAMPLINGS)
def test_host_decoder_is_cv2(jh, sampling):
    for (h, w), q, ri in itertools.product(SIZES, QUALITIES, (0, 1, 4)):
        _assert_cv2(jh, jc.encode(_frame(h, w, h * 31 + w), sampling, q, restart=ri), (h, w, q, ri))


@pytest.mark.parametrize("sampling", jc.SAMPLINGS)
def test_optimised_and_absent_tables(jh, sampling):
    for h, w in SIZES:
        img = _frame(h, w, h + 7 * w)
        _assert_cv2(jh, jc.encode(img, sampling, 85, optimize=True), (h, w, "optimised"))
        _assert_cv2(jh, jc.strip(jc.encode(img, sampling, 85, restart=2), 0xC4), (h, w, "no DHT"))


@pytest.mark.parametrize("width", [1, 2, 3, 4, 5])
def test_narrow_images_upsample_as_cv2(jh, width):
    """Where libjpeg-turbo drops fancy up-sampling to replication (a downsampled width of 2 or less)."""
    for s in ("422", "420", "440", "411"):
        for h in (1, 2, 3, 9):
            _assert_cv2(jh, jc.encode(_frame(h, width, width * 13 + h), s, 95), (s, h, width))


@pytest.mark.parametrize("big_endian", [False, True])
def test_exif_orientation(jh, big_endian):
    base = jc.encode(_frame(37, 53, 5), "420", 90)
    for o in range(1, 9):
        data = jc.with_orientation(base, o, big_endian)
        h = parse(jh, data)
        assert h.status == 0 and h.orientation == o
        assert (h.out_h, h.out_w) == ((53, 37) if o >= 5 else (37, 53))
        _assert_cv2(jh, data, o)


def _exif_without_orientation():
    tiff = b"II" + struct.pack("<HI", 42, 8)
    ifd = struct.pack("<H", 1) + struct.pack("<HHI", 0x010F, 2, 4) + b"cam\0" + struct.pack("<I", 0)
    return jc.app_segment(0xE1, b"Exif\0\0" + tiff + ifd)


def test_exif_orientation_across_app1_segments(jh):
    """cv2 takes the first Orientation tag of any Exif APP1: an XMP APP1 or an Exif APP1 without the tag before it does
    not hide it, and a later Exif APP1 does not override it; values outside 1..8 leave the image as it is."""
    base = jc.encode(_frame(37, 53, 6), "422", 90)
    xmp = jc.app_segment(0xE1, b"http://ns.adobe.com/xap/1.0/\0<x:xmpmeta/>")
    cases = [([xmp, jc.exif(6)], 6), ([_exif_without_orientation(), jc.exif(8, True)], 8),
             ([jc.exif(5), jc.exif(3)], 5), ([jc.exif(9)], 1), ([jc.exif(0)], 1), ([jc.exif(9), jc.exif(6)], 1)]
    for segs, o in cases:
        data = base
        for seg in reversed(segs):                       # each insert lands right after APP0: the list's order
            data = jc.insert(data, seg)
        assert parse(jh, data).orientation == o, o
        _assert_cv2(jh, data, o)


def test_subsequence_decode_equals_sequential(jh):
    rng = np.random.default_rng(7)
    files = [jc.encode(_frame(h, w, i), s, q, restart=ri) for i, ((h, w), s, q, ri) in
             enumerate([((480, 640), "420", 90, 0), ((37, 53), "444", 100, 1), ((17, 33), "gray", 50, 4),
                        ((640, 480), "411", 75, 0), ((16, 16), "440", 10, 0)])]
    files.append(jc.encode(np.full((256, 256), 128, np.uint8), "gray", 75))      # periodic: 6-bit symbol pairs
    for data in files:
        err, ref, _ = coefficients(jh, data, 0)
        assert err == 0
        for words in [1, 2, 32] + list(rng.integers(3, 64, 3)):
            e, c, _ = coefficients(jh, data, words)
            assert e == 0 and np.array_equal(c, ref), words


# ---------------------------------------------------------------- crafted files
def _blocks(nblocks, rng, lo, hi, density):
    b = np.zeros((nblocks, 64), np.int32)
    mask = rng.random((nblocks, 64)) < density
    b[mask] = rng.integers(lo, hi + 1, mask.sum())
    return b


def test_crafted_extreme_coefficients(jh):
    """IDCT outputs far outside 0..255: DC-only blocks of every DC value up to |x| = 1023 after the IDCT, and random
    blocks of large coefficients, in 8- and 16-bit tables, where the range limit saturates."""
    dcs = np.arange(-1023, 1024)
    b = np.zeros((len(dcs), 64), np.int32)
    b[:, 0] = dcs
    _assert_cv2(jh, jc.write(8 * len(dcs), 8, b, [np.full(64, 8)], gray=True), "DC levels")
    rng = np.random.default_rng(3)
    for (luma, gray), (amp, q) in itertools.product((((1, 1), True), ((2, 2), False), ((2, 1), False)),
                                                    ((60, 4), (120, 2))):
        w, h = 40, 24
        bpm = 1 if gray else luma[0] * luma[1] + 2
        n = -(-w // (8 * luma[0])) * -(-h // (8 * luma[1])) * bpm
        blk = _blocks(n, rng, -amp, amp, 0.3)
        blk[:, 0] = rng.integers(-1023, 1024, n)
        for qbits in (8, 16):
            _assert_cv2(jh, jc.write(w, h, blk, [np.full(64, q)] * 2, luma=luma, gray=gray, qbits=qbits),
                        (luma, gray, amp, qbits))


def test_crafted_dc_levels_and_colour_tables(jh):
    """Quantisation tables of 1 and DC-only 4:4:4 blocks reach every Y, Cb and Cr level; plus seeded triples."""
    levels = np.arange(256)
    rng = np.random.default_rng(11)
    trip = [(y, y, y) for y in levels] + [(128, c, 255 - c) for c in levels] + \
           [tuple(t) for t in rng.integers(0, 256, (512, 3))]
    n = len(trip)
    b = np.zeros((n * 3, 64), np.int32)
    for i, (y, cb, cr) in enumerate(trip):
        b[3 * i:3 * i + 3, 0] = [8 * (y - 128), 8 * (cb - 128), 8 * (cr - 128)]
    data = jc.write(8 * n, 8, b, [np.ones(64), np.ones(64)], luma=(1, 1))
    _assert_cv2(jh, data, "levels")
    _assert_cv2(jh, jc.write(8 * n, 8, b, [np.ones(64), np.ones(64)], luma=(1, 1), dht=False, restart=7), "no DHT")


def test_crafted_periodic_streams_need_many_rounds(jh):
    """All-zero blocks repeat one short symbol pair, so a guessed start rarely synchronises: the rounds grow with the
    subsequences and the result is still the sequential decoder's."""
    b = np.zeros((64 * 32, 64), np.int32)
    data = jc.write(64 * 8, 32 * 8, b, [np.full(64, 4)], gray=True)
    _assert_cv2(jh, data, "zeros")
    err, ref, _ = coefficients(jh, data, 0)
    e, c, rounds = coefficients(jh, data, 1)
    assert e == 0 and np.array_equal(c, ref) and rounds > 10


# ---------------------------------------------------------------- refusals
def _reason(jh, data):
    return parse(jh, data).status


def test_every_refusal_reason(jh):
    from centerpose_b200 import _lib
    base = jc.encode(_frame(32, 48, 1), "420", 90)
    R = {v: k for k, v in _lib.JPEG_REFUSALS.items()}
    assert _reason(jh, base) == 0
    assert _reason(jh, b"\x89PNG\r\n\x1a\n" + base) == R["not a JPEG file"]
    assert _reason(jh, jc.encode(_frame(32, 48, 1), "420", 90, progressive=True)) == R["progressive JPEG"]
    assert _reason(jh, jc.patch_marker(base, 0xC0, 0xC9)) == R["arithmetic coding"]
    assert _reason(jh, jc.patch_marker(base, 0xC0, 0xC3)) == R["lossless JPEG"]
    sof = [s for s in jc.markers(base) if s[0] == 0xC0][0]
    p12 = base[:sof[1] + 4] + b"\x0c" + base[sof[1] + 5:]
    assert _reason(jh, p12) == R["samples other than 8 bits"]
    dnl = base[:sof[1] + 5] + b"\x00\x00" + base[sof[1] + 7:]
    assert _reason(jh, dnl) == R["height set by a DNL marker"]
    # 4 components (CMYK), 2 components
    c4 = base[:sof[1] + 9] + b"\x04" + base[sof[1] + 10:]
    assert _reason(jh, c4) == R["not 1 or 3 components"]
    # a non-interleaved scan: the SOS of one component
    sos = jc.markers(base)[-1]
    one = base[:sos[1]] + jc.app_segment(0xDA, b"\x01\x01\x00\x00\x3f\x00") + base[sos[2]:]
    assert _reason(jh, one) == R["more than one scan"]
    # RGB: Adobe transform 0 without JFIF, or component ids R G B
    nojfif = jc.strip(base, 0xE0)
    adobe0 = jc.insert(nojfif, jc.app_segment(0xEE, b"Adobe\x00\x64\x00\x00\x00\x00\x00"))
    assert _reason(jh, adobe0) == R["RGB-coded JPEG"]
    adobe1 = jc.insert(nojfif, jc.app_segment(0xEE, b"Adobe\x00\x64\x00\x00\x00\x00\x01"))
    assert _reason(jh, adobe1) == 0
    rgb = bytearray(nojfif)
    sof2 = [s for s in jc.markers(nojfif) if s[0] == 0xC0][0]
    sos2 = jc.markers(nojfif)[-1]
    for k, c in enumerate(b"RGB"):
        rgb[sof2[1] + 10 + 3 * k] = c
        rgb[sos2[1] + 5 + 2 * k] = c
    assert _reason(jh, bytes(rgb)) == R["RGB-coded JPEG"]
    # other sampling: chroma 2x1
    samp = bytearray(base)
    samp[sof[1] + 14] = 0x21
    assert _reason(jh, bytes(samp)) == R["unsupported chroma sampling"]
    # more pixels than cv2.imread takes (CV_IO_MAX_IMAGE_PIXELS, 2^30); exactly 2^30 is taken
    for (hh, ww), want in (((65535, 65535), R["more than 2^30 pixels"]), ((16385, 65535), R["more than 2^30 pixels"]),
                           ((16384, 65536 - 1), 0)):
        big = base[:sof[1] + 5] + struct.pack(">HH", hh, ww) + base[sof[1] + 9:]
        assert _reason(jh, big) == want, (hh, ww)
    # truncation inside every header segment
    for m, a, b in jc.markers(base):
        for cut in (a + 1, a + 3, b - 1):
            assert _reason(jh, base[:cut]) == R["truncated header"], (hex(m), cut)


def test_cp_jpeg_parse_is_the_host_parser(jh, cplib):
    from centerpose_b200.engine import jpeg_parse
    for data in (jc.encode(_frame(37, 53, 2), "411", 60, restart=3), jc.encode(_frame(8, 8, 2), "420", 90,
                                                                              progressive=True)):
        a, b = jpeg_parse(np.frombuffer(data, np.uint8)), parse(jh, data)
        assert bytes(a) == bytes(b)


# ---------------------------------------------------------------- Python refusals of "jpeg"
def test_jpeg_is_not_a_pixel_format():
    from centerpose_b200 import _lib
    from centerpose_b200.engine import _ALL_FORMATS, check_pixel_format, slot_formats
    assert "jpeg" not in _lib.PIXEL_FORMATS + _lib.SENSOR_FORMATS and "jpeg" not in _lib.PIXEL_FORMAT_CODES
    assert "jpeg" not in _ALL_FORMATS
    for call in (lambda: check_pixel_format("jpeg"), lambda: slot_formats(["bgr", "jpeg"], 2)):
        with pytest.raises(ValueError, match=r"run_batch\(list, pixel_format=\"jpeg\"\)"):
            call()


def test_pipelines_graphs_and_array_forms_refuse_jpeg():
    """The pipelines, the four live-video graphs and the array forms take frames of a fixed shape: each refuses "jpeg"
    (one name, or in a per-slot list) before any device work."""
    import centerpose_b200 as cpb
    from centerpose_b200.detector import MultiCategoryDetector, MultiCategoryTracker, ObjectPoseDetector
    from centerpose_b200.graph import DetectGraph, MultiCategoryDetectGraph
    from centerpose_b200.pipeline import BatchPipeline, TrackPipeline
    from centerpose_b200.tracker import MultiCategoryTrackGraph, TrackGraph
    from tests.test_meta_geometry import _detector

    def shell(cls, tracking):
        d = cls.__new__(cls)
        d.opt = cpb.default_opt("dla_34", tracking_task=tracking)
        return d

    det = _detector("fix_res")
    det.opt.device = "cpu"
    makes = [lambda: BatchPipeline(det, 2, 480, 640, np.eye(3), pixel_format="jpeg"),
             lambda: TrackPipeline(det, 2, np.eye(3), pixel_format="jpeg"),
             lambda: det._array_input(np.zeros((1, 8, 8, 3), np.uint8), np.eye(3), pixel_format="jpeg")]
    for G, cls, tracking in ((DetectGraph, ObjectPoseDetector, False), (TrackGraph, ObjectPoseDetector, True),
                             (MultiCategoryDetectGraph, MultiCategoryDetector, False),
                             (MultiCategoryTrackGraph, MultiCategoryTracker, True)):
        makes.append(lambda G=G, cls=cls, t=tracking: G(shell(cls, t), 2, (480, 640), np.eye(3), pixel_format="jpeg"))
        makes.append(lambda G=G, cls=cls, t=tracking: G(shell(cls, t), 2, [(480, 640)] * 2, np.eye(3),
                                                        pixel_format=["bgr", "jpeg"]))
    for make in makes:
        with pytest.raises(ValueError, match=r"run_batch\(list"):
            make()
