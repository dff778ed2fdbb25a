"""MJPEG cameras on the device: the graph-safe slot decode (cp_jpeg_decode_slots_dev) equals cv2.imdecode and
cp_jpeg_decode bit for bit at every subsequence length, also captured once in a CUDA graph and replayed over frames
whose sampling, quality, restart interval and length change; a corrupt frame sets only its slot's error word; and the
four live-video graphs with "mjpeg" slots give, step for step, bit for bit what run_batch(list, pixel_format="jpeg")
gives on the same encoded frames, with a corrupt frame detecting nothing in its own slot only."""
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.engine import jpeg_parse
from tests import jpeg_craft as jc
from tests.test_gpu_detect_graph import _capacity, _check, _scattered
from tests.test_gpu_detect_graph import _detector as _det_detector
from tests.test_gpu_jpeg import _decode, _frame, _invalid_code, _truncated, _variants, _wrong_rst
from tests.test_gpu_track_graph import _detector as _trk_detector
from tests.test_gpu_track_graph_multi import _check_step, _slot_cameras, _tracker
from tests.test_gpu_undistort import PLUMB

pytestmark = pytest.mark.gpu
P32, P64 = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
STEPS = 5
CATS = ("chair", "cup")


@pytest.fixture(scope="module")
def det_checkpoints(tmp_path_factory):
    d = tmp_path_factory.mktemp("mjpeg_det")
    paths = {c: str(d / (c + ".pth")) for c in CATS}
    for c, seed in zip(CATS, (51, 52)):
        cpb.save_model(paths[c], 1, _det_detector(seed=seed).model)
    return paths


@pytest.fixture(scope="module")
def trk_checkpoints(tmp_path_factory):
    d = tmp_path_factory.mktemp("mjpeg_trk")
    paths = {c: str(d / (c + ".pth")) for c in CATS}
    m = _trk_detector().model
    for c in CATS:
        cpb.save_model(paths[c], 1, m)
    return paths


class _Slots:
    """The slot decode driven by hand: fixed sizes and capacities, one device block, bytes buffer and workspace."""

    def __init__(self, L, hw, max_bytes, words=0):
        self.L, self.S, self.words = L, len(hw), words
        self.hw, self.mb = np.ascontiguousarray(hw, np.int32), np.ascontiguousarray(max_bytes, np.int64)
        self.boffs = np.concatenate([[0], np.cumsum(self.mb)[:-1]]).astype(np.int64)
        sizes = [h * w * 3 for h, w in hw]
        self.oo = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        self.sizes = sizes
        ws = L.cp_jpeg_slots_workspace_bytes(self.S, self.hw.ctypes.data_as(P32), self.mb.ctypes.data_as(P64), words)
        assert ws > 0
        self.ws = torch.empty((ws,), dtype=torch.uint8, device="cuda")
        self.host = np.zeros(L.cp_jpeg_slots_block_bytes(self.S), np.uint8)
        self.block = torch.zeros((self.host.size,), dtype=torch.uint8, device="cuda")
        self.bytes = torch.zeros((int(self.mb.sum()),), dtype=torch.uint8, device="cuda")
        self.out = torch.zeros((sum(sizes),), dtype=torch.uint8, device="cuda")
        self.err = torch.zeros((self.S,), dtype=torch.int32, device="cuda")

    def load(self, files):
        """The block and bytes of one call; files[s] None skips slot s."""
        hs = (_lib.CpJpegHeader * self.S)()
        nb = np.zeros(self.S, np.int64)
        for s, f in enumerate(files):
            if f is not None:
                hs[s], nb[s] = jpeg_parse(np.frombuffer(f, np.uint8)), len(f)
        assert self.L.cp_jpeg_slots_prepare(self.S, self.hw.ctypes.data_as(P32), self.mb.ctypes.data_as(P64),
                                            self.words, hs, nb.ctypes.data_as(P64), self.oo.ctypes.data_as(P64),
                                            self.host.ctypes.data_as(ctypes.c_void_p)) == 0
        self.block.copy_(torch.from_numpy(self.host))
        for s, f in enumerate(files):
            if f is not None:
                o = int(self.boffs[s])
                self.bytes[o:o + len(f)].copy_(torch.from_numpy(np.frombuffer(f, np.uint8).copy()))

    def decode(self):
        assert self.L.cp_jpeg_decode_slots_dev(
            ctypes.c_void_p(self.block.data_ptr()), self.S, self.hw.ctypes.data_as(P32), self.mb.ctypes.data_as(P64),
            self.words, ctypes.c_void_p(self.bytes.data_ptr()), ctypes.c_void_p(self.out.data_ptr()),
            ctypes.c_void_p(self.ws.data_ptr()), ctypes.c_size_t(self.ws.numel()), ctypes.c_void_p(self.err.data_ptr()),
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0

    def images(self):
        host = self.out.cpu().numpy()
        return [host[o:o + n].reshape(h, w, 3) for o, n, (h, w) in zip(self.oo, self.sizes, self.hw)]


def _hw(f):
    h = jpeg_parse(np.frombuffer(f, np.uint8))
    return (h.out_h, h.out_w)


@pytest.mark.parametrize("words", [0, 1, 2, 5])
def test_slot_decode_is_cv2_and_cp_jpeg_decode(words, cplib):
    files = _variants()
    # one frame exactly at its max_bytes, the others in larger slots
    slots = _Slots(cplib, [_hw(f) for f in files], [len(f) if k == 3 else 2 * len(f) + 100 for k, f in enumerate(files)],
                   words)
    slots.load(files)
    slots.decode()
    ref, ref_err = _decode(files, words)
    assert not slots.err.cpu().numpy().any() and not ref_err.any()
    for k, (f, g, r) in enumerate(zip(files, slots.images(), ref)):
        assert np.array_equal(g, jc.decode(f)) and np.array_equal(g, r), k


def _changing(k, hw, seed):
    """Frame k of a camera of decoded size hw: the sampling, quality, restart interval and orientation change every
    frame (a 90-degree EXIF orientation codes the transposed frame)."""
    s = jc.SAMPLINGS[k % len(jc.SAMPLINGS)]
    q, ri, o = (25, 85, 100, 60, 95)[k % 5], (0, 1, 4, 2)[k % 4], (1, 6, 3, 8)[k % 4]
    h, w = (hw[1], hw[0]) if o >= 5 else hw
    data = jc.encode(_frame(h, w, seed + k), s, q, restart=ri, optimize=k % 3 == 2)
    data = jc.with_orientation(data, o, big_endian=k % 2 == 0) if o > 1 else data
    return jc.strip(data, 0xC4) if k % 5 == 4 else data                    # MJPEG: no DHT


def test_captured_slot_decode_replays_changing_frames(cplib):
    hw = [(120, 160), (37, 53), (240, 320), (9, 7)]
    for words in (0, 1):
        slots = _Slots(cplib, hw, [h * w * 3 + 4096 for h, w in hw], words)
        slots.load([None] * len(hw))
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            slots.decode()                      # warm-up, then the capture: a host synchronise would fail it
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            slots.decode()
        for k in range(6):
            files = [_changing(k + s, hw[s], 10 * s) for s in range(len(hw))]
            skip = k % len(hw) if k >= 2 else None
            if skip is not None:
                files[skip] = None
            slots.load(files)
            slots.out.fill_(77)
            g.replay()
            got, err = slots.images(), slots.err.cpu().numpy()
            assert not err.any(), (k, err)
            for s, f in enumerate(files):
                if f is None:
                    assert (got[s] == 77).all(), (k, s)             # a skipped slot's output is not written
                else:
                    assert np.array_equal(got[s], jc.decode(f)), (words, k, s)


def test_corrupt_frames_set_only_their_slot(cplib):
    img = _frame(120, 160, 5)
    good = [jc.encode(img, "420", 90), jc.encode(img, "444", 70, restart=3), jc.encode(img, "gray", 60)]
    bad = {1: (_truncated(jc.encode(img, "420", 90)), _lib.JPEG_ERR_SHORT),
           3: (_invalid_code(jc.encode(img, "422", 90)), _lib.JPEG_ERR_CODE),
           5: (_wrong_rst(jc.encode(img, "420", 90, restart=2)), _lib.JPEG_ERR_RESTART)}
    files = [good[0], bad[1][0], good[1], bad[3][0], good[2], bad[5][0]]
    for words in (0, 1):
        slots = _Slots(cplib, [(120, 160)] * 6, [2 * len(f) for f in files], words)
        slots.load(files)
        slots.decode()
        got, err = slots.images(), slots.err.cpu().numpy()
        for k in range(len(files)):
            if k in bad:
                assert err[k] & bad[k][1], (k, err[k])
            else:
                assert err[k] == 0 and np.array_equal(got[k], jc.decode(files[k])), k


# ---------------------------------------------------------------- the detection graphs
H, W = 480, 640
SIZES = [(480, 640), (720, 1280), (512, 384), (480, 640)]


def _cams(sizes):
    return _slot_cameras(sizes)


def _mjpeg_steps(sizes, seed, steps=STEPS):
    return [[_changing(k + s, hw, seed + 50 * s) for s, hw in enumerate(sizes)] for k in range(steps)]


@pytest.mark.parametrize("S", [1, 4])
def test_detect_graph_one_size(S, cplib):
    det = _det_detector()
    sizes = [(H, W)] * S
    cams = _cams(sizes)
    g = cpb.DetectGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cams, pixel_format="mjpeg")
    assert g.pixel_format == "mjpeg"
    _capacity(det, S)
    hits = 0
    for k, fs in enumerate(_mjpeg_steps(sizes, 500 + S)):
        # bytes, numpy and pinned CPU tensors
        form = [fs[0]] + [np.frombuffer(f, np.uint8) if k % 2 else torch.from_numpy(
            np.frombuffer(f, np.uint8).copy()).pin_memory() for f in fs[1:]]
        got = g(form)
        hits += _check(k, got, det.run_batch(fs, cams, pixel_format="jpeg"), (S,))
        assert not g.decode_errors.any()
    assert hits > 0


def test_detect_graph_mixed_formats_and_distortion(cplib):
    from tests.test_gpu_pixel_formats import encode as colour_encode
    det = _det_detector()
    S, cams = len(SIZES), _cams(SIZES)
    fmts, ref_fmts = ["mjpeg", "nv12", "bgr", "mjpeg"], ["jpeg", "nv12", "bgr", "jpeg"]
    for dists in (None, [PLUMB, None, None, None]):
        g = cpb.DetectGraph(det, slots=S, frame_hw=SIZES, camera_matrix=cams, pixel_format=fmts, distortion=dists,
                            max_frame_bytes=[2 << 20, 1, 1, 2 << 20] if dists is None else None)
        _capacity(det, S)
        hits = 0
        for k, fs in enumerate(_mjpeg_steps(SIZES, 600)):
            fr = [fs[0], colour_encode(_frame(*SIZES[1], 610 + k), "nv12", 0), _frame(*SIZES[2], 620 + k), fs[3]]
            got = g(fr)
            hits += _check(k, got, det.run_batch(fr, cams, pixel_format=ref_fmts, distortion=dists), (S,))
        assert hits > 0


LIVE = [{0, 2, 3}, {0, 2}, {0, 1, 2, 3}, {1, 2}, set(), {0, 1, 3}]


def test_detect_graph_idle_slots(cplib):
    det = _det_detector()
    S, cams = len(SIZES), _cams(SIZES)
    g = cpb.DetectGraph(det, slots=S, frame_hw=SIZES, camera_matrix=cams, pixel_format="mjpeg", idle_slots=True)
    _capacity(det, S)
    hits = 0
    for k, (fs, lv) in enumerate(zip(_mjpeg_steps(SIZES, 700, len(LIVE)), LIVE)):
        fs = [f if i in lv else None for i, f in enumerate(fs)]
        got = g(fs)
        hits += _check(k, got, _scattered(lambda fr, c: det.run_batch(fr, c, pixel_format="jpeg"), fs, cams, (S,)),
                       (S,))
    assert hits > 0


def test_multi_category_detect_graph(det_checkpoints, cplib):
    mdet = cpb.MultiCategoryDetector(cpb.default_opt("dla_34"), det_checkpoints)
    sizes = SIZES[:2]
    cams = _cams(sizes)
    g = cpb.MultiCategoryDetectGraph(mdet, slots=2, frame_hw=sizes, camera_matrix=cams, pixel_format="mjpeg")
    _capacity(mdet, 2)
    hits = 0
    for k, fs in enumerate(_mjpeg_steps(sizes, 800)):
        hits += _check(k, g(fs), mdet.run_batch(fs, cams, pixel_format="jpeg"), (2, 2))
    assert hits > 0


def test_corrupt_frame_in_detect_graph(cplib):
    det = _det_detector()
    S, cams = 3, _cams([(H, W)] * 3)
    g = cpb.DetectGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cams, pixel_format="mjpeg")
    _capacity(det, S)
    for k, fs in enumerate(_mjpeg_steps([(H, W)] * S, 900, 3)):
        want = det.run_batch(fs, cams, pixel_format="jpeg")
        bad = list(fs)
        bad[1] = (_invalid_code, _truncated, _invalid_code)[k](fs[1])
        gp, gn = [t.cpu().numpy() for t in g(bad)]
        err = g.decode_errors.cpu().numpy()
        assert err[1] and not err[[0, 2]].any() and gn[1] == 0, (k, err, gn)
        for s in (0, 2):
            assert gn[s] == want[1][s] and np.array_equal(gp[s], want[0][s]), (k, s)
        assert want[1].sum() > 0


# ---------------------------------------------------------------- the tracking graphs
SCHEDULE = [  # per step: which slots are live ("new": starts a video), slot 1 starts late, slot 2 pauses
    ["new", None, "new", "new"], [True, "new", True, True], [True, True, None, True], [True, True, True, "new"],
    [None, True, True, True], ["new", True, True, True]]


@pytest.mark.parametrize("hungarian", [False, True])
def test_track_graph_idle_slots(hungarian, cplib):
    det = _trk_detector(hungarian)
    S, cams = len(SIZES), _cams(SIZES)
    tg = cpb.TrackGraph(det, slots=S, frame_hw=SIZES, camera_matrix=cams, pixel_format="mjpeg", idle_slots=True,
                        max_frame_bytes=2 << 20)
    total = 0
    for k, (row, fs) in enumerate(zip(SCHEDULE, _mjpeg_steps(SIZES, 1000, len(SCHEDULE)))):
        fs = [None if e is None else f for e, f in zip(row, fs)]
        new = [e == "new" for e in row]
        got = tg(fs, new_video=new)
        total += _check_step(k, got, det.run_batch(fs, cams, track=True, new_video=new, pixel_format="jpeg"), None,
                             (S,))
    assert total > 0


def test_multi_category_track_graph(trk_checkpoints, cplib):
    trk = _tracker(trk_checkpoints, cats=CATS, hungarian=True)
    sizes = [(H, W)] * 2
    cams = _cams(sizes)
    tg = cpb.MultiCategoryTrackGraph(trk, slots=2, frame_hw=(H, W), camera_matrix=cams, pixel_format="mjpeg")
    total = 0
    for k, fs in enumerate(_mjpeg_steps(sizes, 1100)):
        new = [k == 3, False]
        got = tg(fs, new_video=new)
        total += _check_step(k, got, trk.run_batch(fs, cams, new_video=new, pixel_format="jpeg"), None, (2, 2))
    assert total > 0


def test_corrupt_frame_in_track_graph(cplib):
    det = _trk_detector()
    S, sizes = 3, [(H, W)] * 3
    cams = _cams(sizes)
    tg = cpb.TrackGraph(det, slots=S, frame_hw=sizes, camera_matrix=cams, pixel_format=["mjpeg", "mjpeg", "bgr"])
    video = _mjpeg_steps(sizes, 1200, 6)
    for k, fs in enumerate(video):
        fs[2] = _frame(H, W, 1300 + k)
        new = [False, k == 4, False]
        bad = list(fs)
        if k == 2:
            bad[1] = _invalid_code(fs[1])
        gt, gn = [t.cpu().numpy() for t in tg(bad, new_video=new)]
        wt, wn = det.run_batch(fs, cams, track=True, new_video=new, pixel_format=["jpeg", "jpeg", "bgr"])
        err = tg.decode_errors.cpu().numpy()
        assert bool(err[1]) == (k == 2) and not err[[0, 2]].any(), (k, err)
        # slot 1 differs from its corrupt frame on until its new video; the other slots never do
        same = [0, 2] if k in (2, 3) else [0, 1, 2]
        for s in same:
            assert gn[s] == wn[s] and np.array_equal(gt[s], wt[s]), (k, s)
        if k == 2:
            assert wn.sum() > 0
