"""Camera pixel formats on the device: every result in "rgb24", "rgba", "bgra", "yuyv422" and "uyvy422" (and mixes of
them with "bgr" / "nv12" / "i420", one format per frame or slot) equals, bit for bit, the same call on the frames
converted to BGR by cv2.cvtColor:

  * the ops: cp_preprocess_formats on every 4:2:2 (Y, U, V) triple, on ragged batches of odd heights at unaligned byte
    offsets under affines whose taps leave the frame, and on a mixed batch (which also equals the per-frame
    single-format launches); the graph-safe launches (cp_preprocess_slots_dev, cp_preprocess_slots_ragged_dev,
    cp_preprocess_slots_rows_dev over one-format and per-frame tables) with their start-flag twin and store writes;
  * the product paths: both forms of run_batch, detection and track=True, the two multi-category run_batch calls,
    BatchPipeline and TrackPipeline, DetectGraph / TrackGraph at one size and per-slot sizes with idle slots, the
    multi-category graphs, and per-slot mixed formats in run_batch(list, track=True) and in an idle-capable TrackGraph."""
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import affine_from_center_scale
from tests import yuv422_ref
from tests.test_gpu_detect_graph import _capacity, _check, _scattered
from tests.test_gpu_detect_graph import _detector as _det_detector
from tests.test_gpu_track_graph import _detector as _trk_detector
from tests.test_gpu_track_graph_multi import _check_step, _place, _slot_cameras, _tracker
from tests.test_gpu_yuv_input import _cam, _category_checkpoints, _pack
from tests.test_gpu_yuv_input import from_bgr as yuv420_from_bgr
from tests.test_gpu_yuv_input import to_bgr as yuv420_to_bgr

pytestmark = pytest.mark.gpu
NEW = ("rgb24", "rgba", "bgra", "yuyv422", "uyvy422")
MIX = ["nv12", "yuyv422", "rgb24", "bgra"]               # cameras of four kinds
OPT = cpb.default_opt("dla_34")


def to_bgr(f, fmt):
    """cv2.cvtColor of a frame in fmt to BGR."""
    import cv2
    f = f.cpu().numpy() if torch.is_tensor(f) else f
    if fmt == "bgr":
        return f
    if fmt in ("nv12", "i420"):
        return yuv420_to_bgr(f, fmt)
    return cv2.cvtColor(f, getattr(cv2, yuv422_ref.CV2_CODES[fmt]))


def encode(bgr, fmt, seed=0):
    return yuv420_from_bgr(bgr, fmt) if fmt in ("nv12", "i420") else yuv422_ref.from_bgr(bgr, fmt, seed)


def random_frame(h, w, fmt, seed):
    if fmt in ("nv12", "i420"):
        return np.random.default_rng(seed).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    c = 3 if fmt == "bgr" else yuv422_ref.CHANNELS[fmt]
    return np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)


def _bgr_of(frames, fmts):
    return [None if f is None else to_bgr(f, m) for f, m in zip(frames, fmts)]


def _same(got, want, what):
    got, want = got.cpu().numpy(), want.cpu().numpy()
    bad = np.argwhere(got != want)
    assert bad.size == 0, (what, bad[:8])


def _formats_and_bgr(frames, fmts, dst_h, dst_w, trans=None, gaps=None):
    hw = np.array([to_bgr(f, m).shape[:2] for f, m in zip(frames, fmts)], np.int32)
    buf, offs = _pack(frames, gaps)
    got = cpb.preprocess_formats(buf, offs, hw, fmts, dst_h, dst_w, OPT.mean, OPT.std, trans_input=trans)
    bbuf, boffs = _pack([to_bgr(f, m) for f, m in zip(frames, fmts)])
    want = cpb.preprocess_ragged(bbuf, boffs, hw, dst_h, dst_w, OPT.mean, OPT.std, trans_input=trans)
    return got, want


# ---- the ops -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ("yuyv422", "uyvy422"))
def test_every_yuv422_triple(fmt, cplib):
    f = yuv422_ref.exhaustive_yuv422(fmt)
    # scale 1: every output pixel is one source pixel with weight 2^15, so all 2^24 triples are converted
    got, want = _formats_and_bgr([f], [fmt], 4096, 4096, trans=np.eye(2, 3)[None])
    _same(got, want, fmt)


def _affines(sizes, ih, iw):
    """Per frame: fix_res, then a rotation, an anisotropic scale and a 3x up-scaling near the border -- taps leave the
    frame in all but the first."""
    import cv2
    out = []
    for k, (h, w) in enumerate(sizes):
        kind = k % 4
        if kind == 0:
            out.append(affine_from_center_scale(np.array([w / 2., h / 2.], np.float32), float(max(h, w)), iw, ih))
        elif kind == 1:
            M = cv2.getRotationMatrix2D((w * 0.4, h * 0.55), 30.0, iw / (0.6 * max(h, w)))
            M[:, 2] += np.array([iw / 2. - w * 0.4, ih / 2. - h * 0.55])
            out.append(M)
        elif kind == 2:
            out.append(np.array([[iw / w * 1.3, 0.0, -7.5], [0.0, ih / h * 0.8, 11.25]]))
        else:
            out.append(np.array([[3.1, 0.0, -3.1 * (w - 9.3)], [0.0, 2.9, -2.9 * 1.7]]))
    return np.stack(out)


SIZES = [(481, 640), (720, 1280), (37, 62), (1081, 1920)]            # odd heights


@pytest.mark.parametrize("fmt", NEW)
def test_ragged_batch_matches_bgr(fmt, cplib):
    frames = [random_frame(h, w, fmt, seed=10 + i) for i, (h, w) in enumerate(SIZES)]
    trans = _affines(SIZES, 256, 384)
    got, want = _formats_and_bgr(frames, [fmt] * 4, 256, 384, trans=trans, gaps=[3, 1, 7, 5])
    _same(got, want, fmt)
    # the array form's launch (uniform sizes, frame b at b * bytes) and the default fix_res affine
    arr = [random_frame(480, 640, fmt, seed=20 + i) for i in range(3)]
    got, want = _formats_and_bgr(arr, [fmt] * 3, 512, 512)
    _same(got, want, fmt + " uniform")


def test_mixed_batch_matches_bgr_and_the_single_format_launches(cplib):
    fmts = ["bgr", "nv12", "i420"] + list(NEW)
    sizes = [(480, 640), (720, 1280), (36, 62), (481, 640), (37, 62), (1081, 1920), (300, 200), (601, 800)]
    frames = [random_frame(h, w, m, seed=30 + i) for i, ((h, w), m) in enumerate(zip(sizes, fmts))]
    trans = _affines(sizes, 256, 384)
    got, want = _formats_and_bgr(frames, fmts, 256, 384, trans=trans, gaps=[0, 3, 1, 2, 5, 7, 1, 3])
    _same(got, want, "mixed")
    for b, (f, m) in enumerate(zip(frames, fmts)):
        one, _ = _formats_and_bgr([f], [m], 256, 384, trans=trans[b:b + 1])
        _same(got[b:b + 1], one, m)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _f32(v):
    return (ctypes.c_float * 3)(*[float(x) for x in v])


def _table(cplib, packed, offs, hw, fmts, ih, iw, trans):
    """A frame table of one format (when fmts are all one) or of per-frame formats -> (table, launch format)."""
    NS = len(fmts)
    table = torch.zeros(int(cplib.cp_preprocess_frame_table_bytes(NS)), dtype=torch.uint8, device="cuda")
    args = (offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)))
    tr = np.ascontiguousarray(trans, np.float64)
    if len(set(fmts)) == 1:
        code = L.PIXEL_FORMAT_CODES[fmts[0]]
        L.check(cplib.cp_preprocess_frame_table(packed.numel(), *args, code, NS, ih, iw,
                                                tr.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), _p(table), None), "")
        return table, code
    codes = np.array([L.PIXEL_FORMAT_CODES[m] for m in fmts], np.int32)
    L.check(cplib.cp_preprocess_frame_table_formats(packed.numel(), *args, codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                                    NS, ih, iw, tr.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                    _p(table), None), "")
    return table, L.CP_PIX_PER_FRAME


@pytest.mark.parametrize("fmt", NEW + ("mixed",))
def test_graph_safe_launches_match_bgr(fmt, cplib):
    ih, iw = 256, 384
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    m, s = _f32(OPT.mean), _f32(OPT.std)
    sizes = [(480, 640), (721, 1280), (512, 512), (301, 200), (1081, 1920)]     # NV12 first in the mix: even
    fmts = (MIX + ["uyvy422"]) if fmt == "mixed" else [fmt] * 5
    frames = [encode(synth.synthetic_frames(1, h, w, seed=40 + i)[0], f, seed=i) for i, ((h, w), f) in
              enumerate(zip(sizes, fmts))]
    packed, offs = _pack(frames, [3, 1, 2, 5, 1])
    hw = np.array(sizes, np.int32)
    trans = _affines(sizes, ih, iw)
    table, code = _table(cplib, packed, offs, hw, fmts, ih, iw, trans)
    bbuf, boffs = _pack(_bgr_of(frames, fmts))
    want = cpb.preprocess_ragged(bbuf, boffs, hw, ih, iw, OPT.mean, OPT.std, trans_input=trans)
    NS = len(sizes)
    # slots-ragged, with start flags: the starting slots' input also goes to prev, other rows of prev are untouched
    start = torch.tensor([1, 0, 1, 0, 0], dtype=torch.int32, device="cuda")
    out = torch.full((NS, 3, ih, iw), float("nan"), device="cuda")
    prev = torch.full_like(out, 7.0)
    L.check(cplib.cp_preprocess_slots_ragged_dev(_p(packed), _p(table), code, NS, ih, iw, m, s, _p(start), _p(out),
                                                 _p(prev), st), "cp_preprocess_slots_ragged_dev")
    _same(out, want, "slots_ragged")
    for b in range(NS):
        _same(prev[b], want[b] if start[b] else torch.full_like(want[b], 7.0), "twin %d" % b)
    # rows: live rows in any order, slots 1 and 3 idle; the store exchange with start flags
    rows = [4, 0, 2]
    sel = np.array(rows)
    rows_d = torch.tensor(rows, dtype=torch.int32, device="cuda")
    old = torch.randn((NS, 3, ih, iw), device="cuda")
    store, prev = old.clone(), torch.full((3, 3, ih, iw), float("nan"), device="cuda")
    out = torch.full((3, 3, ih, iw), float("nan"), device="cuda")
    L.check(cplib.cp_preprocess_slots_rows_dev(_p(packed), _p(table), code, _p(rows_d), 3, ih, iw, m, s, _p(start),
                                               _p(store), _p(out), _p(prev), st), "cp_preprocess_slots_rows_dev")
    _same(out, want[sel], "rows")
    for k, slot in enumerate(rows):
        _same(prev[k], want[slot] if start[slot] else old[slot], "rows prev %d" % k)
        _same(store[slot], want[slot], "rows store %d" % slot)
    for slot in (1, 3):
        _same(store[slot], old[slot], "idle store %d" % slot)
    if fmt == "mixed":
        return
    # the uniform launch: B frames of one size at b * bytes, with its twin writes
    arr = [encode(synth.synthetic_frames(1, 481, 640, seed=60 + i)[0], fmt, seed=i) for i in range(3)]
    dev = torch.from_numpy(np.stack(arr)).cuda()
    bgr = torch.from_numpy(np.stack(_bgr_of(arr, [fmt] * 3))).cuda()
    tr = np.ascontiguousarray(trans[0], np.float64)
    outs = []
    for src, code1 in ((dev, L.PIXEL_FORMAT_CODES[fmt]), (bgr, L.CP_PIX_BGR)):
        out = torch.full((3, 3, ih, iw), float("nan"), device="cuda")
        prev = torch.full_like(out, 7.0)
        L.check(cplib.cp_preprocess_slots_dev(_p(src), code1, 3, 481, 640, ih, iw,
                                              tr.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), m, s, _p(start),
                                              _p(out), _p(prev), st), "cp_preprocess_slots_dev")
        outs.append((out, prev))
    _same(outs[0][0], outs[1][0], "slots")
    _same(outs[0][1], outs[1][1], "slots twin")


# ---- run_batch ---------------------------------------------------------------------------------------------------------
def _det(frames_bgr):
    from tests.test_gpu_yuv_input import _detector
    return _detector("dla_34", frames_bgr)[0]


@pytest.mark.parametrize("fmt", NEW)
def test_run_batch_matches_bgr(fmt, cplib):
    arr = np.stack([encode(f, fmt, seed=k) for k, f in enumerate(synth.synthetic_frames(3, 481, 640, seed=11))])
    sizes = [(480, 640), (601, 800), (720, 960)]
    lst = [encode(synth.synthetic_frames(1, h, w, seed=20 + i)[0], fmt, seed=i) for i, (h, w) in enumerate(sizes)]
    det = _det(_bgr_of(list(arr) + lst, [fmt] * 6))
    cam = _cam(481, 640)
    wp, wn = det.run_batch(np.stack(_bgr_of(arr, [fmt] * 3)), cam)
    assert wn.sum() > 0
    for src in (arr, torch.from_numpy(arr).pin_memory(), torch.from_numpy(arr).cuda()):
        gp, gn = det.run_batch(src, cam, pixel_format=fmt)
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    cams = np.stack([_cam(h, w) for h, w in sizes])
    wp, wn = det.run_batch(_bgr_of(lst, [fmt] * 3), cams)
    assert wn.sum() > 0
    mixed = [lst[0], torch.from_numpy(lst[1]).pin_memory(), torch.from_numpy(lst[2]).cuda()]
    for pf in (fmt, [fmt] * 3):                          # one name, or the name once per frame
        gp, gn = det.run_batch(mixed, cams, pixel_format=pf)
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)


def test_run_batch_mixed_formats_match_bgr(cplib):
    sizes = [(480, 640), (601, 800), (720, 960), (512, 512)]
    bgr = [synth.synthetic_frames(1, h, w, seed=70 + i)[0] for i, (h, w) in enumerate(sizes)]
    frames = [encode(f, m, seed=i) for i, (f, m) in enumerate(zip(bgr, MIX))]
    det = _det(_bgr_of(frames, MIX))
    cams = np.stack([_cam(h, w) for h, w in sizes])
    wp, wn = det.run_batch(_bgr_of(frames, MIX), cams)
    gp, gn = det.run_batch(frames, cams, pixel_format=MIX)
    assert wn.sum() > 0 and np.array_equal(gn, wn) and np.array_equal(gp, wp)


TRACK_SIZES = [(480, 640), (601, 800), (512, 512), (720, 1280)]
# per step: per slot True (a frame), None (idle), "new" (a new video starts in the slot)
SCHEDULE = [["new", "new", "new", None], [True, True, None, "new"], ["new", True, True, True], [True, None, True, True]]


def _slot_video(fmts, seed):
    bases = [synth.synthetic_frames(1, h, w, seed=seed + i)[0] for i, (h, w) in enumerate(TRACK_SIZES)]
    steps = []
    for k, row in enumerate(SCHEDULE):
        fs = [None if e is None else encode(np.roll(b, (2 * k, 3 * k), axis=(0, 1)), m, seed=k)
              for b, e, m in zip(bases, row, fmts)]
        steps.append((fs, [e == "new" for e in row]))
    return steps


@pytest.mark.parametrize("fmts", [["yuyv422"] * 4, ["rgba"] * 4, MIX], ids=["yuyv422", "rgba", "mixed"])
def test_slot_tracking_matches_bgr(fmts, cplib):
    det = _trk_detector()
    cams = _slot_cameras(TRACK_SIZES)
    pf = fmts[0] if len(set(fmts)) == 1 else fmts
    runs = []
    for conv in (False, True):
        det.reset_tracking()
        out = []
        for fs, new in _slot_video(fmts, seed=300):
            out.append(det.run_batch(_bgr_of(fs, fmts) if conv else fs, cams, track=True, new_video=new,
                                     **({} if conv else {"pixel_format": pf})))
        if len(set(fmts)) == 1:                          # the array form, one size
            arr = np.stack([encode(f, fmts[0], seed=k) for k, f in enumerate(synth.synthetic_frames(4, 512, 512,
                                                                                                     seed=9))])
            out.append(det.run_batch(np.stack(_bgr_of(arr, fmts)) if conv else arr, _cam(512, 512), track=True,
                                     **({} if conv else {"pixel_format": pf})))
        runs.append(out)
    assert sum(int(n.sum()) for _, n in runs[1]) > 0
    for k, ((gt, gn), (wt, wn)) in enumerate(zip(*runs)):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt), k


# ---- several categories and the pipelines --------------------------------------------------------------------------------
def test_multi_category_calls_match_bgr(tmp_path, cplib):
    opt, paths = _category_checkpoints(tmp_path, False)
    mdet = cpb.MultiCategoryDetector(opt, paths)
    arr = np.stack([encode(f, "uyvy422") for f in synth.synthetic_frames(2, 512, 512, seed=5)])
    cam = _cam(512, 512)
    wp, wn = mdet.run_batch(np.stack(_bgr_of(arr, ["uyvy422"] * 2)), cam)
    gp, gn = mdet.run_batch(arr, cam, pixel_format="uyvy422")
    assert (wn.sum(axis=1) > 0).all() and np.array_equal(gn, wn) and np.array_equal(gp, wp)
    lst = [encode(f, m) for f, m in zip(synth.synthetic_frames(2, 512, 512, seed=6), ["bgra", "nv12"])]
    wp, wn = mdet.run_batch(_bgr_of(lst, ["bgra", "nv12"]), cam)
    gp, gn = mdet.run_batch(lst, cam, pixel_format=["bgra", "nv12"])
    assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    opt, paths = _category_checkpoints(tmp_path, True)
    trk = cpb.MultiCategoryTracker(opt, paths)
    cams = _slot_cameras(TRACK_SIZES)
    runs = []
    for conv in (False, True):
        trk.reset_tracking()
        runs.append([trk.run_batch(_bgr_of(fs, MIX) if conv else fs, cams, new_video=new,
                                   **({} if conv else {"pixel_format": MIX}))
                     for fs, new in _slot_video(MIX, seed=500)])
    assert sum(int(n.sum()) for _, n in runs[1]) > 0
    for k, ((gt, gn), (wt, wn)) in enumerate(zip(*runs)):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt), k


def test_pipelines_match_bgr(cplib):
    fmt = "yuyv422"
    batches = [np.stack([encode(f, fmt) for f in synth.synthetic_frames(2, 480, 640, seed=600 + k)]) for k in range(3)]
    det = _det([f for b in batches for f in _bgr_of(b, [fmt] * 2)])
    cam = _cam(480, 640)
    outs = []
    for pf in (fmt, "bgr"):
        pipe = cpb.BatchPipeline(det, batch=2, height=480, width=640, camera_matrix=cam, pixel_format=pf)
        got = []
        for k, b in enumerate(batches):
            b = np.stack(_bgr_of(b, [fmt] * 2)) if pf == "bgr" else b
            if pipe.in_flight == pipe.depth:
                got.append([a.copy() for a in pipe.collect()])
            pipe.submit(torch.from_numpy(b).pin_memory() if k % 2 else b)
        while pipe.in_flight:
            got.append([a.copy() for a in pipe.collect()])
        outs.append(got)
    assert sum(int(n.sum()) for _, n in outs[1]) > 0
    for (gp, gn), (wp, wn) in zip(*outs):
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    # TrackPipeline with BGRA cameras
    trk = _trk_detector()
    cams = _slot_cameras(TRACK_SIZES)
    outs = []
    for pf in ("bgra", "bgr"):
        trk.reset_tracking()
        pipe = cpb.TrackPipeline(trk, slots=4, camera_matrix=cams, pixel_format=pf)
        got = []
        for k, (fs, new) in enumerate(_slot_video(["bgra"] * 4, seed=700)):
            fs = _bgr_of(fs, ["bgra"] * 4) if pf == "bgr" else fs
            if pipe.in_flight == pipe.depth:
                got.append(pipe.collect())
            pipe.submit(fs, new_video=new)
        while pipe.in_flight:
            got.append(pipe.collect())
        outs.append(got)
    assert sum(int(n.sum()) for _, n in outs[1]) > 0
    for (gt, gn), (wt, wn) in zip(*outs):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt)


# ---- the graphs --------------------------------------------------------------------------------------------------------
STEPS = 6
LIVE = [{0, 2, 3}, {0, 1, 2, 3}, {1, 2}, set(), {0, 1, 3}, {0, 1, 2, 3}]


def _graph_video(sizes, fmts, seed, idle):
    bases = [synth.synthetic_frames(1, h, w, seed=seed + i)[0] for i, (h, w) in enumerate(sizes)]
    return [[encode(np.roll(b, (2 * k, 3 * k), axis=(0, 1)), m, seed=k) if (not idle or i in LIVE[k]) else None
             for i, (b, m) in enumerate(zip(bases, fmts))] for k in range(STEPS)]


DETECT_CASES = [  # frame sizes, formats, idle slots, where
    ("one", ["rgb24"] * 3, False, "pinned"),
    ("one", ["uyvy422"] * 4, True, "device"),
    ("per-slot", ["bgra"] * 4, False, "device"),
    ("per-slot", MIX, True, "pinned"),
]


@pytest.mark.parametrize("kind, fmts, idle, where", DETECT_CASES, ids=["rgb24", "uyvy422 idle", "bgra per-slot",
                                                                       "mixed idle"])
def test_detect_graph_matches_bgr(kind, fmts, idle, where, cplib):
    det = _det_detector()
    S = len(fmts)
    sizes = [(481, 640)] * S if kind == "one" else TRACK_SIZES
    cams = _slot_cameras(sizes)
    pf = fmts[0] if len(set(fmts)) == 1 else fmts
    g = cpb.DetectGraph(det, slots=S, frame_hw=sizes[0] if kind == "one" else sizes, camera_matrix=cams,
                        pixel_format=pf, idle_slots=idle)
    assert g.pixel_format == pf
    _capacity(det, S)
    hits = 0
    for k, fs in enumerate(_graph_video(sizes, fmts, seed=320, idle=idle)):
        bgr = _bgr_of(fs, fmts)
        if idle:
            got = g([None if f is None else _place(f, where) for f in fs])
            want = _scattered(lambda fr, c: det.run_batch(fr, c), bgr, cams, (S,))
        elif kind == "one":
            got = g(_place(np.stack(fs), where))
            want = det.run_batch(np.stack(bgr), cams)
        else:
            got = g([_place(f, where) for f in fs])
            want = det.run_batch(bgr, cams)
        hits += _check(k, got, want, (S,))
    assert hits > STEPS // 2, hits


TRACK_CASES = [  # frame sizes, formats, idle slots
    ("one", ["yuyv422"] * 4, True),
    ("per-slot", ["rgba"] * 4, False),
    ("per-slot", MIX, True),
    ("per-slot", ["rgb24", "rgb24", "rgb24", "rgb24"], True),
]


@pytest.mark.parametrize("kind, fmts, idle", TRACK_CASES, ids=["yuyv422 idle", "rgba per-slot", "mixed idle",
                                                               "one name listed"])
def test_track_graph_matches_bgr(kind, fmts, idle, cplib):
    det = _trk_detector(hungarian=True)
    S = len(fmts)
    sizes = [(480, 640)] * S if kind == "one" else TRACK_SIZES
    cams = _slot_cameras(sizes)
    pf = fmts if kind == "per-slot" else fmts[0]
    tg = cpb.TrackGraph(det, slots=S, frame_hw=sizes[0] if kind == "one" else sizes, camera_matrix=cams,
                        pixel_format=pf, idle_slots=idle)
    assert tg._fmt == (L.CP_PIX_PER_FRAME if len(set(fmts)) > 1 else L.PIXEL_FORMAT_CODES[fmts[0]])
    total = 0
    for k, fs in enumerate(_graph_video(sizes, fmts, seed=800, idle=idle)):
        new = [True, False, False, True] if k == 4 else None
        got = tg([None if f is None else _place(f, "device" if k % 2 else "pinned") for f in fs], new_video=new)
        want = det.run_batch(_bgr_of(fs, fmts), cams, track=True, new_video=new)
        total += _check_step(k, got, want, None, (S,))
    assert total > 0


def test_multi_category_graphs_match_bgr(tmp_path, cplib):
    for d in ("det", "trk"):
        (tmp_path / d).mkdir()
    opt, paths = _category_checkpoints(tmp_path / "det", False)
    mdet = cpb.MultiCategoryDetector(opt, paths)
    S, cams = 4, _slot_cameras(TRACK_SIZES)
    g = cpb.MultiCategoryDetectGraph(mdet, slots=S, frame_hw=TRACK_SIZES, camera_matrix=cams, pixel_format=MIX,
                                     idle_slots=True)
    _capacity(mdet, S)
    hits = 0
    for k, fs in enumerate(_graph_video(TRACK_SIZES, MIX, seed=380, idle=True)):
        want = _scattered(lambda fr, c: mdet.run_batch(fr, c), _bgr_of(fs, MIX), cams, (2, S))
        hits += _check(k, g([None if f is None else _place(f, "device") for f in fs]), want, (2, S))
    assert hits > STEPS // 2, hits
    trk = _tracker(_category_checkpoints(tmp_path / "trk", True)[1], cats=("chair", "cup"), hungarian=True)
    tg = cpb.MultiCategoryTrackGraph(trk, slots=S, frame_hw=(480, 640), camera_matrix=_slot_cameras([(480, 640)] * S),
                                     pixel_format="uyvy422")
    total = 0
    for k, fs in enumerate(_graph_video([(480, 640)] * S, ["uyvy422"] * S, seed=820, idle=False)):
        got = tg(_place(np.stack(fs), "pinned"))
        want = trk.run_batch(_bgr_of(fs, ["uyvy422"] * S), _slot_cameras([(480, 640)] * S))
        total += _check_step(k, got, want, None, (2, S))
    assert total > 0
