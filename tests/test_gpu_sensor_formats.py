"""Sensor formats on the device: every result in "gray" and the four Bayer mosaics (and mixes of them with the colour
formats, one format per frame or slot) equals, bit for bit, the same call on the frames converted to BGR by
cv2.cvtColor:

  * the ops: cp_preprocess_formats at 3 x 3, 5 x 7, 1200 x 1920 and a small frame whose taps leave it on every side,
    at unaligned byte offsets; the graph-safe launches (cp_preprocess_slots_dev, cp_preprocess_slots_ragged_dev and
    cp_preprocess_slots_rows_dev) with their twin and exchange writes; cp_preprocess_remap and a table with maps; and a
    CP_PIX_PER_FRAME table holding all thirteen formats;
  * the product paths: both forms of run_batch, detection and track=True, the two multi-category run_batch calls,
    BatchPipeline and TrackPipeline, DetectGraph / TrackGraph at one size and per-slot sizes with idle slots, the
    multi-category graphs, and a per-slot mix in run_batch(list, track=True) and in an idle-capable TrackGraph built
    with distortion=."""
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import affine_from_center_scale
from centerpose_b200.lens import undistort_map
from tests import bayer_ref
from tests.test_gpu_detect_graph import _capacity, _check, _scattered
from tests.test_gpu_detect_graph import _detector as _det_detector
from tests.test_gpu_pixel_formats import _affines, _f32, _p, _same
from tests.test_gpu_pixel_formats import encode as colour_encode
from tests.test_gpu_pixel_formats import to_bgr as colour_to_bgr
from tests.test_gpu_track_graph import _detector as _trk_detector
from tests.test_gpu_track_graph_multi import _check_step, _place, _slot_cameras, _tracker
from tests.test_gpu_undistort import FISHEYE, PLUMB, RATIONAL
from tests.test_gpu_yuv_input import _cam, _category_checkpoints, _pack

pytestmark = pytest.mark.gpu
SENSOR = bayer_ref.FORMATS
MIX = ["bayer_rggb8", "gray", "nv12", "bgr"]             # a mosaic, a mono camera and two colour ones
SIZES4 = [(601, 803), (481, 640), (512, 512), (720, 1280)]   # NV12 third: even
OPT = cpb.default_opt("dla_34")


def to_bgr(f, fmt):
    """cv2.cvtColor of a frame in fmt to BGR."""
    import cv2
    f = f.cpu().numpy() if torch.is_tensor(f) else f
    if fmt in SENSOR:
        return cv2.cvtColor(f, getattr(cv2, bayer_ref.CV2_CODES[fmt]))
    return colour_to_bgr(f, fmt)


def encode(bgr, fmt, seed=0):
    return bayer_ref.from_bgr(bgr, fmt) if fmt in SENSOR else colour_encode(bgr, fmt, seed)


def _bgr_of(frames, fmts):
    return [None if f is None else to_bgr(f, m) for f, m in zip(frames, fmts)]


def _random(h, w, fmt, seed):
    rng = np.random.default_rng(seed)
    if fmt in SENSOR:
        return rng.integers(0, 256, (h, w), dtype=np.uint8)
    if fmt in ("nv12", "i420"):
        return rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    from tests import yuv422_ref
    return rng.integers(0, 256, (h, w, 3 if fmt == "bgr" else yuv422_ref.CHANNELS[fmt]), dtype=np.uint8)


def _formats_and_bgr(frames, fmts, sizes, ih, iw, trans=None, gaps=None):
    hw = np.array(sizes, np.int32)
    buf, offs = _pack(frames, gaps)
    got = cpb.preprocess_formats(buf, offs, hw, fmts, ih, iw, OPT.mean, OPT.std, trans_input=trans)
    bbuf, boffs = _pack(_bgr_of(frames, fmts))
    want = cpb.preprocess_ragged(bbuf, boffs, hw, ih, iw, OPT.mean, OPT.std, trans_input=trans)
    return got, want


# ---- the ops -----------------------------------------------------------------------------------------------------------
OP_SIZES = [(3, 3), (5, 7), (1200, 1920), (41, 57)]
IH, IW = 256, 384


def _op_affines():
    """fix_res for the tiny frames (every output pixel near a border), 1200 x 1920 rotated, and the small frame placed
    inside the output at 3.3x, so taps leave it on every side."""
    tr = _affines(OP_SIZES, IH, IW)
    tr[0] = affine_from_center_scale(np.array([1.5, 1.5], np.float32), 3.0, IW, IH)
    tr[1] = affine_from_center_scale(np.array([3.5, 2.5], np.float32), 7.0, IW, IH)
    tr[3] = np.array([[3.3, 0.0, 61.25], [0.0, 3.3, 40.5]])
    return tr


@pytest.mark.parametrize("fmt", SENSOR)
def test_formats_call_matches_bgr(fmt, cplib):
    frames = [_random(h, w, fmt, seed=10 + i) for i, (h, w) in enumerate(OP_SIZES)]
    got, want = _formats_and_bgr(frames, [fmt] * 4, OP_SIZES, IH, IW, trans=_op_affines(), gaps=[3, 1, 7, 5])
    _same(got, want, fmt)
    w = want.cpu().numpy()
    assert (w[3, :, 0] == w[3, :, 0, 0, None]).all() and (w[3, :, -1] == w[3, :, 0, 0, None]).all(), "border rows"
    # the array form's launch (uniform sizes, frame b at b * H * W) under the default fix_res affine
    arr = [_random(1200, 1920, fmt, seed=20 + i) for i in range(2)]
    got, want = _formats_and_bgr(arr, [fmt] * 2, [(1200, 1920)] * 2, 512, 512)
    _same(got, want, fmt + " uniform")


def _table(cplib, packed, offs, hw, fmts, ih, iw, trans, maps=None):
    """A frame table of one format (when fmts are all one) or of per-frame formats, with maps when given ->
    (table, launch code)."""
    NS = len(fmts)
    table = torch.zeros(int(cplib.cp_preprocess_frame_table_bytes(NS)), dtype=torch.uint8, device="cuda")
    args = (offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)))
    tr = np.ascontiguousarray(trans, np.float64).ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    one = len(set(fmts)) == 1
    code = L.PIXEL_FORMAT_CODES[fmts[0]] if one else L.CP_PIX_PER_FRAME
    codes = np.array([L.PIXEL_FORMAT_CODES[m] for m in fmts], np.int32)
    cp = None if one else codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
    if maps is not None:
        ptrs = (ctypes.c_void_p * NS)(*[None if m is None else m.data_ptr() for m in maps])
        L.check(cplib.cp_preprocess_frame_table_maps(packed.numel(), *args, code, cp, ptrs, NS, ih, iw, tr, _p(table),
                                                     None), "table maps")
        return table, code | L.CP_PIX_REMAP
    if one:
        L.check(cplib.cp_preprocess_frame_table(packed.numel(), *args, code, NS, ih, iw, tr, _p(table), None), "table")
    else:
        L.check(cplib.cp_preprocess_frame_table_formats(packed.numel(), *args, cp, NS, ih, iw, tr, _p(table), None),
                "table formats")
    return table, code


def _check_table_launches(cplib, packed, table, code, want, ih, iw):
    """slots-ragged with start flags (twin writes) and rows with the store exchange, against want [NS,3,ih,iw]."""
    NS = want.shape[0]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    m, s = _f32(OPT.mean), _f32(OPT.std)
    start = torch.tensor([k % 2 == 0 for k in range(NS)], dtype=torch.int32, device="cuda")
    out = torch.full((NS, 3, ih, iw), float("nan"), device="cuda")
    prev = torch.full_like(out, 7.0)
    L.check(cplib.cp_preprocess_slots_ragged_dev(_p(packed), _p(table), code, NS, ih, iw, m, s, _p(start), _p(out),
                                                 _p(prev), st), "cp_preprocess_slots_ragged_dev")
    _same(out, want, "slots_ragged")
    for b in range(NS):
        _same(prev[b], want[b] if start[b] else torch.full_like(want[b], 7.0), "twin %d" % b)
    rows = list(range(NS - 1, 0, -2)) + [0]                      # live rows in any order, some slots idle
    rows_d = torch.tensor(rows, dtype=torch.int32, device="cuda")
    old = torch.randn((NS, 3, ih, iw), device="cuda")
    store, prev = old.clone(), torch.full((len(rows), 3, ih, iw), float("nan"), device="cuda")
    out = torch.full_like(prev, float("nan"))
    L.check(cplib.cp_preprocess_slots_rows_dev(_p(packed), _p(table), code, _p(rows_d), len(rows), ih, iw, m, s,
                                               _p(start), _p(store), _p(out), _p(prev), st), "rows")
    _same(out, want[np.array(rows)], "rows")
    for k, slot in enumerate(rows):
        _same(prev[k], want[slot] if start[slot] else old[slot], "rows prev %d" % k)
        _same(store[slot], want[slot], "rows store %d" % slot)
    for slot in set(range(NS)) - set(rows):
        _same(store[slot], old[slot], "idle store %d" % slot)


@pytest.mark.parametrize("fmt", SENSOR)
def test_graph_safe_launches_match_bgr(fmt, cplib):
    frames = [encode(synth.synthetic_frames(1, h, w, seed=40 + i)[0], fmt) if h > 8 else _random(h, w, fmt, 40 + i)
              for i, (h, w) in enumerate(OP_SIZES)]
    packed, offs = _pack(frames, [3, 1, 2, 5])
    hw, trans = np.array(OP_SIZES, np.int32), _op_affines()
    _, want = _formats_and_bgr(frames, [fmt] * 4, OP_SIZES, IH, IW, trans=trans)
    table, code = _table(cplib, packed, offs, hw, [fmt] * 4, IH, IW, trans)
    _check_table_launches(cplib, packed, table, code, want, IH, IW)
    # the uniform launch: B frames of one size at b * H * W, with its twin writes
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    m, s = _f32(OPT.mean), _f32(OPT.std)
    arr = [encode(synth.synthetic_frames(1, 481, 643, seed=60 + i)[0], fmt) for i in range(3)]
    tr = np.ascontiguousarray(_affines([(481, 643)], IH, IW)[0], np.float64)
    start = torch.tensor([1, 0, 1], dtype=torch.int32, device="cuda")
    outs = []
    for src, c in ((np.stack(arr), L.PIXEL_FORMAT_CODES[fmt]), (np.stack(_bgr_of(arr, [fmt] * 3)), L.CP_PIX_BGR)):
        src = torch.from_numpy(src).cuda()
        out = torch.full((3, 3, IH, IW), float("nan"), device="cuda")
        prev = torch.full_like(out, 7.0)
        L.check(cplib.cp_preprocess_slots_dev(_p(src), c, 3, 481, 643, IH, IW,
                                              tr.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), m, s, _p(start),
                                              _p(out), _p(prev), st), "cp_preprocess_slots_dev")
        outs.append((out, prev))
    _same(outs[0][0], outs[1][0], "slots")
    _same(outs[0][1], outs[1][1], "slots twin")


@pytest.mark.parametrize("fmt", SENSOR + ("mixed",))
def test_remap_launches_match_bgr(fmt, cplib):
    ih, iw = 384, 512
    sizes = [(1200, 1920), (481, 643), (41, 57), (600, 800)]
    fmts = ["bayer_bggr8", "gray", "bayer_grbg8", "bayer_gbrg8"] if fmt == "mixed" else [fmt] * 4
    dists = [PLUMB, None, FISHEYE, RATIONAL]
    frames = [encode(synth.synthetic_frames(1, h, w, seed=80 + i)[0], f) for i, ((h, w), f) in
              enumerate(zip(sizes, fmts))]
    cams = [_cam(h, w) for h, w in sizes]
    packed, offs = _pack(frames, [1, 2, 3, 5])
    hw = np.array(sizes, np.int32)
    trans = np.stack([affine_from_center_scale(np.array([w / 2., h / 2.], np.float32), float(max(h, w)), iw, ih)
                      for h, w in sizes])
    maps = [None if d is None else torch.from_numpy(undistort_map(d, K, s, (ih, iw))).cuda()
            for d, K, s in zip(dists, cams, sizes)]
    got = cpb.preprocess_remap(packed, offs, hw, fmts, maps, ih, iw, OPT.mean, OPT.std, trans_input=trans)
    bbuf, boffs = _pack(_bgr_of(frames, fmts))
    want = cpb.preprocess_remap(bbuf, boffs, hw, "bgr", maps, ih, iw, OPT.mean, OPT.std, trans_input=trans)
    _same(got, want, "remap")
    table, code = _table(cplib, packed, offs, hw, fmts, ih, iw, trans, maps)
    _check_table_launches(cplib, packed, table, code, want, ih, iw)


def test_per_frame_table_of_all_thirteen_formats(cplib):
    fmts = list(L.PIXEL_FORMATS + L.SENSOR_FORMATS)
    assert len(fmts) == 13
    sizes = [(480, 640), (720, 1280), (36, 62), (481, 640), (37, 62), (1081, 1920), (300, 200), (601, 800),
             (1200, 1920), (3, 3), (5, 7), (41, 57), (121, 163)]
    frames = [_random(h, w, m, seed=90 + i) if min(h, w) < 40 else encode(synth.synthetic_frames(1, h, w, 90 + i)[0], m)
              for i, ((h, w), m) in enumerate(zip(sizes, fmts))]
    trans = _affines(sizes, IH, IW)
    got, want = _formats_and_bgr(frames, fmts, sizes, IH, IW, trans=trans, gaps=[k % 5 for k in range(13)])
    _same(got, want, "thirteen")
    packed, offs = _pack(frames, [k % 3 for k in range(13)])
    table, code = _table(cplib, packed, offs, np.array(sizes, np.int32), fmts, IH, IW, trans)
    assert code == L.CP_PIX_PER_FRAME
    _check_table_launches(cplib, packed, table, code, want, IH, IW)
    # each row equals its single-format launch
    for b in range(9, 13):
        one, _ = _formats_and_bgr([frames[b]], [fmts[b]], [sizes[b]], IH, IW, trans=trans[b:b + 1])
        _same(got[b:b + 1], one, fmts[b])


# ---- run_batch ---------------------------------------------------------------------------------------------------------
def _det(frames_bgr):
    from tests.test_gpu_yuv_input import _detector
    return _detector("dla_34", frames_bgr)[0]


@pytest.mark.parametrize("fmt", ["bayer_rggb8", "gray"])
def test_run_batch_matches_bgr(fmt, cplib):
    arr = np.stack([encode(f, fmt) for f in synth.synthetic_frames(3, 481, 643, seed=11)])
    sizes = [(480, 640), (601, 803), (720, 960)]
    lst = [encode(synth.synthetic_frames(1, h, w, seed=20 + i)[0], fmt) for i, (h, w) in enumerate(sizes)]
    det = _det(_bgr_of(list(arr) + lst, [fmt] * 6))
    cam = _cam(481, 643)
    wp, wn = det.run_batch(np.stack(_bgr_of(arr, [fmt] * 3)), cam)
    assert wn.sum() > 0
    for src in (arr, torch.from_numpy(arr).pin_memory(), torch.from_numpy(arr).cuda()):
        gp, gn = det.run_batch(src, cam, pixel_format=fmt)
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    cams = np.stack([_cam(h, w) for h, w in sizes])
    wp, wn = det.run_batch(_bgr_of(lst, [fmt] * 3), cams)
    assert wn.sum() > 0
    mixed = [lst[0], torch.from_numpy(lst[1]).pin_memory(), torch.from_numpy(lst[2]).cuda()]
    for pf in (fmt, [fmt] * 3):
        gp, gn = det.run_batch(mixed, cams, pixel_format=pf)
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    # every pattern in one list, and a per-frame mix with colour formats, with distortion
    pats = list(bayer_ref.BAYER)
    lst4 = [encode(synth.synthetic_frames(1, h, w, seed=30 + i)[0], m) for i, ((h, w), m) in
            enumerate(zip(SIZES4, pats))]
    cams4 = np.stack([_cam(h, w) for h, w in SIZES4])
    wp, wn = det.run_batch(_bgr_of(lst4, pats), cams4)
    gp, gn = det.run_batch(lst4, cams4, pixel_format=pats)
    assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    lst4 = [encode(synth.synthetic_frames(1, h, w, seed=40 + i)[0], m) for i, ((h, w), m) in enumerate(zip(SIZES4, MIX))]
    dists = [PLUMB, None, FISHEYE, None]
    wp, wn = det.run_batch(_bgr_of(lst4, MIX), cams4, distortion=dists)
    gp, gn = det.run_batch(lst4, cams4, pixel_format=MIX, distortion=dists)
    assert np.array_equal(gn, wn) and np.array_equal(gp, wp)


# per step: per slot True (a frame), None (idle), "new" (a new video starts in the slot)
SCHEDULE = [["new", "new", "new", None], [True, True, None, "new"], ["new", True, True, True], [True, None, True, True]]


def _slot_video(fmts, seed, sizes=SIZES4):
    bases = [synth.synthetic_frames(1, h, w, seed=seed + i)[0] for i, (h, w) in enumerate(sizes)]
    steps = []
    for k, row in enumerate(SCHEDULE):
        fs = [None if e is None else encode(np.roll(b, (2 * k, 3 * k), axis=(0, 1)), m, seed=k)
              for b, e, m in zip(bases, row, fmts)]
        steps.append((fs, [e == "new" for e in row]))
    return steps


@pytest.mark.parametrize("fmts", [["bayer_gbrg8"] * 4, MIX], ids=["bayer_gbrg8", "mixed"])
def test_slot_tracking_matches_bgr(fmts, cplib):
    det = _trk_detector()
    cams = _slot_cameras(SIZES4)
    pf = fmts[0] if len(set(fmts)) == 1 else fmts
    runs = []
    for conv in (False, True):
        det.reset_tracking()
        out = []
        for fs, new in _slot_video(fmts, seed=300):
            out.append(det.run_batch(_bgr_of(fs, fmts) if conv else fs, cams, track=True, new_video=new,
                                     **({} if conv else {"pixel_format": pf})))
        if len(set(fmts)) == 1:                          # the array form, one size
            arr = np.stack([encode(f, fmts[0]) for f in synth.synthetic_frames(4, 512, 512, seed=9)])
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
    arr = np.stack([encode(f, "bayer_bggr8") for f in synth.synthetic_frames(2, 512, 512, seed=5)])
    cam = _cam(512, 512)
    wp, wn = mdet.run_batch(np.stack(_bgr_of(arr, ["bayer_bggr8"] * 2)), cam)
    gp, gn = mdet.run_batch(arr, cam, pixel_format="bayer_bggr8")
    assert wn.sum() > 0 and np.array_equal(gn, wn) and np.array_equal(gp, wp)
    lst = [encode(f, m) for f, m in zip(synth.synthetic_frames(2, 512, 512, seed=6), ["gray", "bayer_grbg8"])]
    wp, wn = mdet.run_batch(_bgr_of(lst, ["gray", "bayer_grbg8"]), cam)
    gp, gn = mdet.run_batch(lst, cam, pixel_format=["gray", "bayer_grbg8"])
    assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    opt, paths = _category_checkpoints(tmp_path, True)
    trk = cpb.MultiCategoryTracker(opt, paths)
    cams = _slot_cameras(SIZES4)
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
    fmt = "bayer_rggb8"
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
    # TrackPipeline with mono cameras
    trk = _trk_detector()
    cams = _slot_cameras(SIZES4)
    outs = []
    for pf in ("gray", "bgr"):
        trk.reset_tracking()
        pipe = cpb.TrackPipeline(trk, slots=4, camera_matrix=cams, pixel_format=pf)
        got = []
        for fs, new in _slot_video(["gray"] * 4, seed=700):
            fs = _bgr_of(fs, ["gray"] * 4) if pf == "bgr" else fs
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
    ("one", ["bayer_rggb8"] * 3, False, "pinned"),
    ("one", ["gray"] * 4, True, "device"),
    ("per-slot", ["bayer_bggr8"] * 4, False, "device"),
    ("per-slot", MIX, True, "pinned"),
]


@pytest.mark.parametrize("kind, fmts, idle, where", DETECT_CASES, ids=["bayer_rggb8", "gray idle", "bggr per-slot",
                                                                       "mixed idle"])
def test_detect_graph_matches_bgr(kind, fmts, idle, where, cplib):
    det = _det_detector()
    S = len(fmts)
    sizes = [(481, 643)] * S if kind == "one" else SIZES4
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


TRACK_CASES = [  # frame sizes, formats, idle slots, distortion
    ("one", ["bayer_grbg8"] * 4, True, None),
    ("per-slot", ["gray"] * 4, False, None),
    ("per-slot", MIX, True, [PLUMB, None, FISHEYE, RATIONAL]),
]


@pytest.mark.parametrize("kind, fmts, idle, dists", TRACK_CASES, ids=["grbg idle", "gray per-slot",
                                                                      "mixed idle distortion"])
def test_track_graph_matches_bgr(kind, fmts, idle, dists, cplib):
    det = _trk_detector(hungarian=True)
    S = len(fmts)
    sizes = [(480, 640)] * S if kind == "one" else SIZES4
    cams = _slot_cameras(sizes)
    pf = fmts if kind == "per-slot" else fmts[0]
    tg = cpb.TrackGraph(det, slots=S, frame_hw=sizes[0] if kind == "one" else sizes, camera_matrix=cams,
                        pixel_format=pf, idle_slots=idle, distortion=dists)
    code = L.CP_PIX_PER_FRAME if len(set(fmts)) > 1 else L.PIXEL_FORMAT_CODES[fmts[0]]
    assert tg._fmt == (code | L.CP_PIX_REMAP if dists else code)
    total = 0
    for k, fs in enumerate(_graph_video(sizes, fmts, seed=800, idle=idle)):
        new = [True, False, False, True] if k == 4 else None
        got = tg([None if f is None else _place(f, "device" if k % 2 else "pinned") for f in fs], new_video=new)
        want = det.run_batch(_bgr_of(fs, fmts), cams, track=True, new_video=new, distortion=dists)
        total += _check_step(k, got, want, None, (S,))
    assert total > 0


def test_multi_category_graphs_match_bgr(tmp_path, cplib):
    for d in ("det", "trk"):
        (tmp_path / d).mkdir()
    opt, paths = _category_checkpoints(tmp_path / "det", False)
    mdet = cpb.MultiCategoryDetector(opt, paths)
    S, cams = 4, _slot_cameras(SIZES4)
    g = cpb.MultiCategoryDetectGraph(mdet, slots=S, frame_hw=SIZES4, camera_matrix=cams, pixel_format=MIX,
                                     idle_slots=True)
    _capacity(mdet, S)
    hits = 0
    for k, fs in enumerate(_graph_video(SIZES4, MIX, seed=380, idle=True)):
        want = _scattered(lambda fr, c: mdet.run_batch(fr, c), _bgr_of(fs, MIX), cams, (2, S))
        hits += _check(k, g([None if f is None else _place(f, "device") for f in fs]), want, (2, S))
    assert hits > STEPS // 2, hits
    trk = _tracker(_category_checkpoints(tmp_path / "trk", True)[1], cats=("chair", "cup"), hungarian=True)
    tg = cpb.MultiCategoryTrackGraph(trk, slots=S, frame_hw=(480, 640), camera_matrix=_slot_cameras([(480, 640)] * S),
                                     pixel_format="bayer_rggb8")
    total = 0
    for k, fs in enumerate(_graph_video([(480, 640)] * S, ["bayer_rggb8"] * S, seed=820, idle=False)):
        got = tg(_place(np.stack(fs), "pinned"))
        want = trk.run_batch(_bgr_of(fs, ["bayer_rggb8"] * S), _slot_cameras([(480, 640)] * S))
        total += _check_step(k, got, want, None, (2, S))
    assert total > 0
