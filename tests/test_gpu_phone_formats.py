"""Phone camera frames on the device: every result in "nv21", "yv12" and the four full-range 4:2:0 formats (and mixes of
them with other formats, one per frame or slot) equals, bit for bit, the same call on the frames converted to BGR on the
host (cv2.cvtColor, and for full range the 2x2 chroma replication + COLOR_YCrCb2BGR of tests/phone_ref.py):

  * the ops: cp_preprocess_formats and cp_preprocess_yuv420 at 2 x 2, 6 x 8, 1440 x 1920 and a small frame whose taps
    leave it on every side; the graph-safe launches (uniform, slots-ragged with its twin writes, rows with the store
    exchange); cp_preprocess_remap and a table with maps; a per-frame table of all six next to the other formats;
  * the product paths: both forms of run_batch (detection and track=True, with a "jpeg" frame in a mix, idle slots and
    distortion=), the two multi-category calls, BatchPipeline and TrackPipeline, and the four graphs (one size, per-slot
    sizes, an "mjpeg" slot in a mix, idle slots, distortion=).

And a graph given a camera_matrix on a call steps, at every step, exactly as run_batch with that camera: detection and
tracking, a tracking stream whose camera changes mid-video, a graph with idle slots, and the cameras staying in force
for later calls."""
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import affine_from_center_scale
from centerpose_b200.lens import undistort_map
from tests import phone_ref
from tests.test_gpu_detect_graph import _capacity, _check, _scattered
from tests.test_gpu_detect_graph import _detector as _det_detector
from tests.test_gpu_pixel_formats import _affines, _f32, _p, _same
from tests.test_gpu_sensor_formats import _check_table_launches, _table
from tests.test_gpu_sensor_formats import encode as sensor_encode
from tests.test_gpu_sensor_formats import to_bgr as sensor_to_bgr
from tests.test_gpu_track_graph import _detector as _trk_detector
from tests.test_gpu_track_graph_multi import _check_step, _slot_cameras, _tracker
from tests.test_gpu_undistort import FISHEYE, PLUMB, RATIONAL
from tests.test_gpu_yuv_input import _cam, _category_checkpoints, _pack

pytestmark = pytest.mark.gpu
PHONE = phone_ref.FORMATS
OPT = cpb.default_opt("dla_34")
SIZES4 = [(480, 640), (482, 642), (512, 512), (720, 1280)]      # even: every slot may be 4:2:0
MIX = ["nv21_full", "nv12", "bayer_rggb8", "mjpeg"]             # a phone, a video decoder, a raw sensor, a webcam
RUN_MIX = ["nv21_full", "nv12", "bayer_rggb8", "jpeg"]          # the same cameras through run_batch(list)


def to_bgr(f, fmt):
    """The host conversion of a frame in fmt to BGR: cv2.cvtColor, phone_ref's full-range rule, cv2.imdecode."""
    import cv2
    f = f.cpu().numpy() if torch.is_tensor(f) else f
    if fmt in ("jpeg", "mjpeg"):
        return cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)
    if fmt in PHONE:
        return phone_ref.cv2_bgr(f, fmt)
    return sensor_to_bgr(f, fmt)


def encode(bgr, fmt, seed=0):
    import cv2
    if fmt in ("jpeg", "mjpeg"):
        return cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, 85])[1].reshape(-1)
    return phone_ref.from_bgr(bgr, fmt) if fmt in PHONE else sensor_encode(bgr, fmt, seed)


def _bgr_of(frames, fmts):
    return [None if f is None else to_bgr(f, m) for f, m in zip(frames, fmts)]


def _random(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)


def _place(f, where, fmt):
    if fmt == "mjpeg":                                   # encoded frames stay on the host
        return f
    t = torch.from_numpy(np.ascontiguousarray(f))
    return t.pin_memory() if where == "pinned" else t.cuda()


def _formats_and_bgr(frames, fmts, sizes, ih, iw, trans=None, gaps=None):
    hw = np.array(sizes, np.int32)
    buf, offs = _pack(frames, gaps)
    got = cpb.preprocess_formats(buf, offs, hw, fmts, ih, iw, OPT.mean, OPT.std, trans_input=trans)
    bbuf, boffs = _pack(_bgr_of(frames, fmts))
    want = cpb.preprocess_ragged(bbuf, boffs, hw, ih, iw, OPT.mean, OPT.std, trans_input=trans)
    return got, want


# ---- the ops -----------------------------------------------------------------------------------------------------------
OP_SIZES = [(2, 2), (6, 8), (1440, 1920), (42, 58)]
IH, IW = 256, 384


def _op_affines():
    """fix_res for the tiny frames (every output pixel near a border), 1440 x 1920 rotated, and the small frame placed
    inside the output at 3.3x, so taps leave it on every side."""
    tr = _affines(OP_SIZES, IH, IW)
    tr[0] = affine_from_center_scale(np.array([1.0, 1.0], np.float32), 2.0, IW, IH)
    tr[1] = affine_from_center_scale(np.array([4.0, 3.0], np.float32), 8.0, IW, IH)
    tr[3] = np.array([[3.3, 0.0, 61.25], [0.0, 3.3, 40.5]])
    return tr


@pytest.mark.parametrize("fmt", PHONE)
def test_formats_and_yuv420_calls_match_bgr(fmt, cplib):
    frames = [_random(h, w, seed=10 + i) for i, (h, w) in enumerate(OP_SIZES)]
    trans = _op_affines()
    got, want = _formats_and_bgr(frames, [fmt] * 4, OP_SIZES, IH, IW, trans=trans, gaps=[3, 1, 7, 5])
    _same(got, want, fmt)
    buf, offs = _pack(frames, [3, 1, 7, 5])
    _same(cpb.preprocess_yuv420(buf, offs, np.array(OP_SIZES, np.int32), fmt, IH, IW, OPT.mean, OPT.std,
                                trans_input=trans), want, fmt + " yuv420")
    # camera-like frames of Objectron's size, the array form's launch under the default fix_res affine
    arr = [encode(f, fmt) for f in synth.synthetic_frames(2, 1440, 1920, seed=20)]
    got, want = _formats_and_bgr(arr, [fmt] * 2, [(1440, 1920)] * 2, 512, 512)
    _same(got, want, fmt + " uniform")


@pytest.mark.parametrize("fmt", PHONE)
def test_graph_safe_launches_match_bgr(fmt, cplib):
    frames = [encode(synth.synthetic_frames(1, h, w, seed=40 + i)[0], fmt) if h > 8 else _random(h, w, 40 + i)
              for i, (h, w) in enumerate(OP_SIZES)]
    packed, offs = _pack(frames, [3, 1, 2, 5])
    hw, trans = np.array(OP_SIZES, np.int32), _op_affines()
    _, want = _formats_and_bgr(frames, [fmt] * 4, OP_SIZES, IH, IW, trans=trans)
    table, code = _table(cplib, packed, offs, hw, [fmt] * 4, IH, IW, trans)
    assert code == L.PIXEL_FORMAT_CODES[fmt]
    _check_table_launches(cplib, packed, table, code, want, IH, IW)
    # the uniform launch: B frames of one size at b * 3HW/2, with its twin writes
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    m, s = _f32(OPT.mean), _f32(OPT.std)
    arr = [encode(synth.synthetic_frames(1, 480, 642, seed=60 + i)[0], fmt) for i in range(3)]
    tr = np.ascontiguousarray(_affines([(480, 642)], IH, IW)[0], np.float64)
    start = torch.tensor([1, 0, 1], dtype=torch.int32, device="cuda")
    outs = []
    for src, c in ((np.stack(arr), L.PIXEL_FORMAT_CODES[fmt]), (np.stack(_bgr_of(arr, [fmt] * 3)), L.CP_PIX_BGR)):
        src = torch.from_numpy(src).cuda()
        out = torch.full((3, 3, IH, IW), float("nan"), device="cuda")
        prev = torch.full_like(out, 7.0)
        L.check(cplib.cp_preprocess_slots_dev(_p(src), c, 3, 480, 642, IH, IW,
                                              tr.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), m, s, _p(start),
                                              _p(out), _p(prev), st), "cp_preprocess_slots_dev")
        outs.append((out, prev))
    _same(outs[0][0], outs[1][0], "slots")
    _same(outs[0][1], outs[1][1], "slots twin")


@pytest.mark.parametrize("fmts", [["nv12_full"] * 4, ["yv12", "nv21_full", "i420_full", "bayer_gbrg8"]],
                         ids=["nv12_full", "mixed"])
def test_remap_launches_match_bgr(fmts, cplib):
    ih, iw = 384, 512
    sizes = [(1440, 1920), (480, 642), (42, 58), (600, 800)]
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


def test_per_frame_table_of_every_format(cplib):
    fmts = list(PHONE) + ["nv12", "i420", "bgr", "bayer_rggb8", "gray", "yuyv422", "rgba"]
    sizes = [(480, 640), (720, 1280), (2, 2), (482, 642), (36, 62), (1440, 1920), (300, 200), (600, 800), (121, 163),
             (5, 7), (41, 57), (64, 96), (33, 47)]
    frames = [_random(h, w, 90 + i) if m in PHONE and min(h, w) < 40
              else encode(synth.synthetic_frames(1, h, w, 90 + i)[0], m) for i, ((h, w), m) in enumerate(zip(sizes, fmts))]
    trans = _affines(sizes, IH, IW)
    got, want = _formats_and_bgr(frames, fmts, sizes, IH, IW, trans=trans, gaps=[k % 5 for k in range(13)])
    _same(got, want, "every format")
    packed, offs = _pack(frames, [k % 3 for k in range(13)])
    table, code = _table(cplib, packed, offs, np.array(sizes, np.int32), fmts, IH, IW, trans)
    assert code == L.CP_PIX_PER_FRAME
    _check_table_launches(cplib, packed, table, code, want, IH, IW)
    for b in range(6):                                   # each row equals its single-format launch
        one, _ = _formats_and_bgr([frames[b]], [fmts[b]], [sizes[b]], IH, IW, trans=trans[b:b + 1])
        _same(got[b:b + 1], one, fmts[b])


# ---- run_batch ---------------------------------------------------------------------------------------------------------
def _det(frames_bgr):
    from tests.test_gpu_yuv_input import _detector
    return _detector("dla_34", frames_bgr)[0]


@pytest.mark.parametrize("fmt", ["nv12_full", "nv21", "yv12_full"])
def test_run_batch_matches_bgr(fmt, cplib):
    arr = np.stack([encode(f, fmt) for f in synth.synthetic_frames(3, 480, 642, seed=11)])
    sizes = [(480, 640), (600, 802), (720, 960)]
    lst = [encode(synth.synthetic_frames(1, h, w, seed=20 + i)[0], fmt) for i, (h, w) in enumerate(sizes)]
    det = _det(_bgr_of(list(arr) + lst, [fmt] * 6))
    cam = _cam(480, 642)
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
    # a per-frame mix with a JPEG, with and without distortion
    lst4 = [encode(synth.synthetic_frames(1, h, w, seed=40 + i)[0], m) for i, ((h, w), m) in
            enumerate(zip(SIZES4, RUN_MIX))]
    cams4 = np.stack([_cam(h, w) for h, w in SIZES4])
    for dists in (None, [PLUMB, None, FISHEYE, None]):
        wp, wn = det.run_batch(_bgr_of(lst4, RUN_MIX), cams4, distortion=dists)
        gp, gn = det.run_batch(lst4, cams4, pixel_format=RUN_MIX, distortion=dists)
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    # the array form with distortion
    wp, wn = det.run_batch(np.stack(_bgr_of(arr, [fmt] * 3)), cam, distortion=PLUMB)
    gp, gn = det.run_batch(arr, cam, pixel_format=fmt, distortion=PLUMB)
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


@pytest.mark.parametrize("fmts", [["i420_full"] * 4, RUN_MIX], ids=["i420_full", "mixed"])
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
    arr = np.stack([encode(f, "nv12_full") for f in synth.synthetic_frames(2, 512, 512, seed=5)])
    cam = _cam(512, 512)
    wp, wn = mdet.run_batch(np.stack(_bgr_of(arr, ["nv12_full"] * 2)), cam)
    gp, gn = mdet.run_batch(arr, cam, pixel_format="nv12_full")
    assert wn.sum() > 0 and np.array_equal(gn, wn) and np.array_equal(gp, wp)
    lst = [encode(f, m) for f, m in zip(synth.synthetic_frames(2, 512, 512, seed=6), ["yv12", "nv21_full"])]
    wp, wn = mdet.run_batch(_bgr_of(lst, ["yv12", "nv21_full"]), cam)
    gp, gn = mdet.run_batch(lst, cam, pixel_format=["yv12", "nv21_full"])
    assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    opt, paths = _category_checkpoints(tmp_path, True)
    trk = cpb.MultiCategoryTracker(opt, paths)
    cams = _slot_cameras(SIZES4)
    runs = []
    for conv in (False, True):
        trk.reset_tracking()
        runs.append([trk.run_batch(_bgr_of(fs, RUN_MIX) if conv else fs, cams, new_video=new,
                                   **({} if conv else {"pixel_format": RUN_MIX}))
                     for fs, new in _slot_video(RUN_MIX, seed=500)])
    assert sum(int(n.sum()) for _, n in runs[1]) > 0
    for k, ((gt, gn), (wt, wn)) in enumerate(zip(*runs)):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt), k


def test_pipelines_match_bgr(cplib):
    fmt = "nv21_full"
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
    trk = _trk_detector()
    cams = _slot_cameras(SIZES4)
    outs = []
    for pf in ("yv12", "bgr"):
        trk.reset_tracking()
        pipe = cpb.TrackPipeline(trk, slots=4, camera_matrix=cams, pixel_format=pf)
        got = []
        for fs, new in _slot_video(["yv12"] * 4, seed=700):
            fs = _bgr_of(fs, ["yv12"] * 4) if pf == "bgr" else fs
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


def _graph_video(sizes, fmts, seed, idle, steps=STEPS):
    bases = [synth.synthetic_frames(1, h, w, seed=seed + i)[0] for i, (h, w) in enumerate(sizes)]
    return [[encode(np.roll(b, (2 * k, 3 * k), axis=(0, 1)), m, seed=k) if (not idle or i in LIVE[k]) else None
             for i, (b, m) in enumerate(zip(bases, fmts))] for k in range(steps)]


def _moving_cameras(sizes, k):
    """Per-slot cameras of step k: the focal length and principal point move as a phone's do with focus."""
    cams = _slot_cameras(sizes).copy()
    cams[:, 0, 0] *= 1 + 0.03 * k
    cams[:, 1, 1] *= 1 + 0.025 * k
    cams[:, 0, 2] += 1.5 * k
    cams[:, 1, 2] -= k
    return cams


DETECT_CASES = [  # frame sizes, formats, idle slots, where, a camera per step
    ("one", ["nv12_full"] * 3, False, "pinned", False),
    ("one", ["nv21"] * 4, True, "device", True),
    ("per-slot", ["yv12_full"] * 4, False, "device", True),
    ("per-slot", MIX, True, "pinned", False),
]


@pytest.mark.parametrize("kind, fmts, idle, where, moving", DETECT_CASES,
                         ids=["nv12_full", "nv21 idle moving", "yv12_full per-slot moving", "mixed idle"])
def test_detect_graph_matches_bgr(kind, fmts, idle, where, moving, cplib):
    det = _det_detector()
    S = len(fmts)
    sizes = [(480, 642)] * S if kind == "one" else SIZES4
    cams = _slot_cameras(sizes)
    pf = fmts[0] if len(set(fmts)) == 1 else fmts
    g = cpb.DetectGraph(det, slots=S, frame_hw=sizes[0] if kind == "one" else sizes, camera_matrix=cams,
                        pixel_format=pf, idle_slots=idle)
    assert g.pixel_format == pf
    _capacity(det, S)
    hits = 0
    for k, fs in enumerate(_graph_video(sizes, fmts, seed=320, idle=idle)):
        bgr = _bgr_of(fs, fmts)
        kw = {}
        if moving and k % 3 != 2:                        # a new camera on most steps; the last one stays in force
            cams = _moving_cameras(sizes, k)
            kw = {"camera_matrix": cams if k % 2 else torch.from_numpy(cams)}
        if idle:
            got = g([None if f is None else _place(f, where, m) for f, m in zip(fs, fmts)], **kw)
            want = _scattered(lambda fr, c: det.run_batch(fr, c), bgr, cams, (S,))
        elif kind == "one":
            got = g(_place(np.stack(fs), where, fmts[0]), **kw)
            want = det.run_batch(np.stack(bgr), cams)
        else:
            got = g([_place(f, where, m) for f, m in zip(fs, fmts)], **kw)
            want = det.run_batch(bgr, cams)
        hits += _check(k, got, want, (S,))
    assert hits > STEPS // 2, hits


TRACK_CASES = [  # frame sizes, formats, idle slots, distortion, a camera per step
    ("one", ["nv21_full"] * 4, True, None, True),
    ("per-slot", ["i420_full"] * 4, False, None, True),
    ("per-slot", MIX, True, [PLUMB, None, FISHEYE, RATIONAL], False),
    ("one", ["yv12"] * 2, False, None, False),
]


@pytest.mark.parametrize("kind, fmts, idle, dists, moving", TRACK_CASES,
                         ids=["nv21_full idle moving", "i420_full per-slot moving", "mixed idle distortion", "yv12"])
def test_track_graph_matches_bgr(kind, fmts, idle, dists, moving, cplib):
    det = _trk_detector(hungarian=True)
    S = len(fmts)
    sizes = [(480, 640)] * S if kind == "one" else SIZES4
    cams = _slot_cameras(sizes)
    pf = fmts if kind == "per-slot" else fmts[0]
    tg = cpb.TrackGraph(det, slots=S, frame_hw=sizes[0] if kind == "one" else sizes, camera_matrix=cams,
                        pixel_format=pf, idle_slots=idle, distortion=dists)
    code = L.CP_PIX_PER_FRAME if len(set(fmts)) > 1 else L.PIXEL_FORMAT_CODES[fmts[0]]
    assert tg._fmt == (code | L.CP_PIX_REMAP if dists else code)
    ref = ["jpeg" if m == "mjpeg" else m for m in fmts]
    total = 0
    for k, fs in enumerate(_graph_video(sizes, fmts, seed=800, idle=idle)):
        new = [True, False, False, True][:S] if k == 4 else None
        kw = {}
        if moving and k in (1, 2, 4):                     # the camera changes mid-video, then stays in force
            cams = _moving_cameras(sizes, k)
            kw = {"camera_matrix": cams}
        where = "device" if k % 2 else "pinned"
        if kind == "one" and not idle:
            got = tg(_place(np.stack(fs), where, fmts[0]), new_video=new, **kw)
        else:
            got = tg([None if f is None else _place(f, where, m) for f, m in zip(fs, fmts)], new_video=new, **kw)
        want = det.run_batch(_bgr_of(fs, ref), cams, track=True, new_video=new, distortion=dists)
        total += _check_step(k, got, want, None, (S,))
    assert total > 0


def test_multi_category_graphs_match_bgr(tmp_path, cplib):
    for d in ("det", "trk"):
        (tmp_path / d).mkdir()
    opt, paths = _category_checkpoints(tmp_path / "det", False)
    mdet = cpb.MultiCategoryDetector(opt, paths)
    S = 4
    g = cpb.MultiCategoryDetectGraph(mdet, slots=S, frame_hw=SIZES4, camera_matrix=_slot_cameras(SIZES4),
                                     pixel_format=MIX, idle_slots=True)
    _capacity(mdet, S)
    hits = 0
    for k, fs in enumerate(_graph_video(SIZES4, MIX, seed=380, idle=True)):
        cams = _moving_cameras(SIZES4, k)
        want = _scattered(lambda fr, c: mdet.run_batch(fr, c), _bgr_of(fs, MIX), cams, (2, S))
        got = g([None if f is None else _place(f, "device", m) for f, m in zip(fs, MIX)], camera_matrix=cams)
        hits += _check(k, got, want, (2, S))
    assert hits > STEPS // 2, hits
    trk = _tracker(_category_checkpoints(tmp_path / "trk", True)[1], cats=("chair", "cup"), hungarian=True)
    sizes = [(480, 640)] * S
    tg = cpb.MultiCategoryTrackGraph(trk, slots=S, frame_hw=(480, 640), camera_matrix=_slot_cameras(sizes),
                                     pixel_format="nv12_full")
    total = 0
    for k, fs in enumerate(_graph_video(sizes, ["nv12_full"] * S, seed=820, idle=False)):
        cams = _moving_cameras(sizes, min(k, 3))         # the network's PnP and every category's tracker see it
        got = tg(_place(np.stack(fs), "pinned", "nv12_full"), camera_matrix=cams[0] if k == 5 else cams)
        if k == 5:
            cams = np.stack([cams[0]] * S)
        want = trk.run_batch(_bgr_of(fs, ["nv12_full"] * S), cams)
        total += _check_step(k, got, want, None, (2, S))
    assert total > 0


def test_per_step_camera_refusals_and_default(cplib):
    det = _det_detector()
    sizes = [(480, 640)] * 2
    cams = _slot_cameras(sizes)
    g = cpb.DetectGraph(det, slots=2, frame_hw=(480, 640), camera_matrix=cams, pixel_format="nv21_full",
                        distortion=PLUMB)
    f = np.stack([encode(b, "nv21_full") for b in synth.synthetic_frames(2, 480, 640, seed=3)])
    with pytest.raises(ValueError, match="DetectGraph was built with distortion=: .* no per-step camera_matrix"):
        g(f, camera_matrix=cams)
    g = cpb.DetectGraph(det, slots=2, frame_hw=(480, 640), camera_matrix=cams, pixel_format="nv21_full")
    _capacity(det, 2)
    meta = g.meta.clone()
    for bad in (np.eye(4), np.stack([cams[0]] * 3), torch.from_numpy(cams).cuda()):
        with pytest.raises(ValueError, match="camera_matrix"):
            g(f, camera_matrix=bad)
    nan = cams.copy()
    nan[1, 0, 0] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        g(f, camera_matrix=nan)
    torch.cuda.synchronize()
    assert torch.equal(g.meta, meta)                       # nothing reached the device
    want = det.run_batch(np.stack(_bgr_of(list(f), ["nv21_full"] * 2)), cams)
    _check(0, g(torch.from_numpy(f).cuda()), want, (2,))
    # a new camera, then calls without one keep it; the same camera as at build time gives the build-time steps
    K2 = _moving_cameras(sizes, 3)
    want2 = det.run_batch(np.stack(_bgr_of(list(f), ["nv21_full"] * 2)), K2)
    _check(1, g(torch.from_numpy(f).cuda(), camera_matrix=K2), want2, (2,))
    _check(2, g(torch.from_numpy(f).cuda()), want2, (2,))
    _check(3, g(torch.from_numpy(f).cuda(), camera_matrix=cams), want, (2,))
    assert torch.equal(g.meta, meta)
