"""Lens distortion on the device.  A distorted camera's network input is, bit for bit, the normalised cv2.remap of its
frame converted to BGR through the map of lens.undistort_map (tests/remap_ref.py, pinned against cv2.remap by
tests/test_undistort_cpu.py), and every result equals that of the same call on those fp32 inputs with the meta camera
K_new:

  * the ops: cp_preprocess_remap in every pixel format and over per-frame formats, with mapped and unmapped frames in
    one table (the unmapped rows are today's affine launch); cp_preprocess_slots_ragged_dev / _rows_dev over a table of
    cp_preprocess_frame_table_maps with their twin and exchange writes; maps with half ties, far-outside and non-finite
    entries;
  * the product paths: both forms of run_batch, detection and track=True with idle slots and new_video, the two
    multi-category run_batch calls, BatchPipeline and TrackPipeline, and the four graph classes at one and at per-slot
    frame sizes, with and without idle slots, mixing distorted and undistorted cameras."""
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import affine_from_center_scale
from centerpose_b200.engine import decode_params, make_meta
from centerpose_b200.lens import undistort_map
from tests import remap_ref
from tests.test_gpu_detect_graph import _capacity, _check, _scattered
from tests.test_gpu_detect_graph import _detector as _det_detector
from tests.test_gpu_pixel_formats import MIX, TRACK_SIZES, _bgr_of, _f32, _graph_video, _p, _same, encode, to_bgr
from tests.test_gpu_track_graph import _detector as _trk_detector
from tests.test_gpu_track_graph_multi import _check_step, _place, _slot_cameras, _tracker
from tests.test_gpu_yuv_input import _cam, _category_checkpoints, _pack

pytestmark = pytest.mark.gpu
OPT = cpb.default_opt("dla_34")
FORMATS = ("bgr", "nv12", "i420", "rgb24", "rgba", "bgra", "yuyv422", "uyvy422")
PLUMB = cpb.LensDistortion([-0.28, 0.07, 1e-3, -5e-4, -0.01])
RATIONAL = cpb.LensDistortion([0.3, -0.1, 1e-3, -5e-4, 0.02, 0.6, -0.05, 0.05], "rational_polynomial")
FISHEYE = cpb.LensDistortion([0.05, -0.01, 0.002, -0.0005], "equidistant")


def _widened(K):
    Kn = np.asarray(K, np.float64).copy()
    Kn[0, 0] *= 0.7
    Kn[1, 1] *= 0.7
    return Kn


def _oracle(frame, fmt, dist, K, ih, iw):
    """The contract's network input of one frame [1,3,ih,iw] (dist None: today's affine pre-process)."""
    bgr = to_bgr(frame, fmt)
    h, w = bgr.shape[:2]
    if dist is None:
        from oracle import preprocess_ref
        A = affine_from_center_scale(np.array([w / 2., h / 2.], np.float32), float(max(h, w)), iw, ih)
        return preprocess_ref.pre_process(bgr, iw, ih, OPT.mean, OPT.std, trans_input=A)
    m = undistort_map(dist, K, (h, w), (ih, iw))
    return remap_ref.pre_process_remap(bgr, m[..., 0], m[..., 1], OPT.mean, OPT.std)


def _maps(dists, cams, sizes, ih, iw):
    return [None if d is None else torch.from_numpy(undistort_map(d, K, hw, (ih, iw))).cuda()
            for d, K, hw in zip(dists, cams, sizes)]


# ---- the ops -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS + ("mixed",))
def test_remap_launches_match_the_contract(fmt, cplib):
    ih, iw = 384, 512
    sizes = [(720, 1280), (480, 640), (1080, 1920), (600, 800), (512, 512)]
    fmts = (["bgr"] + MIX) if fmt == "mixed" else [fmt] * 5
    dists = [PLUMB, None, FISHEYE, RATIONAL, cpb.LensDistortion(PLUMB.coeffs, new_camera_matrix=_widened(_cam(512, 512)))]
    frames = [encode(synth.synthetic_frames(1, h, w, seed=10 + i)[0], f, seed=i) for i, ((h, w), f) in
              enumerate(zip(sizes, fmts))]
    cams = [_cam(h, w) for h, w in sizes]
    packed, offs = _pack(frames, [3, 1, 2, 5, 1])
    hw = np.array(sizes, np.int32)
    trans = np.stack([affine_from_center_scale(np.array([w / 2., h / 2.], np.float32), float(max(h, w)), iw, ih)
                      for h, w in sizes])
    maps = _maps(dists, cams, sizes, ih, iw)
    got = cpb.preprocess_remap(packed, offs, hw, fmts, maps, ih, iw, OPT.mean, OPT.std, trans_input=trans)
    for b in range(5):
        _same(got[b:b + 1], torch.from_numpy(_oracle(frames[b], fmts[b], dists[b], cams[b], ih, iw)), "row %d" % b)
    today = cpb.preprocess_formats(packed, offs, hw, fmts, ih, iw, OPT.mean, OPT.std, trans_input=trans)
    _same(got[1], today[1], "unmapped row")                      # the affine launch's bits
    # the graph-safe launches over a table with maps, launched with the CP_PIX_REMAP code
    NS = 5
    table = torch.zeros(int(cplib.cp_preprocess_frame_table_bytes(NS)), dtype=torch.uint8, device="cuda")
    mixed = len(set(fmts)) > 1
    code = L.CP_PIX_PER_FRAME if mixed else L.PIXEL_FORMAT_CODES[fmt]
    codes = np.array([L.PIXEL_FORMAT_CODES[f] for f in fmts], np.int32)
    ptrs = (ctypes.c_void_p * NS)(*[None if m is None else m.data_ptr() for m in maps])
    L.check(cplib.cp_preprocess_frame_table_maps(
        packed.numel(), offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
        hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), code,
        codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)) if mixed else None, ptrs, NS, ih, iw,
        np.ascontiguousarray(trans).ctypes.data_as(ctypes.POINTER(ctypes.c_double)), _p(table), None), "table")
    code |= L.CP_PIX_REMAP
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    m, s = _f32(OPT.mean), _f32(OPT.std)
    start = torch.tensor([1, 0, 1, 0, 1], dtype=torch.int32, device="cuda")
    out = torch.full((NS, 3, ih, iw), float("nan"), device="cuda")
    prev = torch.full_like(out, 7.0)
    L.check(cplib.cp_preprocess_slots_ragged_dev(_p(packed), _p(table), code, NS, ih, iw, m, s, _p(start), _p(out),
                                                 _p(prev), st), "cp_preprocess_slots_ragged_dev")
    _same(out, got, "slots_ragged")
    for b in range(NS):
        _same(prev[b], got[b] if start[b] else torch.full_like(got[b], 7.0), "twin %d" % b)
    rows = [4, 0, 2, 1]
    rows_d = torch.tensor(rows, dtype=torch.int32, device="cuda")
    old = torch.randn((NS, 3, ih, iw), device="cuda")
    store, prev = old.clone(), torch.full((4, 3, ih, iw), float("nan"), device="cuda")
    out = torch.full((4, 3, ih, iw), float("nan"), device="cuda")
    L.check(cplib.cp_preprocess_slots_rows_dev(_p(packed), _p(table), code, _p(rows_d), 4, ih, iw, m, s, _p(start),
                                               _p(store), _p(out), _p(prev), st), "cp_preprocess_slots_rows_dev")
    _same(out, got[np.array(rows)], "rows")
    for k, slot in enumerate(rows):
        _same(prev[k], got[slot] if start[slot] else old[slot], "rows prev %d" % k)
        _same(store[slot], got[slot], "rows store %d" % slot)
    _same(store[3], old[3], "idle store")


def test_remap_on_hand_made_maps(cplib):
    """Half ties of the 1/32 grid, negative and far-outside positions, NaN, +-inf and values beyond the int range."""
    rng = np.random.default_rng(1)
    frame = synth.synthetic_frames(1, 300, 400, seed=3)[0]
    ih, iw = 128, 160
    mx = (rng.integers(-200, 420 * 32, (ih, iw)) / 32 + rng.choice([0, 1 / 64, -1 / 64], (ih, iw))).astype(np.float32)
    my = (rng.integers(-200, 320 * 32, (ih, iw)) / 32 + rng.choice([0, 1 / 64, -1 / 64], (ih, iw))).astype(np.float32)
    bad = np.array([np.nan, np.inf, -np.inf, 1e10, -1e10, 6.7e7, -6.7e7, 2 ** 26, -2 ** 26, 2 ** 26 - 1], np.float32)
    mx[:10, 0], my[:10, 0] = bad, 100.5
    mx[10:20, 0], my[10:20, 0] = 200.25, bad
    mx[20:30, 0], my[20:30, 0] = bad, bad
    packed, offs = _pack([frame])
    mp = torch.from_numpy(np.stack([mx, my], -1)).cuda()
    got = cpb.preprocess_remap(packed, offs, [frame.shape[:2]], "bgr", [mp], ih, iw, OPT.mean, OPT.std)
    _same(got, torch.from_numpy(remap_ref.pre_process_remap(frame, mx, my, OPT.mean, OPT.std)), "hand-made map")


# ---- run_batch against the same calls on the contract's inputs ---------------------------------------------------------
def _rows(frames, fmts, dists, cams, ih, iw):
    """(x [n,3,ih,iw] CUDA of the contract, meta rows [n,16] with K_new, trans_input [n,2,3]) of run_batch's frames."""
    xs, meta, trans = [], [], []
    for f, fmt, d, K in zip(frames, fmts, dists, cams):
        h, w = to_bgr(f, fmt).shape[:2]
        c, s = np.array([w / 2., h / 2.], np.float32), float(max(h, w))
        xs.append(_oracle(f, fmt, d, K, ih, iw))
        meta.append(make_meta(1, c, s, w, h, K if d is None else d.camera(K)).numpy()[0])
        trans.append(affine_from_center_scale(c, s, iw, ih))
    return torch.from_numpy(np.concatenate(xs)).cuda(), np.stack(meta), np.stack(trans)


def _twin(det):
    """A second detector on det's model and plans, with its own slot state: the reference of the tracking calls."""
    return cpb.ObjectPoseDetector(det.opt, model=det.model)


def test_run_batch_detection_matches_the_contract(cplib):
    det = _det_detector()
    ih, iw = det.opt.input_h, det.opt.input_w
    prm = decode_params(det.opt, test_scale=1.0)
    # the array form: one size, one camera, a lens per frame (one undistorted)
    arr = np.stack([encode(f, "nv12") for f in synth.synthetic_frames(3, 720, 1280, seed=31)])
    K = _cam(720, 1280)
    dists = [PLUMB, None, cpb.LensDistortion(FISHEYE.coeffs, "equidistant", new_camera_matrix=_widened(K))]
    x, meta, _ = _rows(list(arr), ["nv12"] * 3, dists, [K] * 3, ih, iw)
    _, wp, wn = det.model.engine(3, ih, iw, x.device).infer(x, torch.from_numpy(meta).cuda(), prm)
    wp, wn = wp.cpu().numpy(), wn.cpu().numpy()
    assert wn.sum() > 0
    for src in (arr, torch.from_numpy(arr).cuda()):
        gp, gn = det.run_batch(src, K, pixel_format="nv12", distortion=dists)
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    # the list form: mixed sizes, formats and lenses, one LensDistortion for every frame
    sizes = [(480, 640), (600, 800), (720, 1280)]
    lst = [encode(synth.synthetic_frames(1, h, w, seed=40 + i)[0], f) for i, ((h, w), f) in
           enumerate(zip(sizes, MIX))]
    cams = np.stack([_cam(h, w) for h, w in sizes])
    x, meta, _ = _rows(lst, MIX[:3], [RATIONAL] * 3, cams, ih, iw)
    _, wp, wn = det.model.engine(3, ih, iw, x.device).infer(x, torch.from_numpy(meta).cuda(), prm)
    gp, gn = det.run_batch(lst, cams, pixel_format=MIX[:3], distortion=RATIONAL)
    assert wn.sum() > 0 and np.array_equal(gn, wn.cpu().numpy()) and np.array_equal(gp, wp.cpu().numpy())
    # no camera distorted: today's bits
    wp, wn = det.run_batch(lst, cams, pixel_format=MIX[:3])
    gp, gn = det.run_batch(lst, cams, pixel_format=MIX[:3], distortion=[None] * 3)
    assert np.array_equal(gn, wn) and np.array_equal(gp, wp)


# per step: per slot True (a frame), None (idle), "new" (a new video starts in the slot)
SCHEDULE = [["new", "new", "new", None], [True, True, None, "new"], ["new", True, True, True], [True, None, True, True]]
SLOT_LENSES = [PLUMB, None, FISHEYE, RATIONAL]


def _slot_video(fmts, seed):
    bases = [synth.synthetic_frames(1, h, w, seed=seed + i)[0] for i, (h, w) in enumerate(TRACK_SIZES)]
    return [([None if e is None else encode(np.roll(b, (2 * k, 3 * k), axis=(0, 1)), m, seed=k)
              for b, e, m in zip(bases, row, fmts)], [e == "new" for e in row]) for k, row in enumerate(SCHEDULE)]


def _track_reference(det, steps, fmts, cams, dists):
    """run_batch(list, track=True) of a detector sharing det's plans, on the contract's inputs with K_new."""
    ref = _twin(det)
    ih, iw, S = det.opt.input_h, det.opt.input_w, len(cams)
    out = []
    for fs, new in steps:
        live = [i for i in range(S) if fs[i] is not None]
        x, meta, trans = _rows([fs[i] for i in live], [fmts[i] for i in live], [dists[i] for i in live],
                               [cams[i] for i in live], ih, iw)
        o = ref._track_out(None, S)
        out.append(ref._track_step(S, live, x, ref._meta_rows(meta), trans, new, None, None, True, o))
    return out


def test_run_batch_tracking_matches_the_contract(cplib):
    det = _trk_detector()
    cams = _slot_cameras(TRACK_SIZES)
    steps = _slot_video(MIX, seed=300)
    want = _track_reference(det, steps, MIX, cams, SLOT_LENSES)
    got = [det.run_batch(fs, cams, track=True, new_video=new, pixel_format=MIX, distortion=SLOT_LENSES)
           for fs, new in steps]
    assert sum(int(n.sum()) for _, n in want) > 0
    for k, ((gt, gn), (wt, wn)) in enumerate(zip(got, want)):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt), k
    # the array form: every slot steps, one camera
    det.reset_tracking()
    K = _cam(480, 640)
    arrs = [np.stack([np.roll(f, (2 * k, 3 * k), axis=(0, 1)) for f in synth.synthetic_frames(4, 480, 640, seed=9)])
            for k in range(3)]
    want = _track_reference(det, [(list(a), None) for a in arrs], ["bgr"] * 4, [K] * 4, SLOT_LENSES)
    for k, a in enumerate(arrs):
        gt, gn = det.run_batch(a, K, track=True, distortion=SLOT_LENSES)
        assert np.array_equal(gn, want[k][1]) and np.array_equal(gt, want[k][0]), k


def test_multi_category_calls_match_the_contract(tmp_path, cplib):
    for d in ("det", "trk"):
        (tmp_path / d).mkdir()
    opt, paths = _category_checkpoints(tmp_path / "det", False)
    mdet = cpb.MultiCategoryDetector(opt, paths)
    ih, iw = opt.input_h, opt.input_w
    sizes = [(480, 640), (720, 1280)]
    lst = [synth.synthetic_frames(1, h, w, seed=50 + i)[0] for i, (h, w) in enumerate(sizes)]
    cams = np.stack([_cam(h, w) for h, w in sizes])
    x, meta, _ = _rows(lst, ["bgr"] * 2, [FISHEYE, None], cams, ih, iw)
    _, wp, wn = mdet.engine(2, ih, iw).infer(x, torch.from_numpy(meta).cuda(), mdet._prms)
    gp, gn = mdet.run_batch(lst, cams, distortion=[FISHEYE, None])
    assert wn.cpu().numpy().sum() > 0
    assert np.array_equal(gn, wn.cpu().numpy()) and np.array_equal(gp, wp.cpu().numpy())
    arr = np.stack([synth.synthetic_frames(1, 480, 640, seed=60 + i)[0] for i in range(2)])
    x, meta, _ = _rows(list(arr), ["bgr"] * 2, [PLUMB] * 2, [cams[0]] * 2, ih, iw)
    _, wp, wn = mdet.engine(2, ih, iw).infer(x, torch.from_numpy(meta).cuda(), mdet._prms)
    gp, gn = mdet.run_batch(arr, cams[0], distortion=PLUMB)
    assert np.array_equal(gn, wn.cpu().numpy()) and np.array_equal(gp, wp.cpu().numpy())
    # the tracker: slots with idle steps and new videos, against its own step on the contract's inputs
    trk = _tracker(_category_checkpoints(tmp_path / "trk", True)[1], cats=("chair", "cup"))
    cams = _slot_cameras(TRACK_SIZES)
    steps = _slot_video(MIX, seed=500)
    got = [trk.run_batch(fs, cams, new_video=new, pixel_format=MIX, distortion=SLOT_LENSES) for fs, new in steps]
    trk.reset_tracking()
    want = []
    for fs, new in steps:
        live = [i for i in range(4) if fs[i] is not None]
        x, meta, trans = _rows([fs[i] for i in live], [MIX[i] for i in live], [SLOT_LENSES[i] for i in live],
                               [cams[i] for i in live], ih, iw)
        want.append(trk._track_step(4, live, x, trk._meta_rows(meta), trans, new, None, None, True,
                                    trk._track_out(None, 4)))
    assert sum(int(n.sum()) for _, n in want) > 0
    for k, ((gt, gn), (wt, wn)) in enumerate(zip(got, want)):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt), k


def test_pipelines_match_run_batch(cplib):
    det = _det_detector()
    K = _cam(480, 640)
    batches = [np.stack(list(synth.synthetic_frames(2, 480, 640, seed=600 + k))) for k in range(3)]
    want = [det.run_batch(b, K, distortion=[PLUMB, FISHEYE]) for b in batches]
    pipe = cpb.BatchPipeline(det, batch=2, height=480, width=640, camera_matrix=K, distortion=[PLUMB, FISHEYE])
    got = []
    for k, b in enumerate(batches):
        if pipe.in_flight == pipe.depth:
            got.append([a.copy() for a in pipe.collect()])
        pipe.submit(torch.from_numpy(b).pin_memory() if k % 2 else b)
    while pipe.in_flight:
        got.append([a.copy() for a in pipe.collect()])
    assert sum(int(n.sum()) for _, n in want) > 0
    for (gp, gn), (wp, wn) in zip(got, want):
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    # TrackPipeline, with a camera changed mid-video: its map is rebuilt
    trk = _trk_detector()
    cams = _slot_cameras(TRACK_SIZES)
    cams2 = cams.copy()
    cams2[2, 0, 0] *= 1.05
    steps = _slot_video(["bgr"] * 4, seed=700)
    want = [trk.run_batch(fs, cams if k < 2 else cams2, track=True, new_video=new, distortion=SLOT_LENSES)
            for k, (fs, new) in enumerate(steps)]
    trk.reset_tracking()
    pipe = cpb.TrackPipeline(trk, slots=4, camera_matrix=cams, distortion=SLOT_LENSES)
    got = []
    for k, (fs, new) in enumerate(steps):
        if pipe.in_flight == pipe.depth:
            got.append(pipe.collect())
        pipe.submit(fs, new_video=new, camera_matrix=cams2 if k == 2 else None)
    while pipe.in_flight:
        got.append(pipe.collect())
    assert sum(int(n.sum()) for _, n in want) > 0
    for (gt, gn), (wt, wn) in zip(got, want):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt)


# ---- the graphs: every step is run_batch(..., distortion=) of the same frames --------------------------------------------
GRAPH_CASES = [  # one frame_hw or one per slot, idle slots
    ("one", False), ("one", True), ("per-slot", False), ("per-slot", True)]


@pytest.mark.parametrize("kind, idle", GRAPH_CASES, ids=["one", "one idle", "per-slot", "per-slot idle"])
def test_detect_graph_matches_run_batch(kind, idle, cplib):
    det = _det_detector()
    S = 4
    sizes = [(480, 640)] * S if kind == "one" else TRACK_SIZES
    fmts = ["bgr"] * S if kind == "one" else MIX
    pf = fmts[0] if kind == "one" else fmts
    cams = _slot_cameras(sizes)
    g = cpb.DetectGraph(det, slots=S, frame_hw=sizes[0] if kind == "one" else sizes, camera_matrix=cams,
                        pixel_format=pf, idle_slots=idle, distortion=SLOT_LENSES)
    assert g._fmt & L.CP_PIX_REMAP
    _capacity(det, S)
    hits = 0
    for k, fs in enumerate(_graph_video(sizes, fmts, seed=320, idle=idle)):
        if idle:
            live = [i for i in range(S) if fs[i] is not None]
            got = g([None if f is None else _place(f, "device") for f in fs])
            want = _scattered(lambda fr, c: det.run_batch(fr, c, pixel_format=[fmts[i] for i in live] if kind !=
                                                          "one" else pf, distortion=[SLOT_LENSES[i] for i in live]),
                              fs, cams, (S,))
        elif kind == "one":
            got = g(_place(np.stack(fs), "pinned"))
            want = det.run_batch(np.stack(fs), cams, pixel_format=pf, distortion=SLOT_LENSES)
        else:
            got = g([_place(f, "pinned") for f in fs])
            want = det.run_batch(fs, cams, pixel_format=pf, distortion=SLOT_LENSES)
        hits += _check(k, got, want, (S,))
    assert hits > 0, hits


@pytest.mark.parametrize("kind, idle", GRAPH_CASES, ids=["one", "one idle", "per-slot", "per-slot idle"])
def test_track_graph_matches_run_batch(kind, idle, cplib):
    det = _trk_detector()
    S = 4
    sizes = [(480, 640)] * S if kind == "one" else TRACK_SIZES
    fmts = ["bgr"] * S if kind == "one" else MIX
    pf = fmts[0] if kind == "one" else fmts
    cams = _slot_cameras(sizes)
    tg = cpb.TrackGraph(det, slots=S, frame_hw=sizes[0] if kind == "one" else sizes, camera_matrix=cams,
                        pixel_format=pf, idle_slots=idle, distortion=SLOT_LENSES)
    total = 0
    for k, fs in enumerate(_graph_video(sizes, fmts, seed=800, idle=idle)):
        new = [True, False, False, True] if k == 4 else None
        if kind == "one" and not idle:
            got = tg(_place(np.stack(fs), "pinned"), new_video=new)
        else:
            got = tg([None if f is None else _place(f, "device" if k % 2 else "pinned") for f in fs], new_video=new)
        want = det.run_batch(fs, cams, track=True, new_video=new, pixel_format=pf, distortion=SLOT_LENSES)
        total += _check_step(k, got, want, None, (S,))
    assert total > 0


def test_multi_category_graphs_match_run_batch(tmp_path, cplib):
    for d in ("det", "trk"):
        (tmp_path / d).mkdir()
    opt, paths = _category_checkpoints(tmp_path / "det", False)
    mdet = cpb.MultiCategoryDetector(opt, paths)
    S, cams = 4, _slot_cameras(TRACK_SIZES)
    g = cpb.MultiCategoryDetectGraph(mdet, slots=S, frame_hw=TRACK_SIZES, camera_matrix=cams, pixel_format=MIX,
                                     idle_slots=True, distortion=SLOT_LENSES)
    _capacity(mdet, S)
    hits = 0
    for k, fs in enumerate(_graph_video(TRACK_SIZES, MIX, seed=380, idle=True)):
        live = [i for i in range(S) if fs[i] is not None]
        want = _scattered(lambda fr, c: mdet.run_batch(fr, c, pixel_format=[MIX[i] for i in live],
                                                       distortion=[SLOT_LENSES[i] for i in live]), fs, cams, (2, S))
        hits += _check(k, g([None if f is None else _place(f, "device") for f in fs]), want, (2, S))
    assert hits > 0, hits
    trk = _tracker(_category_checkpoints(tmp_path / "trk", True)[1], cats=("chair", "cup"))
    one = _slot_cameras([(480, 640)] * S)
    tg = cpb.MultiCategoryTrackGraph(trk, slots=S, frame_hw=(480, 640), camera_matrix=one, pixel_format="uyvy422",
                                     distortion=FISHEYE)
    total = 0
    for k, fs in enumerate(_graph_video([(480, 640)] * S, ["uyvy422"] * S, seed=820, idle=False)):
        got = tg(_place(np.stack(fs), "pinned"))
        want = trk.run_batch(np.stack(fs), one, pixel_format="uyvy422", distortion=FISHEYE)
        total += _check_step(k, got, want, None, (2, S))
    assert total > 0
