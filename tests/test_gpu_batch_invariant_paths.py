"""Batch-invariant detectors (opt.batch_invariant) through the product paths, with split-K left on, on seeded and
calibrated networks:

  * detection: run() of each frame against the matching rows of run_batch(array), run_batch(list) of mixed frame
    sizes, BatchPipeline, DetectGraph (3 slots) and DetectGraph(idle_slots=True) over a late start, a pause, an end and
    an all-idle step, and MultiCategoryDetector.run_batch against its frames one at a time;
  * tracking: a slot's tracks over a 10-step sequence run alone (S = 1) against the same slot among S = 4 whose other
    slots idle and start on a seeded pattern, through run_batch(list, track=True) and TrackGraph(idle_slots=True).

Without the flag none of these hold bit for bit: the default plan's split-K follows the batch (tests/util.py
no_splitk)."""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from tests.test_gpu_track_graph import H, W, _host
from tests.test_gpu_track_graph_multi import _place, _ragged_video, _slot_cameras

pytestmark = pytest.mark.gpu
STEPS = 10


def _calibrated_model(trk, seed):
    opt = cpb.default_opt("dla_34", tracking_task=trk, batch_invariant=True)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    assert m.batch_invariant
    m.load_state_dict(synth.seeded_state_dict(m, seed=seed, offset_std=0.3))
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, 512, 512, seed=5))).cuda()
    with torch.no_grad():
        if trk:
            z = torch.zeros((2, 1, 512, 512), device="cuda")
            synth.calibrate_head_bias(m, m(x, x, z, z.repeat(1, 8, 1, 1))[-1], target=4)
        else:
            synth.calibrate_head_bias(m, m(x)[-1], target=8)
    return opt, m


@pytest.fixture(scope="module")
def detector():
    opt, m = _calibrated_model(False, seed=41)
    return cpb.ObjectPoseDetector(opt, model=m)


def _run_rows(det, frames, cams):
    """run() of each frame alone: its (poses [K, R], n_valid) as run_batch reports them."""
    out = []
    for f, c in zip(frames, cams):
        ret = det.run(np.ascontiguousarray(f), meta_inp={"camera_matrix": c})
        p, n = det._last
        p, n = np.asarray(p)[0].copy(), int(np.asarray(n)[0])
        assert n == len(ret["results"])
        out.append((p, n))
    return out


def _same(rows, poses, n_valid, what, slots=None):
    slots = range(len(rows)) if slots is None else slots
    hits = 0
    for (p, n), s in zip(rows, slots):
        assert int(n_valid[s]) == n, (what, s, int(n_valid[s]), n)
        assert np.array_equal(poses[s, :n], p[:n]), (what, s, np.argwhere(poses[s, :n] != p[:n])[:8])
        hits += n
    return hits


def test_run_batch_array_and_list_and_pipeline_match_run(detector):
    det = detector
    cam = synth.default_camera(W, H)
    frames = synth.synthetic_frames(6, H, W, seed=9)
    rows = _run_rows(det, frames, [cam] * 6)
    hits = 0
    for a, b in ((0, 6), (1, 4), (5, 6)):
        p, n = det.run_batch(frames[a:b], cam)
        hits += _same(rows[a:b], p, n, "run_batch(array) rows %d..%d" % (a, b))
    assert hits > 0
    # a list of mixed frame sizes, each with its camera
    sizes = [(600, 800), (480, 640), (720, 960), (512, 512)]
    mixed = [synth.synthetic_frames(1, h, w, seed=80 + i)[0] for i, (h, w) in enumerate(sizes)]
    cams = np.stack([synth.default_camera(w, h) for h, w in sizes])
    mrows = _run_rows(det, mixed, cams)
    p, n = det.run_batch(mixed, cams)
    assert _same(mrows, p, n, "run_batch(list)") > 0
    p, n = det.run_batch(mixed[1:3], cams[1:3])
    _same(mrows[1:3], p, n, "run_batch(list) of two")
    # BatchPipeline of 2-frame batches
    pipe = cpb.BatchPipeline(det, 2, H, W, cam, depth=2)
    got = []
    for i in range(3):
        if pipe.in_flight == pipe.depth:
            pp, nn = pipe.collect()
            got.append((pp.copy(), nn.copy()))
        pipe.submit(torch.from_numpy(frames[2 * i:2 * i + 2]).pin_memory())
    while pipe.in_flight:
        pp, nn = pipe.collect()
        got.append((pp.copy(), nn.copy()))
    for i, (pp, nn) in enumerate(got[:3]):
        _same(rows[2 * i:2 * i + 2], pp, nn, "BatchPipeline batch %d" % i)


LIVE = [{0, 2}, {0, 1, 2}, {1, 2}, {2}, set(), {0, 1}, {0, 1, 2}, {1}, {0, 1}, {0, 2}]


@pytest.mark.parametrize("idle", [False, True])
def test_detect_graph_matches_run(detector, idle):
    det = detector
    S = 3
    cams = np.stack([synth.default_camera(W + 16 * i, H + 8 * i) for i in range(S)])
    g = cpb.DetectGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cams, idle_slots=idle)
    video = [synth.synthetic_frames(S, H, W, seed=500 + k) for k in range(STEPS)]
    hits = 0
    for k, fs in enumerate(video):
        live = sorted(LIVE[k]) if idle else list(range(S))
        arg = [torch.from_numpy(fs[i]).pin_memory() if i in live else None for i in range(S)] if idle else \
            torch.from_numpy(fs).pin_memory()
        p, n = _host(g(arg))
        rows = _run_rows(det, [fs[i] for i in live], [cams[i] for i in live])
        hits += _same(rows, p, n, "DetectGraph step %d" % k, slots=live)
        for i in set(range(S)) - set(live):
            assert n[i] == 0 and not p[i].any()
    assert hits > 0


def test_multi_category_rows_match_single_frames(tmp_path):
    paths = {}
    for c, s in (("chair", 51), ("cup", 52)):
        opt, m = _calibrated_model(False, seed=s)
        paths[c] = str(tmp_path / (c + ".pth"))
        cpb.save_model(paths[c], 1, m)
    mdet = cpb.MultiCategoryDetector(cpb.default_opt("dla_34", batch_invariant=True), paths)
    cam = synth.default_camera(W, H)
    frames = synth.synthetic_frames(5, H, W, seed=21)
    p, n = mdet.run_batch(frames, cam)
    hits = 0
    for b in range(5):
        p1, n1 = mdet.run_batch(frames[b:b + 1], cam)
        for c in range(2):
            assert int(n[c, b]) == int(n1[c, 0])
            assert np.array_equal(p[c, b], p1[c, 0]), (c, b)
            hits += int(n1[c, 0])
    assert hits > 0


# ---- tracking: slot 0 alone and among four ------------------------------------------------------------------------
S4 = 4
OTHERS = [  # per step, the live slots besides slot 0 (always live): slot 1 starts late, 2 pauses, 3 ends
    {2, 3}, {3}, {1, 2, 3}, {1}, set(), {1, 2}, {1, 2}, {2}, {1}, {1, 2},
]


def test_a_slots_tracks_do_not_depend_on_the_other_slots():
    opt, m = _calibrated_model(True, seed=31)
    sizes = [(H, W), (720, 1280), (H, W), (512, 384)]
    cams = _slot_cameras(sizes)
    video = _ragged_video(sizes, "bgr", seed=900, steps=STEPS)
    alone = cpb.ObjectPoseDetector(opt, model=m)
    shared = cpb.ObjectPoseDetector(opt, model=m)
    graph_det = cpb.ObjectPoseDetector(opt, model=m)
    tg = cpb.TrackGraph(graph_det, slots=S4, frame_hw=sizes, camera_matrix=cams, idle_slots=True)
    total = 0
    for k, fs in enumerate(video):
        steps = [fs[i] if (i == 0 or i in OTHERS[k]) else None for i in range(S4)]
        wt, wn = alone.run_batch([fs[0]], cams[:1], track=True)
        st, sn = shared.run_batch(steps, cams, track=True)
        gt, gn = _host(tg([None if f is None else _place(f, "pinned") for f in steps]))
        n = int(wn[0])
        for what, t, nn in (("run_batch(list, track=True), S = 4", st, sn), ("TrackGraph(idle_slots), S = 4", gt, gn)):
            assert int(nn[0]) == n, (what, k, int(nn[0]), n)
            assert np.array_equal(t[0, :n], wt[0, :n]), (what, k, np.argwhere(t[0, :n] != wt[0, :n])[:8])
        assert wt.shape[-1] == L.CP_TRACK_RECORD
        total += n
    assert total > 0
