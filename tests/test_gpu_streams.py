"""Independent video streams on the device: the ragged pre-process (cp_preprocess_ragged) against cv2, the numpy
restatement and the per-frame kernels; run_batch on mixed-size lists against run(); the tracker's stream maps
(cp_tracker_*_ex) against the entry points without one; slot schedules with restarts and idle slots against each video
run alone; the array and list forms of run_batch(track=True) against each other and the array form's change of input
size against the tracker driven by hand; and TrackPipeline against the same run_batch sequence."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import affine_from_center_scale
from centerpose_b200.engine import _ptr, _stream
from centerpose_b200.tracker import seed_records
from oracle import make_golden_tracker as mg
from oracle import make_golden_tracker_gt as mgt
from oracle import preprocess_ref
from tests.test_gpu_tracker import _frame_records, _opt_from_gold, _tracking_detector
from tests.util import no_splitk

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
SIZES = [(512, 512), (480, 640), (640, 480), (600, 800), (720, 960), (375, 500)]


def _pack(frames):
    offs = np.cumsum([0] + [f.size for f in frames])[:-1].astype(np.int64)
    buf = torch.from_numpy(np.concatenate([f.reshape(-1) for f in frames])).cuda()
    hw = np.array([f.shape[:2] for f in frames], np.int32)
    return buf, offs, hw


def _rotated_crop(h, w, inp):
    """A forward affine that rotates by 30 degrees about a point off the centre and scales a 0.6-sized crop to inp."""
    import cv2
    M = cv2.getRotationMatrix2D((w * 0.4, h * 0.55), 30.0, inp / (0.6 * max(h, w)))
    M[:, 2] += np.array([inp / 2. - w * 0.4, inp / 2. - h * 0.55])
    return M


def test_ragged_preprocess_matches_every_per_frame_path(cplib):
    import cv2
    opt = cpb.default_opt("dla_34")
    mean, std = np.array(opt.mean, np.float32), np.array(opt.std, np.float32)
    frames = [synth.synthetic_frames(1, h, w, seed=60 + i)[0] for i, (h, w) in enumerate(SIZES)]
    buf, offs, hw = _pack(frames)
    # default affines: each frame's fix_res affine from float32 control points (what cp_preprocess builds)
    got = cpb.preprocess_ragged(buf, offs, hw, 512, 512, opt.mean, opt.std).cpu().numpy()
    for b, f in enumerate(frames):
        one = cpb.preprocess(torch.from_numpy(f[None]).cuda(), 512, 512, opt.mean, opt.std).cpu().numpy()[0]
        assert np.array_equal(got[b], one), SIZES[b]
        assert np.array_equal(got[b], preprocess_ref.pre_process(f, 512, 512, mean, std)[0]), SIZES[b]
    # explicit affines: the reference's own fix_res trans_input (cv2.getAffineTransform), one rotated crop
    trans = []
    for h, w in SIZES:
        trans.append(affine_from_center_scale(np.array([w / 2., h / 2.], np.float32), float(max(h, w)), 512, 512))
    trans[3] = _rotated_crop(*SIZES[3], 512)
    got = cpb.preprocess_ragged(buf, offs, hw, 512, 512, opt.mean, opt.std, trans_input=np.stack(trans)).cpu().numpy()
    for b, f in enumerate(frames):
        one = cpb.preprocess(torch.from_numpy(f[None]).cuda(), 512, 512, opt.mean, opt.std,
                             trans_input=trans[b]).cpu().numpy()[0]
        assert np.array_equal(got[b], one), SIZES[b]
        assert np.array_equal(got[b], preprocess_ref.pre_process(f, 512, 512, mean, std, trans_input=trans[b])[0])
        inp = cv2.warpAffine(f, trans[b], (512, 512), flags=cv2.INTER_LINEAR)
        want = ((inp / 255. - mean.reshape(1, 1, 3)) / std.reshape(1, 1, 3)).astype(np.float32).transpose(2, 0, 1)
        assert np.array_equal(got[b], want), SIZES[b]
    # det.pre_process (cv2, the reference's code path) for the fix_res frames
    det = cpb.ObjectPoseDetector(opt, model=cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt))
    for b, f in enumerate(frames):
        if b == 3:
            continue
        images, meta = det.pre_process(f, 1.0, {})
        assert np.array_equal(meta["trans_input"], trans[b])
        assert np.array_equal(got[b], images[0].numpy()), SIZES[b]


def _cam(h, w):
    return synth.default_camera(w, h)


def test_run_batch_mixed_sizes_matches_run(cplib):
    from tests.test_gpu_detector import _detector
    det, opt = _detector()
    sizes = [(600, 800), (480, 640), (720, 960), (512, 512)]
    frames = [synth.synthetic_frames(1, h, w, seed=80 + i)[0] for i, (h, w) in enumerate(sizes)]
    cams = np.stack([_cam(h, w) for h, w in sizes])
    with no_splitk():
        poses, n_valid = det.run_batch(frames, cams)
        assert poses.shape == (4, opt.K, L.CP_POSE_RECORD)
        for b, f in enumerate(frames):
            ret = det.run(f, meta_inp={"camera_matrix": cams[b]})
            p1, n1 = det._last
            assert int(n1[0]) == int(n_valid[b]) == len(ret["results"]), sizes[b]
            n = int(n1[0])
            assert np.array_equal(p1[0, :n], poses[b, :n]), (sizes[b], np.argwhere(p1[0, :n] != poses[b, :n])[:8])
    assert int(n_valid.sum()) > 0
    # pinned and CUDA frames give the same records as numpy frames
    mixed = [torch.from_numpy(frames[0]).pin_memory(), torch.from_numpy(frames[1]).cuda(), frames[2],
             torch.from_numpy(frames[3])]
    p2, n2 = det.run_batch(mixed, cams)
    p3, n3 = det.run_batch(frames, cams)
    assert np.array_equal(p2, p3) and np.array_equal(n2, n3)


# ---- stream maps: NULL, an explicit identity and the entry points without a map ---------------------------------------
def _abi_replay(cplib, name, mode, pose_host, streams=2):
    if name == "greedy":
        gold = json.load(open(mg.OUT))
        meta, frames = mg.make_sequence()
        seeds = [None] * len(frames)
    else:
        gold = json.load(open(os.path.join(GOLDEN, "tracker_seq_%s.json" % name)))
        meta, frames0 = mg.make_sequence()
        frames, seeds = mgt.scenario_frames(name, frames0), mgt.seed_schedule(name, frames0)
    opt = _opt_from_gold(gold["opt"])
    opt.hungarian = bool(gold["opt"].get("hungarian", False))
    trk = cpb.Tracker(opt, streams=streams)
    T = trk.max_tracks
    metat = cpb.make_meta(streams, np.array([256., 256.], np.float32), 512.0, meta["width"], meta["height"],
                          meta["camera_matrix"]).cuda()
    ids = (ctypes.c_int32 * streams)(*range(streams))
    h = trk._h
    outs = []
    for f, dets in enumerate(frames):
        if seeds[f] is not None:
            rec = torch.from_numpy(seed_records(seeds[f], opt)).cuda()
            S = rec.shape[0]
            rec = rec.unsqueeze(0).repeat(streams, 1, 1).contiguous()
            n = torch.full((streams,), S, dtype=torch.int32, device="cuda")
            if mode == "old":
                rc = cplib.cp_tracker_seed(h, streams, _ptr(rec), _ptr(n), S, _stream())
            else:
                rc = cplib.cp_tracker_seed_ex(h, streams, None if mode == "null" else ids, _ptr(rec), _ptr(n), S, _stream())
            assert rc == 0
            torch.cuda.synchronize()
        poses, nv = _frame_records(dets, meta, pose_host, opt.c)
        poses, nv = poses.repeat(streams, 1, 1).contiguous(), nv.repeat(streams).contiguous()
        tr = torch.empty((streams, T, L.CP_TRACK_RECORD), dtype=torch.float32, device="cuda")
        nt = torch.empty((streams,), dtype=torch.int32, device="cuda")
        args = (_ptr(poses), _ptr(nv), poses.shape[1], _ptr(metat), _ptr(tr), _ptr(nt), _stream())
        if mode == "old":
            rc = cplib.cp_tracker_step(h, streams, *args)
        else:
            rc = cplib.cp_tracker_step_ex(h, streams, None if mode == "null" else ids, *args)
        assert rc == 0
        outs.append((tr.cpu().numpy(), nt.cpu().numpy()))
    tin = torch.from_numpy(np.load(os.path.join(GOLDEN, "track_render_gt.npz"))["gt_256_trans_input"].reshape(1, 6)
                           ).repeat(streams, 1).cuda()
    hm = torch.empty((streams, 1, 256, 256), dtype=torch.float32, device="cuda")
    hp = torch.empty((streams, 8, 256, 256), dtype=torch.float32, device="cuda")
    rargs = (_ptr(metat), _ptr(tin), 256, 256)
    if mode == "old":
        rc = cplib.cp_tracker_render(h, streams, *rargs, _ptr(hm), _ptr(hp), _stream())
    else:
        rc = cplib.cp_tracker_render_ex2(h, streams, None if mode == "null" else ids, *rargs, None, _ptr(hm), _ptr(hp),
                                         _stream())
    assert rc == 0
    outs.append((hm.cpu().numpy(), hp.cpu().numpy()))
    return outs


@pytest.mark.parametrize("name", ("greedy",) + tuple(mgt.SCENARIOS))
def test_stream_map_identity_is_bit_identical(name, cplib, pose_host):
    runs = {mode: _abi_replay(cplib, name, mode, pose_host) for mode in ("old", "null", "identity")}
    assert any(int(o[1].sum()) > 0 for o in runs["old"][:-1])
    for mode in ("null", "identity"):
        for a, b in zip(runs["old"], runs[mode]):
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (name, mode)


def test_unlisted_streams_are_untouched(cplib, pose_host):
    """Stream 1 sits out two steps of a 3-stream tracker stepped through maps; its next step equals a stream that never
    paused, and a permuted map steps the same streams as the identity."""
    gold = json.load(open(mg.OUT))
    opt = _opt_from_gold(gold["opt"])
    meta, frames = mg.make_sequence()
    recs = [_frame_records(d, meta, pose_host, opt.c) for d in frames]
    metat = cpb.make_meta(3, np.array([256., 256.], np.float32), 512.0, meta["width"], meta["height"],
                          meta["camera_matrix"]).cuda()
    ref = cpb.Tracker(opt, streams=1)
    want = [ref.step_records(*recs[f], metat[:1].contiguous()) for f in range(4)]
    want = [(t.cpu().numpy(), n.cpu().numpy()) for t, n in want]
    trk = cpb.Tracker(opt, streams=3)
    # stream 1 sees frames 0, 1 then pauses for two steps and sees frames 2, 3; streams 2 and 0 step every time
    sched = [[0, 1, 2], [2, 1, 0], [2, 0], [0, 2], [1, 0, 2], [2, 0, 1]]
    seen = {0: 0, 1: 0, 2: 0}
    for ids in sched:
        fs = [seen[s] for s in ids]
        poses = torch.cat([recs[f][0] for f in fs])
        nv = torch.cat([recs[f][1] for f in fs])
        tr, n = trk.step_records(poses, nv, metat[:len(ids)].contiguous(), stream_ids=ids)
        tr, n = tr.cpu().numpy(), n.cpu().numpy()
        for k, s in enumerate(ids):
            f = seen[s]
            if f < len(want):
                assert int(n[k]) == int(want[f][1][0]), (ids, s, f)
                assert np.array_equal(tr[k], want[f][0][0]), (ids, s, f)
            seen[s] += 1
    assert seen[1] == 4


# ---- slot schedules through run_batch(list, track=True) ----------------------------------------------------------------
VIDEOS = [((480, 640), 5), ((600, 800), 3), ((512, 512), 7), ((375, 500), 4)]     # (size, length); video 1 is seeded
# per step, per slot: (video, frame) or None.  Video 3 restarts slot 0 after video 0 ends; video 1 pauses for two steps
# in slot 1 (then its slot stays idle once it ends); video 2 pauses for two steps in slot 2.
SCHEDULE = [
    [(0, 0), (1, 0), (2, 0)],
    [(0, 1), (1, 1), (2, 1)],
    [(0, 2), None, (2, 2)],
    [(0, 3), None, (2, 3)],
    [(0, 4), (1, 2), None],
    [(3, 0), None, None],
    [(3, 1), None, (2, 4)],
    [(3, 2), None, (2, 5)],
    [(3, 3), None, (2, 6)],
]


def _videos():
    return [[synth.synthetic_frames(1, h, w, seed=1000 + 10 * v + f)[0] for f in range(n)]
            for v, ((h, w), n) in enumerate(VIDEOS)]


def _seed_dets(det, frame, cam):
    """pre_dets for the seeded video: the tracks of a fresh run() on another frame (dicts with every key init_track
    and the heat-map render read)."""
    det.reset_tracking()
    ret = det.run(frame, meta_inp={"camera_matrix": cam})
    det.reset_tracking()
    assert ret["results"]
    return [dict(d) for d in ret["results"]]


def _alone(det, vids, cams, pre):
    """Each video through run() on a fresh tracking detector: per frame (rows [n,320], n)."""
    out = []
    for v, frames in enumerate(vids):
        det.reset_tracking()
        rows = []
        for f, img in enumerate(frames):
            meta = {"camera_matrix": cams[v]}
            if v == 1 and f == 0:
                meta["pre_dets"] = pre
            det.run(img, meta_inp=meta)
            r, n = det.tracker._host()
            rows.append((r[0, :int(n[0])].copy(), int(n[0])))
        out.append(rows)
    det.reset_tracking()
    return out


def _step_args(step, vids, cams, pre):
    frames = [vids[e[0]][e[1]] if e is not None else None for e in step]
    new_video = [e is not None and e[1] == 0 for e in step]
    pre_dets = [pre if (e is not None and e == (1, 0)) else None for e in step]
    slot_cams = np.stack([cams[e[0]] if e is not None else np.eye(3) for e in step])
    return frames, new_video, pre_dets, slot_cams


def test_slot_schedule_matches_each_video_alone(cplib):
    with no_splitk():
        det, opt = _tracking_detector()
        vids = _videos()
        cams = [_cam(h, w) for (h, w), _ in VIDEOS]
        pre = _seed_dets(det, synth.synthetic_frames(1, 512, 512, seed=5)[0], _cam(512, 512))
        want = _alone(det, vids, cams, pre)
        assert sum(n for rows in want for _, n in rows) > 0
        checked = paused = 0
        for step in SCHEDULE:
            frames, new_video, pre_dets, slot_cams = _step_args(step, vids, cams, pre)
            tracks, nt = det.run_batch(frames, slot_cams, track=True, new_video=new_video, pre_dets=pre_dets)
            assert tracks.shape == (3, L.CP_MAX_K, L.CP_TRACK_RECORD)
            for i, e in enumerate(step):
                if e is None:
                    assert int(nt[i]) == 0 and not tracks[i].any()
                    continue
                rows, n = want[e[0]][e[1]]
                assert int(nt[i]) == n, (step, i)
                # ids, ages and counts exactly; every float bit for bit
                assert np.array_equal(tracks[i, :n, L.T_ID], rows[:, L.T_ID])
                assert np.array_equal(tracks[i, :n, L.T_AGE], rows[:, L.T_AGE])
                assert np.array_equal(tracks[i, :n], rows), (step, i, np.argwhere(tracks[i, :n] != rows)[:8])
                checked += 1
                paused += e in ((1, 2), (2, 4))            # the frames right after a two-step pause
        assert checked == sum(e is not None for s in SCHEDULE for e in s) and paused == 2


@pytest.mark.parametrize("gt", (False, True), ids=("tracks", "ground_truth"))
def test_array_and_list_forms_give_identical_tracks(gt, cplib):
    """The same uniform 512x512 uint8 frames through run_batch(array, track=True) and through run_batch(list,
    track=True) with new_video on the first step: at 512 -> 512 both pre-process affines are exactly the identity, so
    every step's tracks agree bit for bit -- also when pre_dets / frame_ids seed the streams from the ground truth."""
    det, opt = _tracking_detector()
    opt.gt_pre_hm_hmhp_first = gt
    cam = _cam(512, 512)
    S, steps = 3, 4
    vids = [synth.synthetic_frames(steps, 512, 512, seed=120 + v) for v in range(S)]
    _, seq = mg.make_sequence()
    runs = []
    for form in ("array", "list"):
        det.reset_tracking()
        got = []
        for f in range(steps):
            batch = np.stack([vids[v][f] for v in range(S)])
            kw = {"pre_dets": [mgt.gt_list(seq[v]) for v in range(S)], "frame_ids": [f] * S} if gt else {}
            if form == "list":
                batch, kw["new_video"] = list(batch), [f == 0] * S
            got.append(det.run_batch(batch, cam, track=True, **kw))
        runs.append(got)
    assert sum(int(n.sum()) for _, n in runs[0]) > 0
    for f, ((ta, na), (tl, nl)) in enumerate(zip(*runs)):
        assert np.array_equal(na, nl), f
        for v in range(S):
            n = int(na[v])
            assert np.array_equal(ta[v, :n], tl[v, :n]), (f, v, np.argwhere(ta[v, :n] != tl[v, :n])[:8])


@pytest.mark.parametrize("seeded", (False, True))
def test_array_input_of_a_new_size_keeps_the_tracks(seeded, cplib):
    """run_batch(fp32 [B,3,h,w], track=True) whose size changes at the same stream count: the new frame is every
    stream's previous frame and the streams are seeded as at a start, but their tracks are not reset -- the same as
    driving the tracker, the heat-map render and the network by hand."""
    from centerpose_b200.engine import decode_params
    det, opt = _tracking_detector()
    cam = _cam(512, 512)
    pre = _seed_dets(det, synth.synthetic_frames(1, 512, 512, seed=5)[0], cam) if seeded else None
    B = 2
    sizes = [(512, 512), (512, 512), (384, 448), (384, 448)]
    xs = [torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(B, h, w, seed=140 + f))).cuda()
          for f, (h, w) in enumerate(sizes)]
    got = [det.run_batch(x, cam, track=True, pre_dets=[pre] * B if seeded else None) for x in xs]
    trk = cpb.Tracker(opt, streams=B)
    prm = decode_params(opt, test_scale=1.0)
    prev = None
    for f, x in enumerate(xs):
        h, w = x.shape[2:]
        c, s = np.array([w / 2., h / 2.], np.float32), float(max(h, w))
        meta = cpb.make_meta(B, c, s, w, h, cam).cuda()
        if prev is None or prev.shape != x.shape:
            prev = x
            if seeded:
                trk.seed([pre] * B)
        hms = trk.render(meta, affine_from_center_scale(c, s, w, h), h, w, modes=[L.RENDER_TRACKS] * B)
        _, poses, nv = det.model.engine(B, h, w, x.device).infer(x, meta, prm, prev, *hms)
        tr, nt = trk.step_records(poses, nv, meta)
        tr, nt = tr.cpu().numpy(), nt.cpu().numpy()
        prev = x
        assert np.array_equal(nt, got[f][1]), f
        for b in range(B):
            n = int(nt[b])
            assert np.array_equal(tr[b, :n], got[f][0][b, :n]), (f, b)
    assert int(got[2][1].sum()) > 0


def test_track_pipeline_matches_run_batch(cplib):
    det, opt = _tracking_detector()
    vids = _videos()
    cams = [_cam(h, w) for (h, w), _ in VIDEOS]
    pre = _seed_dets(det, synth.synthetic_frames(1, 512, 512, seed=5)[0], _cam(512, 512))
    want = []
    for step in SCHEDULE:
        frames, new_video, pre_dets, slot_cams = _step_args(step, vids, cams, pre)
        want.append(det.run_batch(frames, slot_cams, track=True, new_video=new_video, pre_dets=pre_dets))
    det.reset_tracking()
    pipe = cpb.TrackPipeline(det, slots=3, camera_matrix=np.stack([np.eye(3)] * 3), depth=2)
    got = []
    for k, step in enumerate(SCHEDULE):
        frames, new_video, pre_dets, slot_cams = _step_args(step, vids, cams, pre)
        if k % 2:                                            # pinned frames on odd steps, pageable on even ones
            frames = [torch.from_numpy(f).pin_memory() if f is not None else None for f in frames]
        if pipe.in_flight == pipe.depth:
            got.append(pipe.collect())
        pipe.submit(frames, new_video=new_video, pre_dets=pre_dets, camera_matrix=slot_cams)
    while pipe.in_flight:
        got.append(pipe.collect())
    assert len(got) == len(want)
    for (gt, gn), (wt, wn) in zip(got, want):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt)
