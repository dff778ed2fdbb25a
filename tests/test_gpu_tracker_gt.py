"""Ground-truth seeding, ground-truth / empty previous-frame heat maps and the hungarian association on the device:
cp_tracker_seed + cp_tracker_step vs the unmodified reference (tests/golden/tracker_seq_{gt_first,gt_every,hungarian}.json),
cp_tracker_render_ex vs its ground-truth branch (tests/golden/track_render_gt.npz), the solver vs the restatement on
random scenes, and the ground-truth flow of run() / run_batch(track=True)."""
import copy
import ctypes
import json
import os
import types

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from oracle import make_golden_tracker as mg
from oracle import make_golden_tracker_gt as mgt
from oracle import tracker_ref
from tests.test_gpu_tracker import _frame_records, _opt_from_gold
from tests.test_track_core_host import compare_to_golden, summarize_tracks

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _meta(streams, meta):
    return cpb.make_meta(streams, np.array([256., 256.], np.float32), 512.0, meta["width"], meta["height"],
                         meta["camera_matrix"]).cuda()


def _device_replay(name, pose_host, streams=1, stream=0):
    gold = json.load(open(os.path.join(GOLDEN, "tracker_seq_%s.json" % name)))
    opt = _opt_from_gold(gold["opt"])
    opt.hungarian = bool(gold["opt"]["hungarian"])
    meta, frames0 = mg.make_sequence()
    frames = mgt.scenario_frames(name, frames0)
    seeds = mgt.seed_schedule(name, frames0)
    trk = cpb.Tracker(opt, streams=streams)
    metat = _meta(streams, meta)
    got = []
    for f, dets in enumerate(frames):
        if seeds[f] is not None:
            trk.seed([seeds[f] if b == stream else None for b in range(streams)])
        poses, nv = _frame_records(dets, meta, pose_host, opt.c)
        tr, n = trk.step_records(poses.repeat(streams, 1, 1), nv.repeat(streams), metat)
        got.append(summarize_tracks(tr[stream].cpu().numpy(), int(n[stream])))
    return got, gold["frames"], trk


@pytest.mark.parametrize("name", mgt.SCENARIOS)
def test_device_matches_reference_golden(name, cplib, pose_host):
    got, want, _ = _device_replay(name, pose_host)
    compare_to_golden(got, want)


def test_reseeding_one_stream_leaves_the_other_bit_exact(cplib, pose_host):
    gold = json.load(open(os.path.join(GOLDEN, "tracker_seq_gt_first.json")))
    opt = _opt_from_gold(gold["opt"])
    meta, frames = mg.make_sequence()
    metat = _meta(2, meta)
    recs = [_frame_records(d, meta, pose_host, opt.c) for d in frames[:3]]
    outs = []
    for reseed in (False, True):
        trk = cpb.Tracker(opt, streams=2)
        trk.seed([mgt.gt_list(frames[0])] * 2)
        for f in range(3):
            if reseed and f == 2:
                trk.seed([None, mgt.gt_list(frames[1])])
            tr, n = trk.step_records(recs[f][0].repeat(2, 1, 1), recs[f][1].repeat(2), metat)
        outs.append((tr.cpu().numpy(), n.cpu().numpy()))
    assert np.array_equal(outs[0][0][0], outs[1][0][0]) and outs[0][1][0] == outs[1][1][0]
    assert not np.array_equal(outs[0][0][1], outs[1][0][1])


def test_seed_rejects_more_seeds_than_max_tracks(cplib):
    opt = cpb.default_opt("dla_34", tracking_task=True)
    trk = cpb.Tracker(opt, streams=1, max_tracks=4)
    n = torch.tensor([5], dtype=torch.int32, device="cuda")
    seeds = torch.zeros((1, 5, L.CP_SEED_RECORD), dtype=torch.float32, device="cuda")
    rc = cplib.cp_tracker_seed(trk._h, 1, ctypes.c_void_p(seeds.data_ptr()), ctypes.c_void_p(n.data_ptr()), 5, None)
    assert rc == -1 and b"exceed max_tracks" in cplib.cp_last_error()


@pytest.mark.parametrize("case", mgt.GT_RENDER_CASES)
def test_ground_truth_render_matches_reference(case, cplib):
    name, ih, iw = case
    z = np.load(os.path.join(GOLDEN, "track_render_gt.npz"))
    opt = cpb.default_opt("dla_34", tracking_task=True)
    meta, frames = mg.make_sequence()
    trk = cpb.Tracker(opt, streams=1)
    trk.init_track(dict(meta, id=0, pre_dets=mgt.gt_list(frames[0])))
    metat = _meta(1, meta)
    hm, hm_hp = trk.render(metat, z[name + "_trans_input"], ih, iw, modes=[L.RENDER_GT])
    torch.cuda.synchronize()
    for key, got in (("_hm", hm[0].cpu().numpy()), ("_hm_hp", hm_hp[0].cpu().numpy())):
        if name + key in z.files:
            want = z[name + key]
            assert ((got != 0) == (want != 0)).all(), "%s%s: support differs" % (name, key)
            assert np.abs(got - want).max() <= 2e-6
        else:
            sub, ssum, nnz = z[name + key + "_sub4"], z[name + key + "_sum"], z[name + key + "_nnz"]
            assert np.abs(got[:, ::4, ::4] - sub).max() <= 2e-6
            assert ((got != 0).sum(axis=(1, 2)) == nnz).all()
            assert np.allclose(got.astype(np.float64).sum(axis=(1, 2)), ssum, rtol=1e-5, atol=1e-4)
    # mode 2: exact zeros
    hm2, hp2 = trk.render(metat, z[name + "_trans_input"], ih, iw, modes=[L.RENDER_EMPTY])
    assert not hm2.any() and not hp2.any()


def test_render_modes_on_tracks_are_bit_identical(cplib, pose_host):
    gold = json.load(open(mg.OUT))
    opt = _opt_from_gold(gold["opt"])
    meta, frames = mg.make_sequence()
    trk = cpb.Tracker(opt, streams=1)
    metat = _meta(1, meta)
    for dets in frames[:4]:
        trk.step_records(*_frame_records(dets, meta, pose_host, opt.c), metat)
    tr = np.load(os.path.join(GOLDEN, "track_render_gt.npz"))["gt_256_trans_input"]
    a = [t.clone() for t in trk.render(metat, tr, 256, 256)]
    b = trk.render(metat, tr, 256, 256, modes=[L.RENDER_TRACKS])
    assert a[0].any() and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def _scene(rng, M, N):
    def det(c, half, score):
        return {"score": score, "cls": 0, "ct": [float(c[0]), float(c[1])], "tracking": np.zeros(2),
                "bbox": [float(c[0] - half), float(c[1] - half), float(c[0] + half), float(c[1] + half)]}
    tr = [det(rng.integers(0, 64, 2) * 8.0, float(rng.integers(4, 24)), 0.9) for _ in range(M)]
    ds = []
    for _ in range(N):
        if tr and rng.random() < 0.7:
            base = tr[rng.integers(0, M)]
            c = np.array(base["ct"]) + rng.integers(-3, 4, 2) * 4.0        # integer offsets: many equal costs
        else:
            c = rng.integers(0, 64, 2) * 8.0
        ds.append(det(c, float(rng.integers(4, 24)), float(rng.uniform(0.35, 0.95))))
    return tr, ds


def _records(dets, K):
    r = np.zeros((K, L.CP_POSE_RECORD), np.float32)
    for i, d in enumerate(dets):
        r[i, L.P_SCORE], r[i, L.P_CLS] = d["score"], d["cls"]
        r[i, L.P_BBOX:L.P_BBOX + 4], r[i, L.P_CT:L.P_CT + 2] = d["bbox"], d["ct"]
    return r


def test_hungarian_random_scenes_match_restatement(cplib):
    rng = np.random.default_rng(5)
    opt = types.SimpleNamespace(kalman=False, scale_pool=False, use_pnp=False, hungarian=True, new_thresh=0.3, max_age=5,
                                R=20, c="chair", conf_border={"chair": [3, 9]}, show_axes=False, hps_uncertainty=True)
    B, K = 8, 128
    differs = 0
    for rnd in range(3):
        # up to 128 tracks or detections per stream, at most max_tracks = 128 entries after the step
        sizes = [(m, int(rng.integers(1, max(2, 129 - m)))) for m in rng.integers(1, 128, B)]
        scenes = [_scene(rng, int(m), n) for m, n in sizes]
        trk = cpb.Tracker(opt, streams=B)
        metat = cpb.make_meta(B, np.array([256., 256.], np.float32), 512.0, 512, 512, np.eye(3)).cuda()
        want = []
        for f in range(2):
            recs = np.stack([_records(s[f], K) for s in scenes])
            nv = torch.tensor([len(s[f]) for s in scenes], dtype=torch.int32, device="cuda")
            tr, n = trk.step_records(torch.from_numpy(recs).cuda(), nv, metat)
        tr, n = tr.cpu().numpy(), n.cpu().numpy()
        for b, (t0, d1) in enumerate(scenes):
            ids = {}
            for hung in (True, False):
                o = types.SimpleNamespace(**vars(opt))
                o.hungarian = hung
                ref = tracker_ref.TrackerRef(o)
                ref.init_track({})
                ref.step(copy.deepcopy(t0))
                ret, _ = ref.step(copy.deepcopy(d1))
                ids[hung] = [int(t["tracking_id"]) for t in ret]
            assert [int(v) for v in tr[b, :int(n[b]), L.T_ID]] == ids[True], (rnd, b)
            differs += ids[True] != ids[False]
    assert differs > 0


def _gt_detector():
    from tests.test_gpu_tracker import _tracking_detector
    det, opt = _tracking_detector()
    opt.gt_pre_hm_hmhp_first = True
    return det, opt


def test_run_ground_truth_first_frame(cplib):
    det, opt = _gt_detector()
    cam = synth.default_camera(512, 512)
    frames = synth.synthetic_frames(3, 512, 512, seed=77)
    _, seq = mg.make_sequence()
    seen = {}
    orig = det.process

    def spy(images, pre_images=None, pre_hms=None, pre_hm_hp=None, *a, **k):
        seen["in"] = (pre_hms.clone(), pre_hm_hp.clone())
        return orig(images, pre_images, pre_hms, pre_hm_hp, *a, **k)
    det.process = spy
    ids = []
    for f in range(3):
        ret = det.run(frames[f], meta_inp={"camera_matrix": cam, "id": f, "pre_dets": mgt.gt_list(seq[0])})
        assert {"results", "boxes", "output", "tot", "load", "pre", "net", "dec", "post", "merge", "pnp", "track"} == set(ret)
        ids.append({d["tracking_id"] for d in ret["results"]})
        if f == 0:
            ref = cpb.Tracker(opt, streams=1)
            _, meta = det.pre_process(frames[0], 1.0, {"camera_matrix": cam})
            ref.init_track(dict(meta, pre_dets=mgt.gt_list(seq[0])))
            want = ref.render(det._meta_tensor(meta).cuda(), meta["trans_input"], 512, 512, modes=[L.RENDER_GT])
            assert torch.equal(seen["in"][0], want[0]) and torch.equal(seen["in"][1], want[1])
    assert {1, 2, 3, 4, 5} & ids[1] and {1, 2, 3, 4, 5} & ids[2]          # the seeded ids carry on


def test_run_batch_ground_truth_matches_run(cplib):
    from tests.util import no_splitk
    with no_splitk():
        det, opt = _gt_detector()
        cam = synth.default_camera(512, 512)
        vids = [synth.synthetic_frames(3, 512, 512, seed=100 + v) for v in range(2)]
        _, seq = mg.make_sequence()
        pre = [mgt.gt_list(seq[0]), mgt.gt_list(seq[1])]
        per_stream = []
        for v in range(2):
            det.reset_tracking()
            rows = []
            for f in range(3):
                ret = det.run(vids[v][f], meta_inp={"camera_matrix": cam, "id": f, "pre_dets": pre[v]})
                rows.append([(d["tracking_id"], d["score"]) for d in ret["results"]])
            per_stream.append(rows)
        det.reset_tracking()
        for f in range(3):
            tracks, nt = det.run_batch(np.stack([vids[0][f], vids[1][f]]), cam, track=True, pre_dets=pre, frame_ids=[f, f])
            for v in range(2):
                want = per_stream[v][f]
                assert int(nt[v]) == len(want)
                for i, (tid, score) in enumerate(want):
                    assert int(tracks[v, i, L.T_ID]) == tid
                    assert abs(float(tracks[v, i, L.P_SCORE]) - score) <= 1e-5
