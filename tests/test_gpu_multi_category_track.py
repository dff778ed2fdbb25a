"""Multi-category tracking on the GPU, M = 3 tracking checkpoints from different seeds:

  * each model's slice of a cp_plan_create_multi_track plan, given its own previous-frame heat maps (random and different
    per model, so reading another model's maps changes the result), against that checkpoint's own tracking plan, bit for
    bit with a fixed K partition (CP_NO_SPLITK=1), through cp_forward and cp_plan_run_ops;
  * with split-K on, every op of every model against fp64 under LAYER_CEIL;
  * one cp_tracker_create_multi tracker against one tracker per category, and the data's sensitivity to the
    per-category settings;
  * MultiCategoryTracker.run_batch against each category's ObjectPoseDetector.run_batch(track=True).
"""
import json
import os

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.engine import Engine
from oracle import make_golden_tracker as mg
from oracle import make_golden_tracker_gt as mgt
from tests import layer_ref
from tests.plan_steps import _ceiling, _fetch
from tests.test_gpu_tracker import _frame_records, _opt_from_gold
from tests.util import LAYER_CEIL, no_splitk

pytestmark = pytest.mark.gpu

M = 3
SEEDS = (21, 22, 23)
CATS = ("chair", "cup", "laptop")                       # visible_thresh 6 / 3 / 0
BORDERS = {"chair": [3, 9], "cup": [2, 8], "laptop": [4, 10]}


def _track_engines(arch, H, W, B, prec):
    """(multi-track engine, [single tracking engines]) over the seeded state dicts of SEEDS."""
    opt = cpb.default_opt(arch, tracking_task=True)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    kw = dict(tracking=True, tracking_task_gru=m.use_convGRU and m.tracking_task, precision=prec)
    multi = Engine(m._arch(), m.heads, m.head_conv, B, H, W, 0, models=M, **kw)
    singles = [Engine(m._arch(), m.heads, m.head_conv, B, H, W, 0, **kw) for _ in range(M)]
    for i, s in enumerate(SEEDS):
        sd = synth.seeded_state_dict(m, seed=s, offset_std=0.3)
        multi.load_state_dict(sd, model=i)
        singles[i].load_state_dict(sd)
    return multi, singles


def _track_inputs(H, W, B, seed=317):
    """Shared frames and previous frames [B,3,H,W]; per-model heat maps [M,B,1|8,H,W], different for every model."""
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(B, H, W, seed=seed))).cuda()
    pre_img = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(B, H, W, seed=seed + 1))).cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    pre_hm = torch.rand((M, B, 1, H, W), device="cuda", generator=g)
    pre_hm_hp = torch.rand((M, B, 8, H, W), device="cuda", generator=g)
    return x, pre_img, pre_hm, pre_hm_hp


# (label, arch, H, W, batch, precisions)
GEOMETRIES = [
    ("512 b2", "dla_34", 512, 512, 2, ("fp32", "tf32x3", "tf32", "bf16")),
    ("keep_res 832x608", "dla_34", 832, 608, 1, ("tf32x3",)),
    ("dlav1 gru 128x160", "dlav1_34", 128, 160, 2, ("fp32", "tf32x3")),
]
CASES = [(g[0], g[1], g[2], g[3], g[4], p) for g in GEOMETRIES for p in g[5]]


@pytest.mark.parametrize("case", CASES, ids=["%s %s" % (c[0], c[5]) for c in CASES])
def test_track_slice_bit_equal(case):
    label, arch, H, W, B, prec = case
    with no_splitk():
        multi, singles = _track_engines(arch, H, W, B, prec)
        x, pre_img, pre_hm, pre_hm_hp = _track_inputs(H, W, B)
        n_ops = len(multi.op_descs())
        heads = {n: torch.full((M, B, c, H // 4, W // 4), float("nan"), device="cuda") for n, c in multi.heads.items()}
        multi.run_ops(x, 0, n_ops, heads, pre_img, pre_hm, pre_hm_hp)
        got = multi.forward(x, pre_img, pre_hm, pre_hm_hp)
        other = None
        for i, eng in enumerate(singles):
            want = eng.forward(x, pre_img, pre_hm[i], pre_hm_hp[i])
            assert multi.forward_launches == eng.forward_launches
            assert L.load().cp_plan_forward_launches(multi.plan) == eng.L.cp_plan_forward_launches(eng.plan)
            for n in want:
                assert torch.equal(got[n][i], want[n]), (label, prec, "model", i, n)
                assert torch.equal(heads[n][i], want[n]), (label, prec, "model", i, n, "run_ops")
            if i == 1:      # the heat maps matter: model 1 given model 0's maps is another result
                other = eng.forward(x, pre_img, pre_hm[0], pre_hm_hp[0])
                assert not torch.equal(other["hm"], want["hm"])
        with pytest.raises(ValueError, match="pre_hm"):
            multi.forward(x, pre_img, pre_hm[0], pre_hm_hp[0])


def test_track_splitk_ops_under_ceiling():
    """Split-K on, 512 x 512, batch 1: every op of every model against fp64, each model reading its own heat maps."""
    multi, _ = _track_engines("dla_34", 512, 512, 1, "tf32x3")
    x, pre_img, pre_hm, pre_hm_hp = _track_inputs(512, 512, 1)
    ext = [[x, pre_img, pre_hm[i], pre_hm_hp[i]] for i in range(M)]      # model i's view of the four inputs
    heads = {n: torch.full((M, 1, c, 128, 128), float("nan"), device="cuda") for n, c in multi.heads.items()}
    descs = [multi.op_descs(model=i) for i in range(M)]
    bad = []
    for k in range(len(descs[0])):
        wants = []
        with torch.no_grad():
            for i in range(M):
                rd = layer_ref.ActReader(multi.arena(), ext[i], [0], 1)
                wants.append((rd, layer_ref.op_ref(descs[i][k], rd, _fetch, descs[i])))
        multi.run_ops(x, k, k + 1, heads, pre_img, pre_hm, pre_hm_hp)
        torch.cuda.synchronize()
        d = descs[0][k]
        if d["fused_away"]:
            continue
        for i, (rd, want) in enumerate(wants):
            r = 0.0
            for (kind, tgt), ref, S in want:
                got = rd.get(tgt) if kind == "act" else heads[multi.head_names[tgt]][i].double()
                r = max(r, (0.0 if torch.equal(got, ref) else float("inf")) if d["family"] == L.FAM_MAXPOOL
                        else layer_ref.score(got, ref, S))
            if not r <= LAYER_CEIL[_ceiling(d, "tf32x3")]:
                bad.append((i, k, d["name"], r))
    assert not bad, bad


# ---- the tracker ---------------------------------------------------------------------------------------------------
def _cat_opt(hungarian, c=None):
    opt = _opt_from_gold(json.load(open(mg.OUT))["opt"])
    opt.conf_border = dict(BORDERS)
    opt.hungarian = hungarian
    if c is not None:
        opt.c = c
    return opt


@pytest.mark.parametrize("hungarian", (False, True), ids=("greedy", "hungarian"))
def test_tracker_multi_matches_per_category(hungarian, cplib, pose_host):
    """Three categories x two streams in one tracker against one tracker per category, stream 1 idle in two steps:
    tracks, n_tracks and the rendered heat maps bit for bit; and category 0's records stepped with category 1's settings
    give other tracks, so the comparison sees the per-category settings."""
    meta, frames0 = mg.make_sequence()
    name = "hungarian" if hungarian else "gt_first"
    frames, seeds = mgt.scenario_frames(name, frames0), mgt.seed_schedule("gt_first", frames0)
    S = 2
    opt = _cat_opt(hungarian)
    multi = cpb.Tracker(opt, streams=S, categories=CATS)
    assert multi.streams == M * S
    singles = [cpb.Tracker(_cat_opt(hungarian, c), streams=S) for c in CATS]
    swapped = cpb.Tracker(_cat_opt(hungarian, CATS[1]), streams=S)          # category 0's records, category 1's settings
    metat = cpb.make_meta(M * S, np.array([256., 256.], np.float32), 512.0, meta["width"], meta["height"],
                          meta["camera_matrix"]).cuda()
    tin = np.load(os.path.join(os.path.dirname(__file__), "golden", "track_render_gt.npz"))["gt_256_trans_input"].reshape(1, 6)
    recs = [[_frame_records(d, meta, pose_host, c) for c in CATS] for d in frames]
    differs = 0
    for f in range(len(frames)):
        if seeds[f] is not None:
            multi.seed([seeds[f]] * (M * S))
            for t in singles + [swapped]:
                t.seed([seeds[f]] * S)
        live = [0] if f in (2, 3) else [0, 1]
        n = len(live)
        poses = torch.cat([recs[f][m][0] for m in range(M) for _ in live])
        nv = torch.cat([recs[f][m][1] for m in range(M) for _ in live])
        ids = None if n == S else [m * S + s for m in range(M) for s in live]
        tr, nt = multi.step_records(poses, nv, metat[:M * n].contiguous(), stream_ids=ids)
        tr, nt = tr.cpu().numpy(), nt.cpu().numpy()
        sids = None if n == S else live
        for m, t in enumerate(singles):
            p1 = torch.cat([recs[f][m][0] for _ in live])
            n1 = torch.cat([recs[f][m][1] for _ in live])
            wt, wn = t.step_records(p1, n1, metat[:n].contiguous(), stream_ids=sids)
            wt, wn = wt.cpu().numpy(), wn.cpu().numpy()
            assert np.array_equal(nt[m * n:(m + 1) * n], wn), (f, m)
            assert np.array_equal(tr[m * n:(m + 1) * n], wt), (f, m, np.argwhere(tr[m * n:(m + 1) * n] != wt)[:8])
            if m == 0:
                st, sn = swapped.step_records(p1, n1, metat[:n].contiguous(), stream_ids=sids)
                differs += not np.array_equal(st.cpu().numpy(), wt)
        assert nt.sum() > 0
        if n == S:        # the heat maps of every category's tracks, one render
            hm, hp = multi.render(metat, tin, 256, 256)
            for m, t in enumerate(singles):
                whm, whp = t.render(metat[:S].contiguous(), tin, 256, 256)
                assert torch.equal(hm[m * S:(m + 1) * S], whm) and torch.equal(hp[m * S:(m + 1) * S], whp), (f, m)
    assert differs > 0


# ---- the detector ------------------------------------------------------------------------------------------------------
def _checkpoints(tmp_path, hungarian):
    opt = cpb.default_opt("dla_34", tracking_task=True)
    opt.conf_border = dict(BORDERS)
    opt.hungarian = hungarian
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, 512, 512, seed=5))).cuda()
    z = torch.zeros((2, 1, 512, 512), device="cuda")
    paths = {}
    for c, s in zip(CATS, SEEDS):
        m.load_state_dict(synth.seeded_state_dict(m, seed=s, offset_std=0.3))
        synth.calibrate_head_bias(m, m(x, x, z, z.repeat(1, 8, 1, 1))[-1], target=4)
        paths[c] = str(tmp_path / (c + ".pth"))
        cpb.save_model(paths[c], 1, m)
    return opt, paths


def _steps(cam):
    """Per step: (frames, per-slot cameras or one, new_video, seeded (category, slot) or None)."""
    arr = [synth.synthetic_frames(2, 512, 512, seed=40 + k) for k in range(2)]
    lst = [[synth.synthetic_frames(1, 480, 640, seed=60 + k)[0], synth.synthetic_frames(1, 600, 800, seed=70 + k)[0]]
           for k in range(4)]
    cams = np.stack([synth.default_camera(640, 480), synth.default_camera(800, 600)])
    return [
        (arr[0], cam, None, None),
        (arr[1], cam, None, None),
        (lst[0], cams, None, None),
        ([lst[1][0], None], cams, None, None),                   # slot 1 idle
        (lst[2], cams, [True, False], ("cup", 0)),                 # slot 0 restarts, seeded for one category
        (lst[3], cams, None, None),
    ]


@pytest.mark.parametrize("hungarian", (False, True), ids=("greedy", "hungarian"))
def test_detector_matches_per_category(hungarian, tmp_path):
    cam = synth.default_camera(512, 512)
    with no_splitk():
        opt, paths = _checkpoints(tmp_path, hungarian)
        det = cpb.MultiCategoryTracker(opt, paths)
        assert det.categories == list(CATS)
        ones = []
        for c in CATS:
            o = cpb.default_opt("dla_34", tracking_task=True, c=c, load_model=paths[c])
            o.conf_border, o.hungarian = dict(BORDERS), hungarian
            ones.append(cpb.ObjectPoseDetector(o))
        # pre_dets of the seeded slot: the results of a fresh run() of that category on another frame
        seeder = ones[1]
        seeder.run(synth.synthetic_frames(1, 512, 512, seed=9)[0], meta_inp={"camera_matrix": cam})
        pre = [dict(d) for d in seeder.run(synth.synthetic_frames(1, 512, 512, seed=8)[0],
                                           meta_inp={"camera_matrix": cam})["results"]]
        seeder.reset_tracking()
        assert pre
        kept = 0
        found = [0] * M
        prev = None
        for k, (frames, cams, new_video, seeded) in enumerate(_steps(cam)):
            kw = {} if new_video is None else {"new_video": new_video}
            pd = None
            if seeded is not None:
                pd = {seeded[0]: [pre if s == seeded[1] else None for s in range(2)]}
            out = None
            if k == 5:
                out = (torch.empty((M, 2, L.CP_MAX_K, L.CP_TRACK_RECORD), device="cuda"),
                       torch.empty((M, 2), dtype=torch.int32, device="cuda"))
            ret = det.run_batch(frames, cams, pre_dets=pd, to_host=out is None, out=out, **kw)
            if out is not None:
                assert ret[0] is out[0] and ret[1] is out[1]
                ret = (ret[0].cpu().numpy(), ret[1].cpu().numpy())
            tracks, nt = ret
            assert tracks.shape == (M, 2, L.CP_MAX_K, L.CP_TRACK_RECORD) and nt.shape == (M, 2)
            for m, (c, one) in enumerate(zip(CATS, ones)):
                pd1 = None if seeded is None or seeded[0] != c else pd[c]
                wt, wn = one.run_batch(frames, cams, track=True, pre_dets=pd1, **kw)
                assert np.array_equal(nt[m], wn), (k, c, nt[m], wn)
                assert np.array_equal(tracks[m], wt), (k, c, np.argwhere(tracks[m] != wt)[:8])
                found[m] += int(wn.sum())
            if isinstance(frames, list) and frames[1] is None:
                assert (nt[:, 1] == 0).all() and not tracks[:, 1].any()
            if prev is not None:
                for m in range(M):
                    ids = set(tracks[m, 0, :nt[m, 0], L.T_ID].tolist()) & set(prev[m, 0, :prev_n[m, 0], L.T_ID].tolist())
                    kept += bool(ids)
            prev, prev_n = tracks, nt
        assert kept > 0 and all(found), found
        # one category: [1, S, ...], the category alone
        one_cat = cpb.MultiCategoryTracker(opt, {"cup": paths["cup"]})
        solo = cpb.ObjectPoseDetector(cpb.default_opt("dla_34", tracking_task=True, c="cup", load_model=paths["cup"]))
        solo.opt.conf_border, solo.opt.hungarian = dict(BORDERS), hungarian
        for frames, cams, _, _ in _steps(cam)[:3]:
            t1, n1 = one_cat.run_batch(frames, cams)
            wt, wn = solo.run_batch(frames, cams, track=True)
            assert t1.shape == (1, 2, L.CP_MAX_K, L.CP_TRACK_RECORD) and n1.shape == (1, 2)
            assert np.array_equal(n1[0], wn) and np.array_equal(t1[0], wt)
        with pytest.raises(NotImplementedError):
            det.run(synth.synthetic_frames(1, 512, 512, seed=1)[0])
