"""TEST INFRASTRUCTURE ONLY.  Ground-truth seeding, ground-truth previous-frame heat maps and the optimal (hungarian)
association of the UNMODIFIED reference tracker (`utils/tracker.py`, `BaseDetector._get_additional_inputs`, through
`oracle/ref_shims.py`) on the seeded sequence of `oracle/make_golden_tracker.py`:

    tests/golden/tracker_seq_gt_first.json   init_track(meta['pre_dets']) at frame 0 (--gt_pre_hm_hmhp_first)
    tests/golden/tracker_seq_gt_every.json   init_track every frame with the previous frame's list (--gt_pre_hm_hmhp)
    tests/golden/tracker_seq_hungarian.json  --hungarian on a sequence where it differs from the greedy association
    tests/golden/track_render_gt.npz         the ground-truth branch of _get_additional_inputs on the seeded tracks
    tests/golden/tracker_opt_defaults.json   the reference's defaults of the tracker options

    python -m oracle.make_golden_tracker_gt         # needs /root/reference; rewrites the fixtures

Everything but `run_*` is importable without the reference: the tests rebuild the same inputs.  `pre_dets` are built
literally as tools/objectron_eval/eval_video_official.py:422-450 builds them (score 1, 1e-4 stds, one shared array for
kps_ori / kps_pnp / kps_gt) from the 2D keypoints of the sequence's objects, plus two objects without detections that
lie partly outside the frame and one seed at score 0.2 that must not start a track.
"""
import copy
import json
import os
import sys

import numpy as np

from oracle import make_golden_tracker as mg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SCENARIOS = ("gt_first", "gt_every", "hungarian")
GT_RENDER_CASES = [("gt_256", 256, 256), ("gt_320x384", 320, 384)]
OPT_DEFAULT_FIELDS = ("hungarian", "gt_pre_hm_hmhp", "gt_pre_hm_hmhp_first", "empty_pre_hm")


def _moved(det, centre, scale):
    """A copy of a detection dict with its 2D geometry scaled by `scale` about its centre and moved to `centre`
    (heat-map sentinels kept), zero tracking offsets."""
    d = copy.deepcopy(det)
    c0 = np.array(det["ct"], np.float64)
    c1 = np.asarray(centre, np.float64)

    def mv(v):
        a = np.asarray(v, np.float64).reshape(-1, 2).copy()
        keep = a[:, 0] > -1000
        a[keep] = c1 + scale * (a[keep] - c0)
        return a.reshape(-1)
    for k in ("kps", "kps_displacement_mean", "kps_heatmap_mean"):
        d[k] = mv(d[k])
    b = np.asarray(det["bbox"], np.float64).reshape(2, 2)
    d["bbox"] = [float(v) for v in (c1 + scale * (b - c0)).reshape(-1)]
    d["ct"] = [float(c1[0]), float(c1[1])]
    d["tracking"] = np.zeros(2)
    d["tracking_hp"] = np.zeros(16)
    return d


def scenario_frames(name, frames):
    """The detection lists a scenario steps through (deep copies of make_sequence's frames)."""
    frames = copy.deepcopy(frames)
    if name != "hungarian":
        return frames
    src = frames[0][0]
    # frames 1-2: two tracks A / B side by side; in frame 2 d0 is nearest to B but d1 is valid for B only, so greedy
    # gives d0 -> B and starts a new track for d1 while the optimal assignment pairs d0 -> A, d1 -> B
    a, dx = np.array([80.0, 80.0]), 26.0
    frames[1] += [_moved(src, a, 0.35), _moved(src, a + [dx, 0], 0.35)]
    frames[2] += [_moved(src, a + [0.7 * dx, 0], 0.35), _moved(src, a + [1.9 * dx, 0], 0.35)]
    # frame 3: object 2 is missed and A / B get no detection, so three tracks have no valid pairing; four new objects
    # come first in the list, so N > M: the solver pairs those tracks with three of them at 1e18, the post-filter drops
    # these pairs and appends their detections to unmatched_dets after the fourth, which reorders the new ids
    frames[3] = [_moved(src, c, 0.35) for c in ([430.0, 440.0], [80.0, 440.0], [440.0, 80.0], [256.0, 470.0])] + frames[3]
    return frames


def gt_list(dets, width=mg.WIDTH, height=mg.HEIGHT):
    """pre_dets of one frame, eval_video_official.py:422-450: one dict per object of the frame, two ground-truth objects
    without a detection that reach outside the frame (left / below, right), and one seed at score 0.2."""
    objs = [(np.asarray(d["kps"], np.float64).reshape(8, 2), d["obj_scale"]) for d in dets[:3]]
    base = objs[0][0] - objs[0][0].mean(0)
    objs.append((base * 0.15 + [15.0, 500.0], objs[0][1]))          # partly left of and below the frame
    objs.append((base * 0.15 + [515.0, 60.0], objs[0][1]))          # partly right of the frame
    out = []
    for i, (k8, sc) in enumerate(objs + [objs[1]]):
        kps_pix = np.vstack([k8.mean(0, keepdims=True), k8])
        kps_ori = kps_pix / [width, height]                        # normalised 9 x 2
        kps = copy.deepcopy(kps_ori)
        kps[:, 0] = kps_ori[:, 0] * width
        kps[:, 1] = kps_ori[:, 1] * height
        xs, ys = zip(*kps)
        bbox = [min(xs), min(ys), max(xs), max(ys)]
        kps = kps[1:].flatten()
        scale = np.asarray(sc, np.float64) / np.asarray(sc, np.float64)[1]
        out.append({"bbox": bbox, "score": 1 if i < len(objs) else 0.2, "cls": 0, "obj_scale": scale,
                    "obj_scale_uncertainty": np.ones(3) * 1e-4, "tracking": np.zeros(2), "tracking_hp": np.zeros(16),
                    "kps": kps, "kps_displacement_mean": kps, "kps_displacement_std": np.ones(16) * 1e-4,
                    "kps_heatmap_mean": kps, "kps_heatmap_std": np.ones(16) * 1e-4, "kps_heatmap_height": np.ones(8),
                    "kps_fusion_mean": kps, "kps_fusion_std": np.ones(16) * 1e-4, "kps_pnp": kps_ori, "kps_gt": kps_ori,
                    "kps_3d_cam": np.zeros((9, 3)), "kps_ori": kps_ori})
    return out


def seed_schedule(name, frames):
    """Per frame: the list handed to init_track as meta['pre_dets'] (eval_video_official.py:452-456), or None.  With
    gt_pre_hm_hmhp frame f > 0 gets frame f-1's list -- frame 1 gets the very list object frame 0 was seeded with."""
    lists = [gt_list(d) for d in frames]
    if name == "gt_first":
        return [lists[0]] + [None] * (len(frames) - 1)
    if name == "gt_every":
        return [lists[0]] + [lists[f - 1] for f in range(1, len(frames))]
    return [None] * len(frames)


def run_scenario(name, Tracker, pnp_shell, gaussian_fusion, opt):
    """Tracker.step over one scenario; `Tracker` / `pnp_shell` are the reference's or the restatement's."""
    meta, frames0 = mg.make_sequence()
    frames = scenario_frames(name, frames0)
    seeds = seed_schedule(name, frames0)
    trk = Tracker(opt)
    out = []
    for f, dets in enumerate(frames):
        m = dict(meta, id=f)
        if seeds[f] is not None:
            m["pre_dets"] = seeds[f]
        if f == 0 or seeds[f] is not None:                        # base_detector.py:444-454
            trk.init_track(m)
        results = copy.deepcopy(dets)
        boxes = []
        for det in results:
            det["kps_fusion_mean"], det["kps_fusion_std"] = gaussian_fusion(det, opt.hps_uncertainty)
            r = pnp_shell(det, mg.assemble_points(det), m)
            if r is not None:
                boxes.append(r)
        ret, bx = trk.step(results, boxes)
        out.append(mg.summarize(ret, bx))
    return out


def _ref_opt(name):
    from oracle import ref_shims
    ref_shims.install()
    opt = ref_shims.make_opt("dla_34", tracking_task=True, rep_mode=1, c="chair")
    opt.hungarian = name == "hungarian"
    opt.gt_pre_hm_hmhp = name == "gt_every"
    opt.gt_pre_hm_hmhp_first = name == "gt_first"
    return opt


def run_reference(name):
    sys.path.insert(0, ROOT)
    from oracle import tracker_ref
    opt = _ref_opt(name)
    from lib.utils.tracker import Tracker
    from lib.utils.pnp.cuboid_pnp_shell import pnp_shell

    def shell(det, pts, meta):
        return pnp_shell(opt, meta, det, pts, det["obj_scale"], OPENCV_RETURN=opt.show_axes)
    frames = run_scenario(name, Tracker, shell, tracker_ref.gaussian_fusion, opt)
    opts = {k: getattr(opt, k) for k in ("kalman", "scale_pool", "hungarian", "use_pnp", "new_thresh", "max_age", "R", "c",
                                         "show_axes", "hps_uncertainty")}
    opts["conf_border"] = opt.conf_border[opt.c]
    return {"scenario": name, "opt": opts, "frames": frames}


def run_reference_render_gt():
    """The unmodified ground-truth branch of `_get_additional_inputs` (base_detector.py:166-209) on the tracks seeded
    from frame 0's pre_dets (gt_pre_hm_hmhp_first, meta['id'] == 0)."""
    import types
    import torch
    opt = _ref_opt("gt_first")
    opt.device = torch.device("cpu")
    from lib.utils.tracker import Tracker
    from lib.detectors.base_detector import BaseDetector
    stub = types.SimpleNamespace(opt=opt)
    stub._trans_bbox = lambda *a: BaseDetector._trans_bbox(stub, *a)
    meta, frames = mg.make_sequence()
    out = {}
    for name, ih, iw in GT_RENDER_CASES:
        trk = Tracker(opt)
        trk.init_track(dict(meta, id=0, pre_dets=gt_list(frames[0])))
        rm = dict(mg.render_meta(ih, iw), id=0)
        hm, hm_hp, _ = BaseDetector._get_additional_inputs(stub, trk.tracks, rm, with_hm=True, with_hm_hp=True)
        for key, v in (("_hm", hm.numpy()[0]), ("_hm_hp", hm_hp.numpy()[0])):
            if ih * iw <= 256 * 256:
                out[name + key] = v
            else:
                out[name + key + "_sub4"] = np.ascontiguousarray(v[:, ::4, ::4])
                out[name + key + "_sum"] = v.astype(np.float64).sum(axis=(1, 2))
                out[name + key + "_nnz"] = (v != 0).sum(axis=(1, 2)).astype(np.int64)
        out[name + "_trans_input"] = rm["trans_input"]
        print(name, "tracks", len(trk.tracks), "hm_hp nnz per joint", [int((c != 0).sum()) for c in hm_hp[0]])
    return out


def run_reference_defaults():
    from oracle import ref_shims
    opt = ref_shims.make_opt("dla_34", tracking_task=True, rep_mode=1, c="chair")
    return {k: bool(getattr(opt, k)) for k in OPT_DEFAULT_FIELDS}


if __name__ == "__main__":
    for sc in SCENARIOS:
        g = run_reference(sc)
        path = os.path.join(GOLDEN, "tracker_seq_%s.json" % sc)
        with open(path, "w") as f:
            json.dump(g, f)
        print("wrote", path, [[t["tracking_id"] for t in fr["tracks"]] for fr in g["frames"]])
    np.savez_compressed(os.path.join(GOLDEN, "track_render_gt.npz"), **run_reference_render_gt())
    with open(os.path.join(GOLDEN, "tracker_opt_defaults.json"), "w") as f:
        json.dump(run_reference_defaults(), f)
    print("wrote track_render_gt.npz, tracker_opt_defaults.json")
