"""TrackGraph over several categories and over slots of different frame sizes, on the device.  Every case runs a 12-step
synthetic video through the graph, interleaved step by step with the host-driven path on the same object, and checks
every step's tracks and n_tracks bit for bit:

  * MultiCategoryTrackGraph (chair / cup / laptop, with their own visible_thresh and conf_border) against
    MultiCategoryTracker.run_batch's array form: 1 and 4 slots, greedy and Hungarian association, BGR, NV12 and I420,
    pinned and device frames, a new video on one slot at step 5 and on every slot at step 9, opt.empty_pre_hm;
  * TrackGraph with one frame_hw per slot (480 x 640, 720 x 1280, 1440 x 1080 and odd sizes, a camera per slot) against
    run_batch(list, track=True), and MultiCategoryTrackGraph with per-slot sizes against MultiCategoryTracker.run_batch
    (list);
  * cp_preprocess_slots_ragged_dev alone against cp_preprocess_ragged / cp_preprocess_yuv420, with prev written on the
    start rows only;
  * the captured graphs hold kernels, memsets and empty nodes only, and a step is (frame copies + 1) host-to-device
    copies and one graph launch; replay from reset() repeats itself and the tracker's slot state is left alone."""
import collections
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import affine_from_center_scale
from centerpose_b200.engine import preprocess_ragged, preprocess_yuv420
from tests.test_gpu_track_graph import (CU_GRAPH_NODE_TYPE_EMPTY, CU_GRAPH_NODE_TYPE_KERNEL, CU_GRAPH_NODE_TYPE_MEMSET,
                                        H, STEPS, W, _cameras, _detector, _host, _new_video, _node_types, _video)
from tests.test_gpu_yuv_input import from_bgr

pytestmark = pytest.mark.gpu
CATS = ("chair", "cup", "laptop")                       # visible_thresh 6 / 3 / 0
SEEDS = (21, 22, 23)
BORDERS = {"chair": [3, 9], "cup": [2, 8], "laptop": [4, 10]}
SIZES = [(480, 640), (720, 1280), (1440, 1080)]
ODD = [(481, 641), (720, 1279), (1441, 1079)]


@pytest.fixture(scope="module")
def checkpoints(tmp_path_factory):
    """One seeded tracking checkpoint per category, heat-map biases calibrated to about 4 objects per frame."""
    opt = cpb.default_opt("dla_34", tracking_task=True)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, 512, 512, seed=5))).cuda()
    z = torch.zeros((2, 1, 512, 512), device="cuda")
    d = tmp_path_factory.mktemp("ckpt")
    paths = {}
    for c, s in zip(CATS, SEEDS):
        m.load_state_dict(synth.seeded_state_dict(m, seed=s, offset_std=0.3))
        with torch.no_grad():
            synth.calibrate_head_bias(m, m(x, x, z, z.repeat(1, 8, 1, 1))[-1], target=4)
        paths[c] = str(d / (c + ".pth"))
        cpb.save_model(paths[c], 1, m)
    return paths


def _tracker(paths, cats=CATS, hungarian=False, empty_pre_hm=False):
    opt = cpb.default_opt("dla_34", tracking_task=True)
    opt.conf_border, opt.hungarian, opt.empty_pre_hm = dict(BORDERS), hungarian, empty_pre_hm
    trk = cpb.MultiCategoryTracker(opt, {c: paths[c] for c in cats})
    assert trk.categories == list(cats)
    return trk


def _restart(trk, new):
    """The array form of run_batch starts a slot's video when the slot has not started in the slot state (the rule
    run_batch(list) applies to new_video)."""
    if new is not None and trk._slots is not None:
        for i, n in enumerate(new):
            if n:
                trk._slots.started[i] = False


def _place(f, where):
    t = torch.from_numpy(np.ascontiguousarray(f))
    return t.pin_memory() if where == "pinned" else t.cuda()


def _check_step(k, got, want, new, lead):
    gt, gn = _host(got)
    wt, wn = want
    assert gt.shape == lead + (L.CP_MAX_K, L.CP_TRACK_RECORD) and gn.shape == lead
    assert np.array_equal(gn, wn), (k, gn, wn)
    assert np.array_equal(gt, wt), (k, np.argwhere(gt != wt)[:8])
    if new is not None:                                  # a new video numbers its tracks from 1 again
        g2, n2 = gt.reshape((-1,) + gt.shape[-3:]), gn.reshape((-1,) + gn.shape[-1:])
        for i in np.flatnonzero(new):
            for t, n in zip(g2, n2):
                assert n[i] == 0 or t[i, :n[i], L.T_ID].min() == 1
    return int(wn.sum())


# ---- several categories, one frame size ------------------------------------------------------------------------------
MULTI_CASES = [  # slots, hungarian, pixel format, where the frames are, opt.empty_pre_hm
    (1, False, "bgr", "pinned", False),
    (4, True, "nv12", "device", False),
    (4, False, "i420", "pinned", False),
    (1, True, "i420", "device", False),
    (4, False, "bgr", "device", True),
]


@pytest.mark.parametrize("S, hungarian, fmt, where, empty", MULTI_CASES)
def test_multi_category_graph_matches_run_batch(S, hungarian, fmt, where, empty, checkpoints, cplib):
    trk = _tracker(checkpoints, hungarian=hungarian, empty_pre_hm=empty)
    cam = _cameras(S)
    tg = cpb.MultiCategoryTrackGraph(trk, slots=S, frame_hw=(H, W), camera_matrix=cam, pixel_format=fmt)
    assert trk._slots is None and tg.eng.models == len(CATS)
    total = 0
    for k, f in enumerate(_video(S, fmt, seed=170 + S)):
        new = _new_video(k, S)
        got = tg(_place(f, where), new_video=new)
        _restart(trk, new)
        total += _check_step(k, got, trk.run_batch(f, cam, pixel_format=fmt), new, (len(CATS), S))
    assert total > 0


# ---- one frame size per slot --------------------------------------------------------------------------------------
def _ragged_video(sizes, fmt, seed, steps=STEPS):
    """Per step one frame per slot, each of its own size: noise shifted a few pixels every step."""
    bases = [synth.synthetic_frames(1, h, w, seed=seed + i)[0] for i, (h, w) in enumerate(sizes)]
    out = []
    for k in range(steps):
        fs = [np.roll(b, (2 * k, 3 * k), axis=(0, 1)) for b in bases]
        out.append(fs if fmt == "bgr" else [from_bgr(g, fmt) for g in fs])
    return out


def _slot_cameras(sizes):
    return np.stack([synth.default_camera(w, h) for h, w in sizes])


RAGGED_CASES = [(SIZES, "bgr"), (SIZES, "nv12"), (SIZES, "i420"), (ODD, "bgr")]


@pytest.mark.parametrize("sizes, fmt", RAGGED_CASES, ids=["bgr", "nv12", "i420", "bgr odd sizes"])
def test_per_slot_sizes_match_run_batch_list(sizes, fmt, cplib):
    det = _detector(hungarian=fmt == "nv12")
    S, cams = len(sizes), _slot_cameras(sizes)
    tg = cpb.TrackGraph(det, slots=S, frame_hw=sizes, camera_matrix=cams, pixel_format=fmt)
    assert tg.per_slot and det._slots is None
    total = 0
    for k, fs in enumerate(_ragged_video(sizes, fmt, seed=300)):
        new = _new_video(k, S)
        got = tg([_place(f, "pinned" if i % 2 else "device") for i, f in enumerate(fs)], new_video=new)
        want = det.run_batch(fs, cams, track=True, new_video=new, pixel_format=fmt)
        total += _check_step(k, got, want, new, (S,))
    assert total > 0


def test_multi_category_per_slot_sizes_match_run_batch_list(checkpoints, cplib):
    trk = _tracker(checkpoints, cats=CATS[:2])
    sizes = SIZES[:2]
    S, cams = len(sizes), _slot_cameras(sizes)
    tg = cpb.MultiCategoryTrackGraph(trk, slots=S, frame_hw=sizes, camera_matrix=cams)
    total = 0
    for k, fs in enumerate(_ragged_video(sizes, "bgr", seed=400)):
        new = _new_video(k, S)
        got = tg([_place(f, "pinned") for f in fs], new_video=new)
        total += _check_step(k, got, trk.run_batch(fs, cams, new_video=new), new, (2, S))
    assert total > 0


# ---- the kernel alone ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["bgr", "nv12", "i420"])
def test_slots_ragged_kernel_matches_the_ragged_calls(fmt, cplib):
    sizes = (ODD if fmt == "bgr" else SIZES) + [(512, 512)]
    frames = [synth.synthetic_frames(1, h, w, seed=500 + i)[0] for i, (h, w) in enumerate(sizes)]
    frames = frames if fmt == "bgr" else [from_bgr(f, fmt) for f in frames]
    B, ih, iw = len(frames), 512, 512
    offs, o = [], 3                                    # odd byte offsets, a gap between frames
    for f in frames:
        offs.append(o)
        o += f.size + 5
    packed = torch.zeros(o, dtype=torch.uint8)
    for f, off in zip(frames, offs):
        packed[off:off + f.size] = torch.from_numpy(f.reshape(-1))
    packed = packed.cuda()
    offs, hw = np.array(offs, np.int64), np.array(sizes, np.int32)
    # rotated / anisotropic affines as well as the fix_res one
    trans = np.stack([affine_from_center_scale(np.array([w / 2., h / 2.], np.float32), float(max(h, w)), iw, ih)
                      for h, w in sizes])
    trans[1, 0, 1] += 0.05
    trans[2, 1, 1] *= 0.9
    mean, std = (0.408, 0.447, 0.470), (0.289, 0.274, 0.278)
    if fmt == "bgr":
        want = preprocess_ragged(packed, offs, hw, ih, iw, mean, std, trans_input=trans)
    else:
        want = preprocess_yuv420(packed, offs, hw, fmt, ih, iw, mean, std, trans_input=trans)
    fcode = {"bgr": L.CP_PIX_BGR, "nv12": L.CP_PIX_NV12, "i420": L.CP_PIX_I420}[fmt]
    table = torch.zeros(int(cplib.cp_preprocess_frame_table_bytes(B)), dtype=torch.uint8, device="cuda")
    tr = np.ascontiguousarray(trans, np.float64)
    L.check(cplib.cp_preprocess_frame_table(packed.numel(), offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                            hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), fcode, B, ih, iw,
                                            tr.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                            ctypes.c_void_p(table.data_ptr()), None), "cp_preprocess_frame_table")
    m, s = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    start = torch.tensor([1, 0, 1, 0], dtype=torch.int32, device="cuda")
    out = torch.full((B, 3, ih, iw), float("nan"), device="cuda")
    prev = torch.full_like(out, float("nan"))
    st = torch.cuda.current_stream().cuda_stream
    args = (ctypes.c_void_p(packed.data_ptr()), ctypes.c_void_p(table.data_ptr()), fcode, B, ih, iw, m, s)
    L.check(cplib.cp_preprocess_slots_ragged_dev(*args, ctypes.c_void_p(start.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                                 ctypes.c_void_p(prev.data_ptr()), ctypes.c_void_p(st)),
            "cp_preprocess_slots_ragged_dev")
    assert torch.equal(out, want)
    for b in range(B):
        if start[b]:
            assert torch.equal(prev[b], want[b]), b
        else:
            assert torch.isnan(prev[b]).all(), b
    # without start / prev: the same network input
    out2 = torch.full_like(out, float("nan"))
    L.check(cplib.cp_preprocess_slots_ragged_dev(*args, None, ctypes.c_void_p(out2.data_ptr()), None,
                                                 ctypes.c_void_p(st)), "cp_preprocess_slots_ragged_dev")
    assert torch.equal(out2, want)


# ---- graph structure, replay and state ---------------------------------------------------------------------------------
def _profile_steps(tg, steps):
    for f in steps[:2]:
        tg(f)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for f in steps[2:]:
            tg(f)
        torch.cuda.synchronize()
    return collections.Counter(e.name for e in prof.events()), len(steps) - 2


@pytest.mark.parametrize("kind", ["several categories", "per-slot sizes"])
def test_a_step_is_frame_copies_and_one_graph_launch(kind, checkpoints, cplib):
    if kind == "several categories":
        S = 2
        tg = cpb.MultiCategoryTrackGraph(_tracker(checkpoints, hungarian=True), slots=S, frame_hw=(H, W),
                                         camera_matrix=synth.default_camera(W, H))
        steps = [torch.from_numpy(f).pin_memory() for f in _video(S, "bgr", seed=197, steps=6)]
        copies_per_step = 2
    else:
        S = len(SIZES)
        tg = cpb.TrackGraph(_detector(hungarian=True), slots=S, frame_hw=SIZES, camera_matrix=_slot_cameras(SIZES),
                            pixel_format="nv12")
        steps = [[torch.from_numpy(f).pin_memory() for f in fs] for fs in _ragged_video(SIZES, "nv12", 600, steps=6)]
        copies_per_step = S + 1
    kinds = [_node_types(g) for g in tg.graphs]
    assert kinds[0] == kinds[1]
    assert set(kinds[0]) <= {CU_GRAPH_NODE_TYPE_KERNEL, CU_GRAPH_NODE_TYPE_MEMSET, CU_GRAPH_NODE_TYPE_EMPTY}, kinds[0]
    assert kinds[0][CU_GRAPH_NODE_TYPE_KERNEL] >= tg.eng.forward_launches + 5
    names, n = _profile_steps(tg, steps)
    # the copies the host issues, and on the device host-to-device copies only (counted from the issuing side: the
    # device-side copy records of a later profiler session in the same process are not always complete)
    copies = {k: c for k, c in names.items() if k.startswith("Memcpy")}
    assert names["cudaMemcpyAsync"] == copies_per_step * n, names
    assert copies and all(k.startswith("Memcpy HtoD") for k in copies), copies
    assert names["cudaGraphLaunch"] == n
    assert names["cudaLaunchKernel"] == 0 and names["cudaMemsetAsync"] == 0
    assert names["cudaStreamSynchronize"] == 0 and names["cudaEventSynchronize"] == 0, names


def test_multi_category_replay_and_the_trackers_slots(checkpoints, cplib):
    """Replay from reset() repeats itself; trk.run_batch steps around the graph give what a tracker that never saw the
    graph gives, and trk._slots stays the same object."""
    S, cam = 2, synth.default_camera(W, H)
    vid = _video(S, "bgr", seed=190, steps=6)
    ref = _tracker(checkpoints)
    want = [ref.run_batch(f, cam) for f in vid]
    trk = _tracker(checkpoints)
    got = [trk.run_batch(f, cam) for f in vid[:2]]
    slots = trk._slots
    tg = cpb.MultiCategoryTrackGraph(trk, slots=S, frame_hw=(H, W), camera_matrix=cam)
    runs = []
    for _ in range(2):
        tg.reset()
        runs.append([_host(tg(torch.from_numpy(f).cuda(), new_video=_new_video(k, S))) for k, f in enumerate(vid)])
    assert sum(int(n.sum()) for _, n in runs[0]) > 0
    for (a_t, a_n), (b_t, b_n) in zip(*runs):
        assert np.array_equal(a_n, b_n) and np.array_equal(a_t, b_t)
    assert trk._slots is slots
    got += [trk.run_batch(f, cam) for f in vid[2:]]
    for (gt, gn), (wt, wn) in zip(got, want):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt)
    # what the graph does not take
    with pytest.raises(NotImplementedError, match="pre_dets seeding runs through MultiCategoryTracker.run_batch"):
        tg(vid[0], pre_dets={"cup": [[], []]})
    with pytest.raises(ValueError, match=r"idle slots and mixed sizes run through MultiCategoryTracker.run_batch\(list\) "
                                         r"or a MultiCategoryTrackGraph built with one frame_hw per slot"):
        tg([vid[0][0], None])
    rg = cpb.TrackGraph(_detector(), slots=2, frame_hw=SIZES[:2], camera_matrix=_slot_cameras(SIZES[:2]))
    fs = _ragged_video(SIZES[:2], "bgr", 700, steps=1)[0]
    with pytest.raises(ValueError, match=r"slot 1 is idle; idle slots run through run_batch\(list, track=True\)"):
        rg([fs[0], None])
    with pytest.raises(ValueError, match=r"slot 1 takes uint8 \[720, 1280, 3\] frames \(bgr, frame_hw \(720, 1280\)\)"):
        rg([fs[0], fs[0]])
    with pytest.raises(ValueError, match="frames is a list of 2 frames"):
        rg(np.stack([fs[0], fs[0]]))
