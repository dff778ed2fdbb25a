"""DetectGraph and MultiCategoryDetectGraph on the device.  Every case runs a 10-step synthetic video through the graph,
interleaved step by step with run_batch on the same detector, and checks every step's poses and n_valid bit for bit:

  * DetectGraph against run_batch's array form: 1 and 3 slots, BGR, NV12 and I420, pinned and device frames, tf32x3,
    one bf16 case and one res_18 case;
  * one frame_hw per slot (480 x 640 and 720 x 1280, a camera per slot) against run_batch(list);
  * idle cameras (a late start, a pause, an end and an all-idle step) against run_batch(list) of the live frames with
    their cameras, scattered to the slots;
  * MultiCategoryDetectGraph (M = 2, and M = 1) against MultiCategoryDetector.run_batch, with and without idle slots;
  * the captured graph holds kernels and memsets only, and a call is one copy per live frame (plus the control block
    with idle slots) and one graph launch, profiled in a child process so that this process never starts the profiler.

The reference runs on a plan of the graph's capacity: split-K is chosen from the plan's workspace, which its max batch
sizes, and run_batch keeps the largest plan it has made.  So every detector's plan is made at S frames (_capacity)
before the first step."""
import subprocess
import sys

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from tests.test_gpu_track_graph import (CU_GRAPH_NODE_TYPE_EMPTY, CU_GRAPH_NODE_TYPE_KERNEL, CU_GRAPH_NODE_TYPE_MEMSET,
                                        H, W, _cameras, _host, _node_types, _video)
from tests.test_gpu_track_graph_multi import _place, _profile_steps, _ragged_video, _slot_cameras
from tests.util import ROOT

pytestmark = pytest.mark.gpu
STEPS = 10
SIZES = [(480, 640), (720, 1280)]
CATS = ("chair", "cup")


def _calibrated(m, seed, opt):
    """Seeded weights with the heat-map biases calibrated to about 8 objects per frame on the 512 x 512 network input of
    one 480 x 640 frame like the test videos' (one frame, so the model's plan holds one frame until _capacity grows
    it)."""
    m.load_state_dict(synth.seeded_state_dict(m, seed=seed, offset_std=0.3))
    f = torch.from_numpy(synth.synthetic_frames(1, H, W, seed=5)).cuda()
    x = cpb.preprocess(f, opt.input_h, opt.input_w, opt.mean, opt.std)
    with torch.no_grad():
        synth.calibrate_head_bias(m, m(x)[-1], target=8)
    return m


def _detector(arch="dla_34", precision="tf32x3", seed=41):
    opt = cpb.default_opt(arch)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    m.precision = precision
    det = cpb.ObjectPoseDetector(opt, model=_calibrated(m, seed, opt))
    assert det.model.precision == precision and not getattr(opt, "tracking_task", False)
    return det


def _capacity(det, S):
    """Make the detector's plan hold S frames, the graph's capacity (see the module docstring)."""
    ih, iw = det.opt.input_h, det.opt.input_w
    eng = det.engine(S, ih, iw) if isinstance(det, cpb.MultiCategoryDetector) else det.model.engine(S, ih, iw)
    assert eng.max_batch == S


@pytest.fixture(scope="module")
def checkpoints(tmp_path_factory):
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    d = tmp_path_factory.mktemp("det_ckpt")
    paths = {}
    for c, s in zip(CATS, (51, 52)):
        paths[c] = str(d / (c + ".pth"))
        cpb.save_model(paths[c], 1, _calibrated(m, s, opt))
    return paths


def _check(k, got, want, lead):
    gp, gn = _host(got)
    wp, wn = want
    assert gp.shape == lead + (100, L.CP_POSE_RECORD) and gn.shape == lead and gn.dtype == np.int32
    assert np.array_equal(gn, wn), (k, gn, wn)
    assert np.array_equal(gp, wp), (k, np.argwhere(gp != wp)[:8])
    return int(wn.sum() > 0)


def _scattered(run, fs, cams, lead):
    """The reference of a step with idle slots: run (run_batch) on the live frames with their cameras, its rows scattered
    to the slots, zeros for the idle ones."""
    live = [i for i, f in enumerate(fs) if f is not None]
    S = len(fs)
    poses = np.zeros(lead[:-1] + (S, 100, L.CP_POSE_RECORD), np.float32)
    n = np.zeros(lead[:-1] + (S,), np.int32)
    if live:
        p, c = run([fs[i] for i in live], np.stack([cams[i] for i in live]))
        poses[..., live, :, :], n[..., live] = p, c
    return poses, n


CASES = [  # slots, pixel format, where the frames are, arch, precision
    (1, "bgr", "pinned", "dla_34", "tf32x3"),
    (3, "nv12", "device", "dla_34", "tf32x3"),
    (3, "i420", "pinned", "dla_34", "tf32x3"),
    (3, "bgr", "device", "dla_34", "bf16"),
    (1, "nv12", "pinned", "res_18", "tf32x3"),
]


@pytest.mark.parametrize("S, fmt, where, arch, precision", CASES)
def test_graph_matches_run_batch(S, fmt, where, arch, precision, cplib):
    det = _detector(arch, precision)
    cams = _cameras(S)
    g = cpb.DetectGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cams, pixel_format=fmt)
    assert len(g.graphs) == 1
    _capacity(det, S)
    hits = 0
    for k, f in enumerate(_video(S, fmt, seed=300 + S, steps=STEPS)):
        got = g(_place(f, where))
        # the same detector's run_batch between graph calls: the graph has its own plan and buffers
        hits += _check(k, got, det.run_batch(f, cams, pixel_format=fmt), (S,))
    assert hits > STEPS // 2, hits


@pytest.mark.parametrize("fmt, where", [("bgr", "pinned"), ("nv12", "device")])
def test_per_slot_sizes_match_run_batch_list(fmt, where, cplib):
    det = _detector()
    S, cams = len(SIZES), _slot_cameras(SIZES)
    g = cpb.DetectGraph(det, slots=S, frame_hw=SIZES, camera_matrix=cams, pixel_format=fmt)
    _capacity(det, S)
    hits = 0
    for k, fs in enumerate(_ragged_video(SIZES, fmt, seed=320, steps=STEPS)):
        got = g([_place(f, where) for f in fs])
        hits += _check(k, got, det.run_batch(fs, cams, pixel_format=fmt), (S,))
    assert hits > STEPS // 2, hits


S_IDLE = 4
LIVE = [  # per step, the live slots: slot 1 starts late, slot 0 pauses, slot 2 ends, one step with every camera idle
    {0, 2, 3}, {0, 2}, {0, 1, 2, 3}, {1, 2}, {2}, set(), {0, 1, 3}, {0, 1}, {1, 3}, {0, 1, 3},
]


def test_the_idle_pattern_covers_what_it_must():
    assert {len(lv) for lv in LIVE} == set(range(S_IDLE + 1)) and len(LIVE) == STEPS
    first = [min(k for k, lv in enumerate(LIVE) if i in lv) for i in range(S_IDLE)]
    last = [max(k for k, lv in enumerate(LIVE) if i in lv) for i in range(S_IDLE)]
    assert first[1] > 0 and last[2] < STEPS - 3
    ks = [k for k, lv in enumerate(LIVE) if 0 in lv]
    assert any(b - a > 1 for a, b in zip(ks, ks[1:]))                  # slot 0 pauses and resumes


def _idle_steps(sizes, fmt, seed):
    video = _ragged_video(sizes, fmt, seed, steps=STEPS)
    return [[f if i in lv else None for i, f in enumerate(fs)] for fs, lv in zip(video, LIVE)]


@pytest.mark.parametrize("kind, fmt, where", [("one", "bgr", "pinned"), ("per-slot", "nv12", "device")])
def test_idle_graph_matches_run_batch_of_the_live_frames(kind, fmt, where, cplib):
    det = _detector()
    sizes = [(H, W)] * S_IDLE if kind == "one" else SIZES + [(512, 384), (480, 640)]
    cams = _slot_cameras(sizes)
    g = cpb.DetectGraph(det, slots=S_IDLE, frame_hw=(H, W) if kind == "one" else sizes, camera_matrix=cams,
                        pixel_format=fmt, idle_slots=True)
    assert len(g.graphs) == S_IDLE
    _capacity(det, S_IDLE)
    hits = 0
    for k, fs in enumerate(_idle_steps(sizes, fmt, seed=340)):
        got = g([None if f is None else _place(f, where) for f in fs])
        want = _scattered(lambda fr, c: det.run_batch(fr, c, pixel_format=fmt), fs, cams, (S_IDLE,))
        hits += _check(k, got, want, (S_IDLE,))
        for i in range(S_IDLE):
            if fs[i] is None:
                assert want[1][i] == 0 and not want[0][i].any()
    assert hits > STEPS // 2, hits
    # every slot live as one array with one frame_hw
    if kind == "one":
        f = _video(S_IDLE, fmt, seed=360, steps=1)[0]
        _check(0, g(_place(f, where)), det.run_batch(f, cams, pixel_format=fmt), (S_IDLE,))


@pytest.mark.parametrize("cats, S, idle, fmt, where", [
    (CATS, 3, False, "bgr", "pinned"),
    (CATS, S_IDLE, True, "i420", "device"),
    (CATS[:1], 2, False, "nv12", "device"),
])
def test_multi_category_graph_matches_run_batch(cats, S, idle, fmt, where, checkpoints, cplib):
    opt = cpb.default_opt("dla_34")
    mdet = cpb.MultiCategoryDetector(opt, {c: checkpoints[c] for c in cats})
    M = len(cats)
    lead = (M, S)
    if idle:
        sizes = SIZES + [(512, 384), (480, 640)]
        cams = _slot_cameras(sizes)
        g = cpb.MultiCategoryDetectGraph(mdet, slots=S, frame_hw=sizes, camera_matrix=cams, pixel_format=fmt,
                                         idle_slots=True)
        steps = _idle_steps(sizes, fmt, seed=380)
    else:
        cams = _cameras(S)
        g = cpb.MultiCategoryDetectGraph(mdet, slots=S, frame_hw=(H, W), camera_matrix=cams, pixel_format=fmt)
        steps = _video(S, fmt, seed=390, steps=STEPS)
    assert g.eng.models == M and g.categories == list(cats)
    _capacity(mdet, S)
    hits = 0
    for k, fs in enumerate(steps):
        if idle:
            got = g([None if f is None else _place(f, where) for f in fs])
            want = _scattered(lambda fr, c: mdet.run_batch(fr, c, pixel_format=fmt), fs, cams, lead)
        else:
            got = g(_place(fs, where))
            want = mdet.run_batch(fs, cams, pixel_format=fmt)
        hits += _check(k, got, want, lead)
    assert hits > STEPS // 2, hits


def test_a_call_is_frame_copies_and_one_graph_launch(cplib):
    """_launch_structure in a child process: torch.profiler initialises CUPTI for the rest of a process, and the tests
    of later files that count the profiler's copy records expect a process in which no earlier test profiled."""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "from tests.test_gpu_detect_graph import _launch_structure; _launch_structure()"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])


def _launch_structure():
    """The captured graphs hold kernels and memsets only; a call is one copy per live frame (plus the control block with
    idle slots) and one graph launch, with no kernel launch, memset or synchronisation from the host; an all-idle call
    launches nothing."""
    det = _detector()
    S = 2
    g = cpb.DetectGraph(det, slots=S, frame_hw=(H, W), camera_matrix=synth.default_camera(W, H), pixel_format="nv12")
    kinds = _node_types(g.graphs[0])
    assert set(kinds) <= {CU_GRAPH_NODE_TYPE_KERNEL, CU_GRAPH_NODE_TYPE_MEMSET, CU_GRAPH_NODE_TYPE_EMPTY}, kinds
    assert kinds[CU_GRAPH_NODE_TYPE_KERNEL] >= g.eng.forward_launches + 3          # the pre-process and the decode
    names, n = _profile_steps(g, [torch.from_numpy(f).pin_memory() for f in _video(S, "nv12", seed=400, steps=6)])
    assert names["cudaMemcpyAsync"] == n and names["cudaGraphLaunch"] == n, names
    assert names["cudaLaunchKernel"] == 0 and names["cudaMemsetAsync"] == 0
    assert names["cudaStreamSynchronize"] == 0 and names["cudaEventSynchronize"] == 0, names
    # with idle slots: one copy per live frame, one control copy and one launch; an all-idle call launches nothing
    ig = cpb.DetectGraph(det, slots=3, frame_hw=SIZES + [(512, 384)], camera_matrix=_slot_cameras(SIZES + [(512, 384)]),
                         idle_slots=True)
    for n_live, kd in enumerate((_node_types(x) for x in ig.graphs), 1):
        assert set(kd) <= {CU_GRAPH_NODE_TYPE_KERNEL, CU_GRAPH_NODE_TYPE_MEMSET, CU_GRAPH_NODE_TYPE_EMPTY}, (n_live, kd)
    video = _ragged_video(SIZES + [(512, 384)], "bgr", 410, steps=6)
    live = [{0, 1, 2}, {0, 2}, {1}, {0, 1}, {2}, {0, 1, 2}]
    steps = [[torch.from_numpy(f).pin_memory() if i in lv else None for i, f in enumerate(fs)]
             for fs, lv in zip(video, live)]
    names, n = _profile_steps(ig, steps)
    assert names["cudaMemcpyAsync"] == sum(len(lv) for lv in live[2:]) + n, names
    assert names["cudaGraphLaunch"] == n and names["cudaLaunchKernel"] == 0, names
    names, _ = _profile_steps(ig, [[None] * 3] * 4)
    assert names["cudaGraphLaunch"] == 0 and names["cudaMemcpyAsync"] == 0, names
    p, c = _host(ig([None] * 3))
    assert not p.any() and not c.any()
