"""TrackGraph on the device: 12-step synthetic videos through the captured step against run_batch(track=True)'s array
form on the same detector, every step's tracks and n_tracks bit for bit (1 and 8 slots, greedy and Hungarian
association, BGR and NV12 frames, host-pinned and device frames, a new video on one slot at step 5 and on every slot at
step 9, opt.empty_pre_hm); the same inputs replayed twice from a reset; the detector's own slot state untouched by the
graph; and a step that is two host-to-device copies and one graph launch of kernels and memsets only."""
import collections
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from tests.test_gpu_yuv_input import from_bgr

pytestmark = pytest.mark.gpu
STEPS = 12
H, W = 480, 640
NEW = {5: (0,), 9: "all"}          # step -> the slots that start a new video with that frame


def _detector(hungarian=False, empty_pre_hm=False):
    """A seeded tf32x3 tracking detector whose heat-map biases are calibrated to about 4 objects per frame."""
    opt = cpb.default_opt("dla_34", tracking_task=True)
    opt.hungarian, opt.empty_pre_hm = hungarian, empty_pre_hm
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    m.load_state_dict(synth.seeded_state_dict(m, seed=31, offset_std=0.3))
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, 512, 512, seed=5))).cuda()
    z = torch.zeros((2, 1, 512, 512), device="cuda")
    with torch.no_grad():
        synth.calibrate_head_bias(m, m(x, x, z, z.repeat(1, 8, 1, 1))[-1], target=4)
    det = cpb.ObjectPoseDetector(opt, model=m)
    assert det.model.precision == "tf32x3"
    return det


def _video(S, fmt, seed, steps=STEPS):
    """Per step the uint8 frames of S slots: a noise frame per slot, shifted a few pixels every step."""
    base = synth.synthetic_frames(S, H, W, seed=seed)
    out = []
    for k in range(steps):
        f = np.roll(base, (2 * k, 3 * k), axis=(1, 2))
        out.append(f if fmt == "bgr" else np.stack([from_bgr(g, fmt) for g in f]))
    return out


def _cameras(S):
    return np.stack([synth.default_camera(W + 16 * i, H + 8 * i) for i in range(S)])


def _new_video(k, S):
    slots = NEW.get(k)
    return None if slots is None else [slots == "all" or i in slots for i in range(S)]


def _reference_step(det, frames, cam, fmt, new):
    """run_batch(track=True)'s array form; a slot whose video starts is one that has not started in the detector's
    slot state (the rule run_batch applies to new_video in its list form)."""
    if new is not None:
        for i, n in enumerate(new):
            if n:
                det._slots.started[i] = False
    return det.run_batch(frames, cam, track=True, pixel_format=fmt)


def _host(pair):
    return pair[0].cpu().numpy(), pair[1].cpu().numpy()


CASES = [  # slots, hungarian, pixel format, where the frames are, opt.empty_pre_hm
    (1, False, "bgr", "pinned", False),
    (8, False, "nv12", "device", False),
    (8, True, "bgr", "device", False),
    (1, True, "nv12", "pinned", False),
    (8, False, "bgr", "pinned", True),
]


@pytest.mark.parametrize("S, hungarian, fmt, where, empty", CASES)
def test_graph_matches_run_batch(S, hungarian, fmt, where, empty, cplib):
    det = _detector(hungarian, empty)
    cam = _cameras(S)
    tg = cpb.TrackGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam, pixel_format=fmt)
    assert det._slots is None                          # building the graph leaves the detector's slot state alone
    total = 0
    for k, f in enumerate(_video(S, fmt, seed=70 + S)):
        src = torch.from_numpy(f).pin_memory() if where == "pinned" else torch.from_numpy(f).cuda()
        new = _new_video(k, S)
        gt, gn = _host(tg(src, new_video=new))
        # the same detector's run_batch, interleaved step by step with the graph: the two keep separate slot states
        wt, wn = _reference_step(det, f, cam, fmt, new)
        assert np.array_equal(gn, wn), (k, gn, wn)
        assert np.array_equal(gt, wt), (k, np.argwhere(gt != wt)[:8])
        total += int(wn.sum())
        if new is not None:                            # a new video numbers its tracks from 1 again
            for i in np.flatnonzero(new):
                assert gn[i] == 0 or gt[i, :gn[i], L.T_ID].min() == 1
    assert total > 0


def test_replay_is_stable_and_refusals(cplib):
    det = _detector()
    S = 2
    tg = cpb.TrackGraph(det, slots=S, frame_hw=(H, W), camera_matrix=synth.default_camera(W, H))
    vid = [torch.from_numpy(f).cuda() for f in _video(S, "bgr", seed=90, steps=6)]
    runs = []
    for _ in range(2):
        tg.reset()
        runs.append([_host(tg(f, new_video=_new_video(k, S))) for k, f in enumerate(vid)])
    assert sum(int(n.sum()) for _, n in runs[0]) > 0
    for (a_t, a_n), (b_t, b_n) in zip(*runs):
        assert np.array_equal(a_n, b_n) and np.array_equal(a_t, b_t)
    # what the fixed-shape form does not take
    with pytest.raises(NotImplementedError, match="pre_dets seeding runs through run_batch"):
        tg(vid[0], pre_dets=[[], []])
    with pytest.raises(ValueError, match=r"idle slots and mixed sizes run through run_batch\(list, track=True\)"):
        tg([vid[0][0], None])
    with pytest.raises(ValueError, match=r"frames must be uint8 \[2, 480, 640, 3\]"):
        tg(torch.zeros((2, 600, 800, 3), dtype=torch.uint8))
    with pytest.raises(ValueError, match="3 new_video entries for 2 slots"):
        tg(vid[0], new_video=[True, False, True])


def test_graph_leaves_the_detectors_slots_alone(cplib):
    """run_batch(track=True) steps, a TrackGraph built and stepped in between, then more run_batch steps: the same
    results as a detector that never saw the graph."""
    S, cam = 2, synth.default_camera(W, H)
    vid = _video(S, "bgr", seed=95, steps=4)
    ref = _detector()
    want = [ref.run_batch(f, cam, track=True) for f in vid]
    det = _detector()
    got = [det.run_batch(f, cam, track=True) for f in vid[:2]]
    slots = det._slots
    tg = cpb.TrackGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam)
    for f in vid[2:]:
        tg(f)
    assert det._slots is slots
    got += [det.run_batch(f, cam, track=True) for f in vid[2:]]
    for (gt, gn), (wt, wn) in zip(got, want):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt)


CU_GRAPH_NODE_TYPE_KERNEL, CU_GRAPH_NODE_TYPE_MEMSET, CU_GRAPH_NODE_TYPE_EMPTY = 0, 2, 5


def _node_types(graph):
    cu = ctypes.CDLL("libcuda.so.1")
    raw = ctypes.c_void_p(graph.raw_cuda_graph())
    n = ctypes.c_size_t(0)
    assert cu.cuGraphGetNodes(raw, None, ctypes.byref(n)) == 0
    nodes = (ctypes.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(raw, nodes, ctypes.byref(n)) == 0
    types = collections.Counter()
    for nd in nodes:
        t = ctypes.c_int(-1)
        assert cu.cuGraphNodeGetType(ctypes.c_void_p(nd), ctypes.byref(t)) == 0
        types[t.value] += 1
    return types


def test_a_step_is_two_copies_and_one_graph_launch(cplib):
    det = _detector(hungarian=True)
    S = 2
    tg = cpb.TrackGraph(det, slots=S, frame_hw=(H, W), camera_matrix=synth.default_camera(W, H))
    # the captured step: kernels and memsets (the render clears its maps), no copy, host callback or allocation
    kinds = [_node_types(g) for g in tg.graphs]
    assert kinds[0] == kinds[1]
    assert set(kinds[0]) <= {CU_GRAPH_NODE_TYPE_KERNEL, CU_GRAPH_NODE_TYPE_MEMSET, CU_GRAPH_NODE_TYPE_EMPTY}, kinds[0]
    # network + decode, then reset, pre-process, render, association and step
    assert kinds[0][CU_GRAPH_NODE_TYPE_KERNEL] >= tg.eng.forward_launches + 5
    vid = [torch.from_numpy(f).pin_memory() for f in _video(S, "bgr", seed=97, steps=6)]
    for f in vid[:2]:
        tg(f)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for f in vid[2:]:
            tg(f)
        torch.cuda.synchronize()
    names = collections.Counter(e.name for e in prof.events())
    steps = len(vid) - 2
    copies = {n: c for n, c in names.items() if n.startswith("Memcpy")}
    assert sum(copies.values()) == 2 * steps and all(n.startswith("Memcpy HtoD") for n in copies), copies
    assert names["cudaGraphLaunch"] == steps
    assert names["cudaLaunchKernel"] == 0 and names["cudaMemsetAsync"] == 0
    assert names["cudaStreamSynchronize"] == 0 and names["cudaEventSynchronize"] == 0, names
