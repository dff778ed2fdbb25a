"""TrackGraph and MultiCategoryTrackGraph built with idle_slots=True, on the device.  Every case runs a scripted 12-step
schedule of 4 slots through the graph and through run_batch(list, track=True) of a detector whose slot state starts
fresh (MultiCategoryTracker.run_batch(list) for several categories), and checks every step's tracks and n_tracks bit for
bit.  The schedule has a slot that starts late, one that pauses and resumes (its previous frame is then its last live
frame), one that ends, new_video on a live slot and on an idle slot, an all-idle step and every live count 0..4.

  * one frame_hw and one per slot, BGR and NV12, greedy and Hungarian association, opt.empty_pre_hm, pinned and device
    frames, and M = 2 categories;
  * the schedule replayed twice after reset() gives the same steps, and the detector's slot state is left alone;
  * cp_preprocess_slots_rows_dev alone against cp_preprocess_ragged / cp_preprocess_yuv420 on the mapped frames, with
    the store / prev exchange with and without start flags, and cp_gather_rows_dev with -1 entries;
  * every captured graph holds kernels and memsets only; a step of L live slots is L frame copies, one control copy and
    one graph launch, and an all-idle call launches no graph."""
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
                                        H, W, _detector, _host, _node_types)
from tests.test_gpu_track_graph_multi import (SIZES, _check_step, _place, _profile_steps, _ragged_video,
                                              _slot_cameras, _tracker, checkpoints)  # noqa: F401 (a fixture)
from tests.test_gpu_yuv_input import from_bgr

pytestmark = pytest.mark.gpu
S = 4
# per step: the live slots, and new_video (None or one flag per slot)
SCHEDULE = [
    ({0, 2, 3}, None),                      # slot 1 starts late
    ({0, 2}, None),
    ({0, 1, 2, 3}, None),                   # slot 1's first frame
    ({1, 2}, None),                         # slot 0 pauses ...
    ({2}, None),
    ({0, 1, 2, 3}, None),                   # ... and resumes from its frame of step 2
    (set(), None),                          # every slot idle
    ({0, 1, 2}, [True, False, False, True]),  # a new video on live slot 0; slot 3 is idle, so its flag is ignored
    ({0, 1, 3}, None),                      # slot 2 has ended
    ({0, 1}, None),
    ({1, 3}, [False, False, False, True]),
    ({0, 1, 3}, None),
]
ONE = [(H, W)] * S
PER_SLOT = [SIZES[0], SIZES[1], SIZES[2], (512, 384)]


def test_the_schedule_covers_what_it_must():
    counts = {len(live) for live, _ in SCHEDULE}
    assert counts == set(range(S + 1))
    first = [min(k for k, (live, _) in enumerate(SCHEDULE) if i in live) for i in range(S)]
    assert max(first) > 0                                          # a late start
    last = [max(k for k, (live, _) in enumerate(SCHEDULE) if i in live) for i in range(S)]
    assert min(last) < len(SCHEDULE) - 3                           # a slot that ends
    assert any(new is not None and any(new[i] for i in live) for live, new in SCHEDULE)
    assert any(new is not None and any(new[i] for i in range(S) if i not in live) for live, new in SCHEDULE)


def _steps(sizes, fmt, seed):
    """Per step the list of S entries: the slot's frame, or None when it is idle."""
    video = _ragged_video(sizes, fmt, seed, steps=len(SCHEDULE))
    return [[f if i in live else None for i, f in enumerate(fs)] for fs, (live, _) in zip(video, SCHEDULE)]


def _graph_input(fs, where, sizes, array_when_full):
    """The graph's argument: the frames placed on the host (pinned) or the device; an all-live step of one frame size is
    passed as one [S, ...] array when array_when_full."""
    if array_when_full and all(f is not None for f in fs) and len(set(sizes)) == 1:
        return _place(np.stack(fs), where)
    return [None if f is None else _place(f, where) for f in fs]


CASES = [  # frame sizes, pixel format, hungarian, where the frames are, opt.empty_pre_hm
    ("one", "bgr", False, "pinned", False),
    ("one", "nv12", True, "device", False),
    ("per-slot", "bgr", True, "device", False),
    ("per-slot", "nv12", False, "pinned", True),
]


@pytest.mark.parametrize("kind, fmt, hungarian, where, empty", CASES)
def test_idle_graph_matches_run_batch_list(kind, fmt, hungarian, where, empty, cplib):
    det = _detector(hungarian, empty)
    sizes = ONE if kind == "one" else PER_SLOT
    cams = _slot_cameras(sizes)
    tg = cpb.TrackGraph(det, slots=S, frame_hw=sizes[0] if kind == "one" else sizes, camera_matrix=cams,
                        pixel_format=fmt, idle_slots=True)
    assert det._slots is None and len(tg.graphs) == S
    total = 0
    for k, fs in enumerate(_steps(sizes, fmt, seed=800)):
        new = SCHEDULE[k][1]
        got = tg(_graph_input(fs, where, sizes, array_when_full=kind == "one"), new_video=new)
        want = det.run_batch(fs, cams, track=True, new_video=new, pixel_format=fmt)
        total += _check_step(k, got, want, None, (S,))
        for i in range(S):
            if fs[i] is None:
                assert want[1][i] == 0 and not want[0][i].any()
    assert total > 0


def test_multi_category_idle_graph_matches_run_batch_list(checkpoints, cplib):  # noqa: F811
    trk = _tracker(checkpoints, cats=("chair", "cup"), hungarian=True)
    cams = _slot_cameras(ONE)
    tg = cpb.MultiCategoryTrackGraph(trk, slots=S, frame_hw=(H, W), camera_matrix=cams, idle_slots=True)
    assert trk._slots is None
    total = 0
    for k, fs in enumerate(_steps(ONE, "bgr", seed=820)):
        new = SCHEDULE[k][1]
        got = tg(_graph_input(fs, "pinned", ONE, array_when_full=False), new_video=new)
        total += _check_step(k, got, trk.run_batch(fs, cams, new_video=new), None, (2, S))
    assert total > 0


def test_replay_after_reset_and_the_detectors_slots(cplib):
    """The schedule twice from reset() gives the same steps; run_batch(track=True) steps around the graph give what a
    detector that never saw the graph gives."""
    cam = _slot_cameras(ONE)
    ref = _detector()
    pre = _steps(ONE, "bgr", seed=840)[:2]
    want = [ref.run_batch(fs, cam, track=True) for fs in pre]
    det = _detector()
    got = [det.run_batch(pre[0], cam, track=True)]
    slots = det._slots
    tg = cpb.TrackGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam, idle_slots=True)
    runs = []
    for _ in range(2):
        tg.reset()
        runs.append([_host(tg([None if f is None else _place(f, "device") for f in fs], new_video=SCHEDULE[k][1]))
                     for k, fs in enumerate(_steps(ONE, "bgr", seed=850))])
    assert sum(int(n.sum()) for _, n in runs[0]) > 0
    for (a_t, a_n), (b_t, b_n) in zip(*runs):
        assert np.array_equal(a_n, b_n) and np.array_equal(a_t, b_t)
    assert det._slots is slots
    got.append(det.run_batch(pre[1], cam, track=True))
    for (gt, gn), (wt, wn) in zip(got, want):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt)
    # what the graph still does not take
    with pytest.raises(NotImplementedError, match="pre_dets seeding runs through run_batch"):
        tg([None] * S, pre_dets=[[]] * S)


# ---- the kernels alone -------------------------------------------------------------------------------------------------
def _packed(frames):
    offs, o = [], 3                                    # odd byte offsets, a gap between frames
    for f in frames:
        offs.append(o)
        o += f.size + 5
    packed = torch.zeros(o, dtype=torch.uint8)
    for f, off in zip(frames, offs):
        packed[off:off + f.size] = torch.from_numpy(f.reshape(-1))
    return packed.cuda(), np.array(offs, np.int64)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("fmt", ["bgr", "nv12"])
def test_rows_kernel_matches_the_ragged_calls_and_exchanges_prev(fmt, cplib):
    sizes = [(481, 641), (720, 1280), (512, 512), (300, 200), (1440, 1080)] if fmt == "bgr" else \
        [(480, 640), (720, 1280), (512, 512), (300, 200), (1440, 1080)]
    frames = [synth.synthetic_frames(1, h, w, seed=900 + i)[0] for i, (h, w) in enumerate(sizes)]
    frames = frames if fmt == "bgr" else [from_bgr(f, fmt) for f in frames]
    NS, ih, iw = len(frames), 256, 384
    packed, offs = _packed(frames)
    hw = np.array(sizes, np.int32)
    trans = np.stack([affine_from_center_scale(np.array([w / 2., h / 2.], np.float32), float(max(h, w)), iw, ih)
                      for h, w in sizes])
    trans[1, 0, 1] += 0.05
    mean, std = (0.408, 0.447, 0.470), (0.289, 0.274, 0.278)
    fcode = {"bgr": L.CP_PIX_BGR, "nv12": L.CP_PIX_NV12}[fmt]
    table = torch.zeros(int(cplib.cp_preprocess_frame_table_bytes(NS)), dtype=torch.uint8, device="cuda")
    tr = np.ascontiguousarray(trans, np.float64)
    L.check(cplib.cp_preprocess_frame_table(packed.numel(), offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                            hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), fcode, NS, ih, iw,
                                            tr.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), _p(table), None),
            "cp_preprocess_frame_table")
    rows = [3, 0, 4]                                   # live rows in any order, slots 1 and 2 idle
    sel = np.array(rows)
    if fmt == "bgr":
        want = preprocess_ragged(packed, offs[sel], hw[sel], ih, iw, mean, std, trans_input=trans[sel])
    else:
        want = preprocess_yuv420(packed, offs[sel], hw[sel], fmt, ih, iw, mean, std, trans_input=trans[sel])
    m, s = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rows_d = torch.tensor(rows, dtype=torch.int32, device="cuda")
    B = len(rows)

    def run(start, store, prev):
        out = torch.full((B, 3, ih, iw), float("nan"), device="cuda")
        L.check(cplib.cp_preprocess_slots_rows_dev(_p(packed), _p(table), fcode, _p(rows_d), B, ih, iw, m, s, _p(start),
                                                   _p(store), _p(out), _p(prev), st), "cp_preprocess_slots_rows_dev")
        return out
    assert torch.equal(run(None, None, None), want)     # without the exchange: the ragged pre-process of the rows
    old = torch.randn((NS, 3, ih, iw), device="cuda")
    for start in (None, torch.tensor([1, 0, 0, 1, 0], dtype=torch.int32, device="cuda")):
        store, prev = old.clone(), torch.full((B, 3, ih, iw), float("nan"), device="cuda")
        assert torch.equal(run(start, store, prev), want)
        for k, slot in enumerate(rows):
            starts = start is not None and bool(start[slot])
            assert torch.equal(prev[k], want[k] if starts else old[slot]), (k, slot)
            assert torch.equal(store[slot], want[k]), slot
        for slot in (1, 2):                            # idle slots keep their stored frame
            assert torch.equal(store[slot], old[slot]), slot


def test_gather_rows(cplib):
    src = torch.randn((6, 37), dtype=torch.float64, device="cuda")
    m = torch.tensor([5, -1, 0, 2, -1], dtype=torch.int32, device="cuda")
    dst = torch.full((5, 37), float("nan"), dtype=torch.float64, device="cuda")
    L.check(cplib.cp_gather_rows_dev(_p(src), _p(dst), 37 * 8, 5, _p(m), None), "cp_gather_rows_dev")
    torch.cuda.synchronize()
    for i, r in enumerate(m.tolist()):
        assert torch.equal(dst[i], src[r] if r >= 0 else torch.zeros_like(src[0])), i
    one = torch.arange(4, dtype=torch.int32, device="cuda") + 7             # 4-byte rows
    got = torch.full((3,), -5, dtype=torch.int32, device="cuda")
    L.check(cplib.cp_gather_rows_dev(_p(one), _p(got), 4, 3, _p(torch.tensor([-1, 3, 1], dtype=torch.int32,
                                                                               device="cuda")), None), "gather")
    assert got.tolist() == [0, 10, 8]


# ---- graph structure ---------------------------------------------------------------------------------------------------
def test_a_step_is_live_frame_copies_a_control_copy_and_one_graph_launch(cplib):
    tg = cpb.TrackGraph(_detector(hungarian=True), slots=S, frame_hw=PER_SLOT, camera_matrix=_slot_cameras(PER_SLOT),
                        pixel_format="nv12", idle_slots=True)
    kinds = [_node_types(g) for g in tg.graphs]
    for n, kd in enumerate(kinds, 1):
        assert set(kd) <= {CU_GRAPH_NODE_TYPE_KERNEL, CU_GRAPH_NODE_TYPE_MEMSET, CU_GRAPH_NODE_TYPE_EMPTY}, (n, kd)
        # network + decode, then reset, pre-process, three gathers, render, association, step and two scatters
        assert kd[CU_GRAPH_NODE_TYPE_KERNEL] >= tg.eng.forward_launches + 10, (n, kd)
    video = _ragged_video(PER_SLOT, "nv12", 860, steps=6)
    live = [{0, 1, 2, 3}, {0, 2}, {1}, {0, 1, 3}, {2, 3}, {0}]
    steps = [[torch.from_numpy(f).pin_memory() if i in lv else None for i, f in enumerate(fs)]
             for fs, lv in zip(video, live)]
    names, n = _profile_steps(tg, steps)
    frames = sum(len(lv) for lv in live[2:])
    assert names["cudaMemcpyAsync"] == frames + n, names
    assert names["cudaGraphLaunch"] == n
    assert names["cudaLaunchKernel"] == 0 and names["cudaMemsetAsync"] == 0
    assert names["cudaStreamSynchronize"] == 0 and names["cudaEventSynchronize"] == 0, names
    # an all-idle call: zeros, and no graph
    names, n = _profile_steps(tg, [[None] * S] * 4)
    assert names["cudaGraphLaunch"] == 0 and names["cudaMemcpyAsync"] == 0, names
    t, c = _host(tg([None] * S))
    assert not t.any() and not c.any()
