"""Ragged batches and per-stream tracking without a GPU: the new entry points are declared, exported and bound; bad
stream maps and ragged frame layouts are refused with CP_ERR_INVALID before any device work; the host-side argument
checks of run_batch(list); and the layout of the per-frame track-record all-gather, round-tripped under gloo."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from centerpose_b200 import _lib
from centerpose_b200.detector import camera_per_frame, check_frames, check_slot_list
from centerpose_b200.dist import PoseBuffer, shard_range, slot_layout
from tests.test_abi import _declared_symbols

NEW = ("cp_preprocess_ragged", "cp_tracker_step_ex", "cp_tracker_render_ex2", "cp_tracker_seed_ex")


def _ids(*v):
    return (ctypes.c_int32 * len(v))(*v)


def test_new_symbols_declared_exported_and_bound(cplib):
    for s in NEW:
        assert s in _declared_symbols() and s in _lib.EXPORTS and hasattr(cplib, s)
    assert cplib.cp_version() == 1


@pytest.mark.parametrize("ids, msg", [((0, 0), b"duplicate stream id 0"), ((1, 2, 1), b"duplicate stream id 1"),
                                      ((0, -1), b"stream id -1 out of range")])
def test_bad_stream_maps_are_refused(cplib, ids, msg):
    B = len(ids)
    rc = cplib.cp_tracker_step_ex(None, B, _ids(*ids), None, None, 100, None, None, None, None)
    assert rc == -1 and msg in cplib.cp_last_error() and b"cp_tracker_step" in cplib.cp_last_error()
    rc = cplib.cp_tracker_render_ex2(None, B, _ids(*ids), None, None, 8, 8, None, None, None, None)
    assert rc == -1 and msg in cplib.cp_last_error() and b"cp_tracker_render" in cplib.cp_last_error()
    rc = cplib.cp_tracker_seed_ex(None, B, _ids(*ids), None, None, 1, None)
    assert rc == -1 and msg in cplib.cp_last_error() and b"cp_tracker_seed" in cplib.cp_last_error()


def test_identity_map_passes_the_map_check(cplib):
    # a valid map gets as far as the null-tracker check
    rc = cplib.cp_tracker_step_ex(None, 3, _ids(2, 0, 1), None, None, 100, None, None, None, None)
    assert rc == -1 and b"null argument" in cplib.cp_last_error()


def _ragged(cplib, offsets, hw, nbytes, frames=1, out=1, trans=None):
    offs = np.asarray(offsets, np.int64)
    hw = np.asarray(hw, np.int32).reshape(-1, 2)
    m = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
    s = (ctypes.c_float * 3)(0.3, 0.3, 0.3)
    return cplib.cp_preprocess_ragged(ctypes.c_void_p(frames), nbytes, offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                      hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), ctypes.c_void_p(out), len(offs),
                                      64, 64, trans, m, s, None)


def test_ragged_preprocess_validates_the_layout(cplib):
    assert _ragged(cplib, [0], [[10, 10]], 300, out=0) == -1 and b"null argument" in cplib.cp_last_error()
    assert _ragged(cplib, [0, 300], [[10, 10], [10, 10]], 599) == -1
    assert b"frame 1 (10 x 10 at byte 300) lies outside the 599-byte buffer" in cplib.cp_last_error()
    assert _ragged(cplib, [-3], [[10, 10]], 300) == -1 and b"outside" in cplib.cp_last_error()
    assert _ragged(cplib, [0, 0], [[10, 10], [0, 4]], 300) == -1 and b"frame 1 has size 0 x 4" in cplib.cp_last_error()


def test_ragged_frame_checks():
    ok = np.zeros((4, 6, 3), np.uint8)
    check_frames([ok, torch.zeros((5, 3, 3), dtype=torch.uint8)], allow_idle=False)
    check_frames([ok, None], allow_idle=True)
    with pytest.raises(ValueError, match="idle"):
        check_frames([ok, None], allow_idle=False)
    with pytest.raises(TypeError, match="uint8"):
        check_frames([ok.astype(np.float32)], allow_idle=False)
    with pytest.raises(TypeError, match="uint8"):
        check_frames([torch.zeros((4, 6, 3))], allow_idle=False)
    with pytest.raises(ValueError, match=r"\[H,W,3\]"):
        check_frames([np.zeros((4, 6, 4), np.uint8)], allow_idle=False)
    with pytest.raises(ValueError, match="empty"):
        check_frames([], allow_idle=True)
    with pytest.raises(ValueError, match="2 new_video entries for 3 slots"):
        check_slot_list([True, False], 3, "new_video", bool)
    assert check_slot_list(None, 3, "pre_dets") is None
    cam = np.eye(3)
    assert len(camera_per_frame(cam, 4)) == 4
    assert np.array_equal(camera_per_frame(np.stack([cam * 2, cam]), 2)[0], cam * 2)
    with pytest.raises(ValueError, match="one \\[3,3\\] per frame"):
        camera_per_frame(np.stack([cam] * 3), 2)


def test_stream_map_length_is_checked():
    from centerpose_b200.tracker import _stream_map
    assert _stream_map(None, 4) is None
    assert list(_stream_map([3, 1], 2)) == [3, 1]
    with pytest.raises(ValueError, match="3 stream ids for a batch of 2"):
        _stream_map([0, 1, 2], 2)


def test_slot_layout_covers_every_slot_once():
    for slots in (1, 5, 8, 32):
        for world in (1, 2, 3, 4):
            b, order = slot_layout(slots, world)
            assert len(order) == slots and len(set(order)) == slots and max(order) < world * b
            for r in range(world):
                lo, hi = shard_range(slots, r, world)
                assert order[lo:hi] == list(range(r * b, r * b + hi - lo))


def _worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        S, T, R = 5, 16, _lib.CP_TRACK_RECORD
        b, order = slot_layout(S, world)
        lo, hi = shard_range(S, rank, world)
        g = torch.Generator().manual_seed(0)
        full = torch.randn(S, T, R, generator=g)
        nt = torch.arange(3, 3 + S, dtype=torch.int32)
        buf = PoseBuffer(b, T, "cpu", world=world, R=R, pin=False)
        buf.poses[:hi - lo].copy_(full[lo:hi])
        buf.n_valid[:hi - lo].copy_(nt[lo:hi])
        buf.all_gather()
        buf.to_host()
        hp, hn = buf.host_views()
        ok = np.array_equal(hp[order], full.numpy()) and hn[order].tolist() == nt.tolist()
        dp, dn = buf.views(buf.gathered)
        ok = ok and torch.equal(dp[order], full) and torch.equal(dn[order], nt)
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


def test_track_gather_world2_gloo():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=True)
    assert ret[0] and ret[1]
