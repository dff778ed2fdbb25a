"""MJPEG cameras in the live-video graphs: python scripts/mjpeg_graph.py [--cameras 1 8] [--sizes 720x1280 1080x1920]

1. The decode alone, 1 and 8 frames: cp_jpeg_decode (host-driven synchronisation rounds, a fresh workspace per call as
   run_batch makes it) against cp_jpeg_decode_slots_dev (one chained synchronisation launch), CUDA events around
   `--reps` calls after 5 warm-up calls, alternated, `--rounds` rounds.  Both outputs are checked against cv2 first.
2. DetectGraph and TrackGraph steps at each size and camera count, 4:2:2 quality-85 frames (the common UVC layout) in
   pinned host memory.  Arms, their order rotated every step:
     host-imdecode  cv2.imdecode on a thread pool into pinned BGR buffers, then the BGR graph
     run_batch      run_batch(list, pixel_format="jpeg") (track=True for tracking)
     mjpeg          the graph built with pixel_format="mjpeg" (max_frame_bytes at its default, H * W * 3)
     mjpeg-1MB      the same with max_frame_bytes=1 MB
   Every arm's outputs are compared with the mjpeg arm's at every step (they must be identical).  Per arm the median
   and mean wall time of a step (a host clock around the call, ending in a device synchronise) over `--steps` steps
   after `--warmup`, for each of `--rounds` rounds, and the device memory each graph took to build.

Seeded dla_34 weights (tf32x3) with heat-map biases calibrated to about 4 objects per frame.  The card name, power
limit and maximum SM clock are printed first, in the same run; they are part of the numbers.  Prints JSON lines.
"""
import argparse
import ctypes
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import _lib, synth  # noqa: E402
from centerpose_b200.engine import jpeg_decode, jpeg_parse  # noqa: E402
from scripts.yuv_input import gpu_state, make_detector  # noqa: E402
from tests import jpeg_craft as jc  # noqa: E402


def encoded(h, w, n, seed):
    """n camera-like frames: the photographs of tests/data resized to h x w and shifted, 4:2:2 at quality 85.  (Noise
    frames would be about 2 MB at 1080p, far above what a webcam sends, and decode unlike camera content.)"""
    import cv2
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "data")
    base = [cv2.resize(cv2.imread(os.path.join(root, "frame_%d.png" % k)), (w, h)) for k in range(2)]
    return [jc.encode(np.roll(base[(seed + i) % 2], (4 * i, 6 * i), axis=(0, 1)), "422", 85) for i in range(n)]


def decode_alone(dev, h, w, args):
    import cv2
    L = _lib.load()
    p32, p64 = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
    for B in (1, 8):
        files = encoded(h, w, B, seed=40 + B)
        hs = [jpeg_parse(np.frombuffer(f, np.uint8)) for f in files]
        boffs = np.cumsum([0] + [len(f) for f in files[:-1]]).astype(np.int64)
        src = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to(dev)
        oo = np.arange(B, dtype=np.int64) * h * w * 3
        out = torch.empty((B * h * w * 3,), dtype=torch.uint8, device=dev)
        # the slot form: slot s's bytes at the prefix sum of max_bytes, here the default H * W * 3
        hw = np.array([(h, w)] * B, np.int32)
        mb = np.full(B, h * w * 3, np.int64)
        sbytes = torch.zeros((int(mb.sum()),), dtype=torch.uint8, device=dev)
        for s, f in enumerate(files):
            sbytes[s * h * w * 3:s * h * w * 3 + len(f)].copy_(torch.from_numpy(np.frombuffer(f, np.uint8).copy()))
        host = np.zeros(L.cp_jpeg_slots_block_bytes(B), np.uint8)
        _lib.check(L.cp_jpeg_slots_prepare(B, hw.ctypes.data_as(p32), mb.ctypes.data_as(p64), 0,
                                           (_lib.CpJpegHeader * B)(*hs),
                                           np.array([len(f) for f in files], np.int64).ctypes.data_as(p64),
                                           oo.ctypes.data_as(p64), host.ctypes.data_as(ctypes.c_void_p)), "prepare")
        block = torch.from_numpy(host).to(dev)
        ws = torch.empty((L.cp_jpeg_slots_workspace_bytes(B, hw.ctypes.data_as(p32), mb.ctypes.data_as(p64), 0),),
                         dtype=torch.uint8, device=dev)
        err = torch.zeros((B,), dtype=torch.int32, device=dev)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

        def host_driven():
            jpeg_decode(hs, src, boffs, out, oo)

        def slots():
            _lib.check(L.cp_jpeg_decode_slots_dev(ctypes.c_void_p(block.data_ptr()), B, hw.ctypes.data_as(p32),
                                                  mb.ctypes.data_as(p64), 0, ctypes.c_void_p(sbytes.data_ptr()),
                                                  ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(ws.data_ptr()),
                                                  ctypes.c_size_t(ws.numel()), ctypes.c_void_p(err.data_ptr()), stream),
                       "cp_jpeg_decode_slots_dev")

        arms = {"cp_jpeg_decode": host_driven, "slot_decode": slots}
        want = np.stack([cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR) for f in files])
        for a, call in arms.items():
            out.zero_()
            call()
            assert np.array_equal(out.cpu().numpy().reshape(want.shape), want), a
        times = {a: [] for a in arms}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for a, call in arms.items():
                for _ in range(5):
                    call()
                e0.record()
                for _ in range(args.reps):
                    call()
                e1.record()
                torch.cuda.synchronize()
                times[a].append(e0.elapsed_time(e1) / args.reps * 1e3)
        for a, us in times.items():
            print(json.dumps({"decode_alone": a, "frames": B, "frame": "%dx%d" % (w, h), "sampling": "422",
                              "quality": 85, "mean_bytes": int(np.mean([len(f) for f in files])),
                              "us_per_call": [round(v, 1) for v in us]}))


def built(make):
    """A graph and the device memory its building took."""
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    g = make()
    torch.cuda.synchronize()
    return g, torch.cuda.memory_allocated() - m0


def graph_steps(dev, kind, S, h, w, pool, args):
    import cv2
    det = make_detector(dev, tracking=kind == "track")
    cls = cpb.TrackGraph if kind == "track" else cpb.DetectGraph
    cam = synth.default_camera(w, h)
    gbgr, mem_bgr = built(lambda: cls(det, slots=S, frame_hw=(h, w), camera_matrix=cam))
    gmj, mem_mj = built(lambda: cls(det, slots=S, frame_hw=(h, w), camera_matrix=cam, pixel_format="mjpeg"))
    gmj1, mem_mj1 = built(lambda: cls(det, slots=S, frame_hw=(h, w), camera_matrix=cam, pixel_format="mjpeg",
                                      max_frame_bytes=1 << 20))
    files = encoded(h, w, 4, seed=700)
    src = [[torch.from_numpy(np.frombuffer(files[(t + s) % 4], np.uint8).copy()).pin_memory() for s in range(S)]
           for t in range(4)]
    bgr = [torch.empty((S, h, w, 3), dtype=torch.uint8).pin_memory() for _ in range(2)]
    cams = np.stack([cam] * S)
    track = {"track": True} if kind == "track" else {}

    def timed(call):
        t0 = time.perf_counter()
        out = call()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        return dt, [x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x) for x in out]

    def host_imdecode(frames, t):
        dst = bgr[t % 2]

        def one(s):
            dst[s].numpy()[...] = cv2.imdecode(frames[s].numpy(), cv2.IMREAD_COLOR)
        list(pool.map(one, range(S)))
        return gbgr(dst)

    arms = {"host-imdecode": host_imdecode,
            "run_batch": lambda frames, t: det.run_batch(list(frames), cams, pixel_format="jpeg", **track),
            "mjpeg": lambda frames, t: gmj(frames),
            "mjpeg-1MB": lambda frames, t: gmj1(frames)}
    names = list(arms)
    same_rb = True
    for r in range(args.rounds):
        times = {a: [] for a in arms}
        for t in range(args.warmup + args.steps):
            frames = src[t % 4]
            order = names[t % len(names):] + names[:t % len(names)]
            outs = {}
            for a in order:
                dt, outs[a] = timed(lambda: arms[a](frames, t))
                if t >= args.warmup:
                    times[a].append(dt * 1e3)
            # the graphs must agree bit for bit; run_batch's plan may hold more frames than S (the calibration
            # made one of 8), and the split-K choice follows a plan's capacity, so its agreement is reported
            for a in ("host-imdecode", "mjpeg-1MB"):
                assert all(np.array_equal(x, y) for x, y in zip(outs[a], outs["mjpeg"])), (kind, S, t, a)
            same_rb &= all(np.array_equal(x, y) for x, y in zip(outs["run_batch"], outs["mjpeg"]))
        for a, ms in times.items():
            print(json.dumps({"graph": kind, "cameras": S, "frame": "%dx%d" % (w, h), "sampling": "422",
                              "quality": 85, "round": r, "arm": a, "median_ms": round(float(np.median(ms)), 3),
                              "mean_ms": round(float(np.mean(ms)), 3), "steps": len(ms), "graphs_identical": True,
                              "run_batch_identical": same_rb}))
    print(json.dumps({"graph": kind, "cameras": S, "frame": "%dx%d" % (w, h), "graph_bytes": {
        "bgr": mem_bgr, "mjpeg": mem_mj, "mjpeg-1MB": mem_mj1}}))
    del gbgr, gmj, gmj1, det
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--sizes", nargs="+", default=["720x1280", "1080x1920"])
    ap.add_argument("--kinds", nargs="+", default=["detect", "track"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--threads", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mjpeg_graph.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_state(), "host_cpus": os.cpu_count(), "imdecode_threads": args.threads}))
    sizes = [tuple(int(v) for v in s.split("x")) for s in args.sizes]
    for h, w in sizes:
        decode_alone(dev, h, w, args)
    with ThreadPoolExecutor(args.threads) as pool:
        for kind in args.kinds:
            for h, w in sizes:
                for S in args.cameras:
                    graph_steps(dev, kind, S, h, w, pool, args)


if __name__ == "__main__":
    main()
