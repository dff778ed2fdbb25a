"""Lens distortion fused into the pre-process against undistorting on the host: python scripts/undistort.py
[--cameras 1 8] [--steps 20] [--warmup 5] [--rounds 2]

1. The pre-process call alone on 32 device-resident 1920x1080 frames to a 512x512 input, in BGR and NV12: one frame
   table with each frame's fix_res affine against the same table with a plumb_bob coordinate map per frame, both
   launched through cp_preprocess_slots_ragged_dev (CUDA events, warmed up, `--reps` calls per measurement, the arms
   alternated, `--rounds` rounds).  The mapped table's output is checked against cp_preprocess_remap first.
2. DetectGraph steps at each of `--cameras` cameras of `--height` x `--width` BGR frames in pinned host memory, every
   camera with the same plumb_bob lens.  Two arms, alternated step by step, `--rounds` times:
     host-remap  cv2.remap of every frame at full resolution (fixed-point maps of cv2.initUndistortRectifyMap, built
                 once) into pinned BGR buffers, then a BGR graph with camera K_new
     fused       the raw frames go to a graph built with distortion= (the map read inside the pre-process)
   Per arm the median wall time of a step (a host clock around the host work and the call, ending in a device
   synchronise) over `--steps` steps after `--warmup`.  The fused arm's first step is checked against
   run_batch(..., distortion=) on the same frames (identical).  The arms resample differently (twice against once), so
   their records differ by design; the largest keypoint difference between records matched by nearest centre (within
   8 px) is printed for information only.

Seeded dla_34 weights (tf32x3) with heat-map biases calibrated to about 4 objects per frame.  The card name, power
limit and maximum SM clock are printed first, in the same run; they are part of the numbers.  Prints JSON lines.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import _lib as L  # noqa: E402
from centerpose_b200 import synth  # noqa: E402
from centerpose_b200.engine import _ptr, map_pointers  # noqa: E402
from centerpose_b200.lens import undistort_map  # noqa: E402
from scripts.camera_formats import encode  # noqa: E402
from scripts.yuv_input import gpu_state, make_detector  # noqa: E402

LENS = cpb.LensDistortion([-0.28, 0.07, 1e-3, -5e-4, -0.01])


def preprocess_calls(dev, args):
    B, h, w, ih, iw = 32, 1080, 1920, 512, 512
    opt = cpb.default_opt("dla_34")
    lib = L.load()
    K = synth.default_camera(w, h)
    mp = torch.from_numpy(undistort_map(LENS, K, (h, w), (ih, iw))).to(dev)
    base = synth.synthetic_frames(4, h, w, seed=900)
    m, s = (ctypes.c_float * 3)(*opt.mean), (ctypes.c_float * 3)(*opt.std)
    hw = np.array([(h, w)] * B, np.int32)
    out = torch.empty((B, 3, ih, iw), dtype=torch.float32, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    times = {}
    arms = []
    for fmt in ("bgr", "nv12"):
        frames = [encode(base[b % 4], fmt) for b in range(B)]
        offs = np.arange(B, dtype=np.int64) * frames[0].size
        buf = torch.from_numpy(np.concatenate([f.reshape(-1) for f in frames])).to(dev)
        code = L.PIXEL_FORMAT_CODES[fmt]
        p64, p32 = offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
        tables = {}
        for arm in ("affine", "map"):
            t = torch.zeros(int(lib.cp_preprocess_frame_table_bytes(B)), dtype=torch.uint8, device=dev)
            if arm == "affine":
                L.check(lib.cp_preprocess_frame_table(buf.numel(), p64, p32, code, B, ih, iw, None, _ptr(t), st), arm)
                tables[arm] = (t, code)
            else:
                L.check(lib.cp_preprocess_frame_table_maps(buf.numel(), p64, p32, code, None,
                                                           map_pointers([mp] * B, B, ih, iw, dev, "undistort"), B, ih,
                                                           iw, None, _ptr(t), st), arm)
                tables[arm] = (t, code | L.CP_PIX_REMAP)
        for arm, (t, c) in tables.items():
            def call(buf=buf, t=t, c=c):
                L.check(lib.cp_preprocess_slots_ragged_dev(_ptr(buf), _ptr(t), c, B, ih, iw, m, s, None, _ptr(out), None,
                                                           st), "cp_preprocess_slots_ragged_dev")
            arms.append(("%s %s" % (fmt, arm), call))
        arms[-1][1]()
        want = cpb.preprocess_remap(buf, offs, hw, fmt, [mp] * B, ih, iw, opt.mean, opt.std)
        assert torch.equal(out, want), fmt
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, call in arms:
            for _ in range(5):
                call()
            e0.record()
            for _ in range(args.reps):
                call()
            e1.record()
            torch.cuda.synchronize()
            times.setdefault(name, []).append(e0.elapsed_time(e1) / args.reps * 1e3)
    for name, us in times.items():
        print(json.dumps({"preprocess_call": name, "frames": B, "src": "%dx%d" % (w, h), "dst": "%dx%d" % (iw, ih),
                          "us_per_call": [round(v, 1) for v in us]}))


def _kps_diff(a, b, radius=8.0):
    """Largest |keypoint difference| in px between each record of a and the record of b with the nearest centre, over
    pairs whose centres are within `radius` px (information only)."""
    (pa, na), (pb, nb) = a, b
    worst = 0.0
    for i in range(na.shape[0]):
        ca, cb = pa[i, :na[i], L.P_CT:L.P_CT + 2], pb[i, :nb[i], L.P_CT:L.P_CT + 2]
        if len(ca) and len(cb):
            d = np.linalg.norm(ca[:, None] - cb[None], axis=-1)
            for r, j in enumerate(d.argmin(1)):
                if d[r, j] <= radius:
                    kd = np.abs(pa[i, r, L.P_KPS:L.P_KPS + 16] - pb[i, j, L.P_KPS:L.P_KPS + 16]).max()
                    worst = max(worst, float(kd))
    return worst


def graph_steps(dev, S, args):
    import cv2
    h, w = args.height, args.width
    det = make_detector(dev, tracking=False)
    K = synth.default_camera(w, h)
    Kn = LENS.camera(K)
    fused = cpb.DetectGraph(det, slots=S, frame_hw=(h, w), camera_matrix=K, distortion=LENS)
    host = cpb.DetectGraph(det, slots=S, frame_hw=(h, w), camera_matrix=Kn)
    m1, m2 = cv2.initUndistortRectifyMap(K, LENS.coeffs, None, Kn, (w, h), cv2.CV_16SC2)
    pool = synth.synthetic_frames(4, h, w, seed=700)
    src = [torch.from_numpy(np.stack([pool[(t + s) % 4] for s in range(S)])).pin_memory() for t in range(4)]
    bgr = [torch.empty((S, h, w, 3), dtype=torch.uint8).pin_memory() for _ in range(2)]
    # run_batch on a detector whose plan holds S frames, as the graph's (split-K follows the plan's capacity)
    model = cpb.create_model(det.opt.arch, det.opt.heads, det.opt.head_conv, det.opt)
    model.load_state_dict(det.model.state_dict())
    want = cpb.ObjectPoseDetector(det.opt, model=model).run_batch(src[0], K, distortion=LENS)
    got = fused(src[0])
    torch.cuda.synchronize()
    assert all(np.array_equal(x.cpu().numpy(), y) for x, y in zip(got, want)), S
    times, worst = {"host-remap": [], "fused": []}, 0.0
    for _ in range(args.rounds):
        for t in range(args.steps + args.warmup):
            frames = src[t % 4]
            t0 = time.perf_counter()
            got = fused(frames)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            got = [x.cpu().numpy() for x in got]
            t2 = time.perf_counter()
            dst = bgr[t % 2]
            for i in range(S):
                cv2.remap(frames[i].numpy(), m1, m2, cv2.INTER_LINEAR, dst=dst[i].numpy(),
                          borderMode=cv2.BORDER_CONSTANT, borderValue=0)
            ref = host(dst)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
            worst = max(worst, _kps_diff(got, [x.cpu().numpy() for x in ref]))
            if t >= args.warmup:
                times["fused"].append((t1 - t0) * 1e3)
                times["host-remap"].append((t3 - t2) * 1e3)
    for arm, ms in times.items():
        print(json.dumps({"graph": "detect", "cameras": S, "frame": "%dx%d" % (w, h), "arm": arm,
                          "median_ms": round(float(np.median(ms)), 3), "mean_ms": round(float(np.mean(ms)), 3),
                          "steps": len(ms)}))
    print(json.dumps({"graph": "detect", "cameras": S, "fused_equals_run_batch": True,
                      "max_kps_diff_px_between_arms": round(worst, 3)}))
    del fused, host, det, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("undistort.py measures on a CUDA device; none is available")
    import cv2
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_state(), "cv2_threads": cv2.getNumThreads(), "host_cpus": os.cpu_count()}))
    preprocess_calls(dev, args)
    for S in args.cameras:
        graph_steps(dev, S, args)


if __name__ == "__main__":
    main()
