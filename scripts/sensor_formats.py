"""Sensor formats against host conversion: python scripts/sensor_formats.py [--cameras 1 8] [--steps 20]

1. The pre-process call alone, per format, on 32 device-resident 1920x1200 frames to a 512x512 input (CUDA events,
   5 warm-up calls, `--reps` calls per measurement, the formats alternated, `--rounds` rounds): BGR through
   cp_preprocess_ragged, each Bayer pattern and "gray" through cp_preprocess_formats.  Every arm's output is checked
   against the BGR call on the cv2.cvtColor-converted frames first.
2. DetectGraph and TrackGraph steps at each of `--cameras` cameras, "bayer_rggb8" frames of `--height` x `--width` in
   pinned host memory.  Two arms, alternated step by step (their order swaps every step):
     host-cvt  cv2.cvtColor(COLOR_BayerBG2BGR) on the host into pinned BGR buffers, then the BGR graph
     bayer     the mosaics go to a graph built with pixel_format="bayer_rggb8" (1 B/px uploaded instead of 3)
   The outputs of the two arms are compared every step (they must be identical).  Per arm the median and mean wall
   time of a step (a host clock around the conversion and the call, ending in a device synchronise) over `--steps`
   steps after `--warmup`.

Seeded dla_34 weights (tf32x3) with heat-map biases calibrated to about 4 objects per frame.  The card name, power
limit and maximum SM clock are printed first, in the same run; they are part of the numbers.  Prints JSON lines.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import synth  # noqa: E402
from scripts.yuv_input import gpu_state, make_detector  # noqa: E402
from tests import bayer_ref  # noqa: E402

ARMS = ("bgr",) + bayer_ref.FORMATS


def to_bgr(f, fmt):
    import cv2
    return f if fmt == "bgr" else cv2.cvtColor(f, getattr(cv2, bayer_ref.CV2_CODES[fmt]))


def preprocess_calls(dev, args):
    B, h, w = 32, 1200, 1920
    opt = cpb.default_opt("dla_34")
    base = synth.synthetic_frames(4, h, w, seed=900)
    arms = {f: [base[b % 4] if f == "bgr" else bayer_ref.from_bgr(base[b % 4], f) for b in range(B)] for f in ARMS}
    hw = np.array([(h, w)] * B, np.int32)
    bufs, offs = {}, {}
    for a, frames in arms.items():
        sizes = [f.size for f in frames]
        offs[a] = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        bufs[a] = torch.from_numpy(np.concatenate([f.reshape(-1) for f in frames])).to(dev)
    out = torch.empty((B, 3, 512, 512), dtype=torch.float32, device=dev)

    def call(a):
        if a == "bgr":
            cpb.preprocess_ragged(bufs[a], offs[a], hw, 512, 512, opt.mean, opt.std, out=out)
        else:
            cpb.preprocess_formats(bufs[a], offs[a], hw, a, 512, 512, opt.mean, opt.std, out=out)

    for a, frames in arms.items():          # each arm against the BGR call on the cv2 conversion of its own bytes
        bgr = torch.from_numpy(np.stack([to_bgr(f, a) for f in frames])).to(dev).reshape(-1)
        want = cpb.preprocess_ragged(bgr, np.arange(B, dtype=np.int64) * (h * w * 3), hw, 512, 512, opt.mean, opt.std)
        call(a)
        assert torch.equal(out, want), a
    times = {a: [] for a in arms}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for a in arms:
            for _ in range(5):
                call(a)
            e0.record()
            for _ in range(args.reps):
                call(a)
            e1.record()
            torch.cuda.synchronize()
            times[a].append(e0.elapsed_time(e1) / args.reps * 1e3)
    for a, us in times.items():
        print(json.dumps({"preprocess_call": a, "frames": B, "src": "%dx%d" % (w, h), "dst": "512x512",
                          "us_per_call": [round(v, 1) for v in us], "source_bytes": int(bufs[a].numel())}))


def graph_steps(dev, kind, S, args):
    import cv2
    fmt = "bayer_rggb8"
    h, w = args.height, args.width
    det = make_detector(dev, tracking=kind == "track")
    cls = cpb.TrackGraph if kind == "track" else cpb.DetectGraph
    cam = synth.default_camera(w, h)
    graw = cls(det, slots=S, frame_hw=(h, w), camera_matrix=cam, pixel_format=fmt)
    gbgr = cls(det, slots=S, frame_hw=(h, w), camera_matrix=cam)
    pool = [bayer_ref.from_bgr(f, fmt) for f in synth.synthetic_frames(4, h, w, seed=700)]
    total = args.steps + args.warmup
    src = [torch.from_numpy(np.stack([pool[(t + s) % 4] for s in range(S)])).pin_memory() for t in range(4)]
    bgr = [torch.empty((S, h, w, 3), dtype=torch.uint8).pin_memory() for _ in range(2)]
    code = getattr(cv2, bayer_ref.CV2_CODES[fmt])
    times = {"host-cvt": [], "bayer": []}

    def raw_arm(frames):
        t0 = time.perf_counter()
        out = graw(frames)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, [x.cpu().numpy() for x in out]

    def host_arm(frames, dst):
        t0 = time.perf_counter()
        for s in range(S):
            cv2.cvtColor(frames[s].numpy(), code, dst=dst[s].numpy())
        out = gbgr(dst)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, [x.cpu().numpy() for x in out]

    for t in range(total):
        frames = src[t % 4]
        # a tracking graph carries state between steps, so both arms see the same frames in the same order; only
        # which of them runs first alternates
        if t % 2:
            dt_h, want = host_arm(frames, bgr[t % 2])
            dt_r, got = raw_arm(frames)
        else:
            dt_r, got = raw_arm(frames)
            dt_h, want = host_arm(frames, bgr[t % 2])
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), (kind, S, t)
        if t >= args.warmup:
            times["bayer"].append(dt_r * 1e3)
            times["host-cvt"].append(dt_h * 1e3)
    for arm, ms in times.items():
        print(json.dumps({"graph": kind, "cameras": S, "format": fmt, "frame": "%dx%d" % (w, h), "arm": arm,
                          "median_ms": round(float(np.median(ms)), 3), "mean_ms": round(float(np.mean(ms)), 3),
                          "steps": len(ms), "identical": True}))
    del graw, gbgr, det
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--height", type=int, default=1200)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sensor_formats.py measures on a CUDA device; none is available")
    import cv2
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_state(), "cv2_threads": cv2.getNumThreads(), "host_cpus": os.cpu_count()}))
    preprocess_calls(dev, args)
    for kind in ("detect", "track"):
        for S in args.cameras:
            graph_steps(dev, kind, S, args)


if __name__ == "__main__":
    main()
