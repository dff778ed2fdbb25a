"""Phone formats against NV12 and host conversion: python scripts/phone_formats.py [--cameras 1 8] [--steps 20]

1. The pre-process call alone, per format, on 32 device-resident 1920x1440 frames (Objectron's size) to a 512x512
   input (CUDA events, 5 warm-up calls, `--reps` calls per measurement, the formats alternated, `--rounds` rounds):
   "nv12" and each phone format ("nv21", "yv12" and the four full-range formats) through cp_preprocess_formats.  Every
   arm's output is checked against the BGR call on the host-converted frames first.
2. DetectGraph and TrackGraph steps at each of `--cameras` cameras, "nv12_full" frames of `--height` x `--width` in
   pinned host memory, as ARKit delivers them.  Two arms, alternated step by step (their order swaps every step):
     host-cvt   the chroma replicated per 2x2 block and cv2.cvtColor(COLOR_YCrCb2BGR) on the host into pinned BGR
                buffers, then the BGR graph
     nv12_full  the frames go to a graph built with pixel_format="nv12_full" (1.5 B/px uploaded instead of 3)
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
from tests import phone_ref  # noqa: E402

ARMS = ("nv12",) + phone_ref.FORMATS


def to_bgr(f, fmt):
    return phone_ref.cv2_bgr(f, fmt)


def full_to_bgr(frame, h, dst):
    """The host conversion of one nv12_full frame into dst: the chroma replicated per 2x2 block, then
    COLOR_YCrCb2BGR."""
    import cv2
    uv = frame[h:].reshape(h // 2, -1, 2)
    cr = cv2.resize(uv[..., 1], None, fx=2, fy=2, interpolation=cv2.INTER_NEAREST)
    cb = cv2.resize(uv[..., 0], None, fx=2, fy=2, interpolation=cv2.INTER_NEAREST)
    cv2.cvtColor(cv2.merge([frame[:h], cr, cb]), cv2.COLOR_YCrCb2BGR, dst=dst)


def preprocess_calls(dev, args):
    B, h, w = 32, 1440, 1920
    opt = cpb.default_opt("dla_34")
    base = synth.synthetic_frames(4, h, w, seed=900)
    arms = {f: [phone_ref.from_bgr(base[b % 4], f) for b in range(B)] for f in ARMS}
    hw = np.array([(h, w)] * B, np.int32)
    bufs, offs = {}, {}
    for a, frames in arms.items():
        sizes = [f.size for f in frames]
        offs[a] = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        bufs[a] = torch.from_numpy(np.concatenate([f.reshape(-1) for f in frames])).to(dev)
    out = torch.empty((B, 3, 512, 512), dtype=torch.float32, device=dev)

    def call(a):
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
    fmt = "nv12_full"
    h, w = args.height, args.width
    det = make_detector(dev, tracking=kind == "track")
    cls = cpb.TrackGraph if kind == "track" else cpb.DetectGraph
    cam = synth.default_camera(w, h)
    graw = cls(det, slots=S, frame_hw=(h, w), camera_matrix=cam, pixel_format=fmt)
    gbgr = cls(det, slots=S, frame_hw=(h, w), camera_matrix=cam)
    pool = [phone_ref.from_bgr(f, fmt) for f in synth.synthetic_frames(4, h, w, seed=700)]
    total = args.steps + args.warmup
    src = [torch.from_numpy(np.stack([pool[(t + s) % 4] for s in range(S)])).pin_memory() for t in range(4)]
    bgr = [torch.empty((S, h, w, 3), dtype=torch.uint8).pin_memory() for _ in range(2)]
    times = {"host-cvt": [], fmt: []}

    def raw_arm(frames):
        t0 = time.perf_counter()
        out = graw(frames)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, [x.cpu().numpy() for x in out]

    def host_arm(frames, dst):
        t0 = time.perf_counter()
        for s in range(S):
            full_to_bgr(frames[s].numpy(), h, dst[s].numpy())
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
            times[fmt].append(dt_r * 1e3)
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
    ap.add_argument("--height", type=int, default=1440)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("phone_formats.py measures on a CUDA device; none is available")
    import cv2
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_state(), "cv2_threads": cv2.getNumThreads(), "host_cpus": os.cpu_count()}))
    preprocess_calls(dev, args)
    for kind in ("detect", "track"):
        for S in args.cameras:
            graph_steps(dev, kind, S, args)


if __name__ == "__main__":
    main()
