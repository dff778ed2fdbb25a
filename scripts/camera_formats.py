"""Camera pixel formats against host conversion: python scripts/camera_formats.py [--cameras 1 8] [--steps 20]

1. The pre-process call alone, per format, on 32 device-resident 1920x1080 frames to a 512x512 input (CUDA events,
   warmed up, `--reps` calls per measurement, the formats alternated, `--rounds` rounds): BGR through
   cp_preprocess_ragged, the camera formats through cp_preprocess_formats, and one mixed batch of all eight formats.
   Every format's output is checked against the BGR call on the cv2.cvtColor-converted frames first.
2. DetectGraph and TrackGraph steps at each of `--cameras` cameras, packed YUV 4:2:2 frames ("uyvy422" for detection,
   "yuyv422" for tracking) of `--height` x `--width` in pinned host memory.  Two arms, alternated step by step:
     host-cvt  cv2.cvtColor(COLOR_YUV2BGR_UYVY / _YUYV) on the host into pinned BGR buffers, then the BGR graph
     422       the 4:2:2 frames go to a graph built with that pixel_format (2 B/px uploaded instead of 3)
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
from tests import yuv422_ref  # noqa: E402

FORMATS = ("bgr", "nv12", "i420", "rgb24", "rgba", "bgra", "yuyv422", "uyvy422")


def encode(bgr, fmt):
    import cv2
    if fmt in ("nv12", "i420"):
        h, w = bgr.shape[:2]
        i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
        if fmt == "i420":
            return i420
        c = i420[h:].reshape(-1)
        return np.concatenate([i420[:h], np.stack([c[:h * w // 4], c[h * w // 4:]], axis=-1).reshape(h // 2, w)])
    return yuv422_ref.from_bgr(bgr, fmt)


def to_bgr(f, fmt):
    import cv2
    if fmt == "bgr":
        return f
    code = {"nv12": "COLOR_YUV2BGR_NV12", "i420": "COLOR_YUV2BGR_I420"}.get(fmt) or yuv422_ref.CV2_CODES[fmt]
    return cv2.cvtColor(f, getattr(cv2, code))


def preprocess_calls(dev, args):
    B, h, w = 32, 1080, 1920
    opt = cpb.default_opt("dla_34")
    base = synth.synthetic_frames(4, h, w, seed=900)
    arms = {f: [encode(base[b % 4], f) for b in range(B)] for f in FORMATS}
    arms["mixed"] = [arms[FORMATS[b % len(FORMATS)]][b] for b in range(B)]
    fmts = {f: [f] * B for f in FORMATS}
    fmts["mixed"] = [FORMATS[b % len(FORMATS)] for b in range(B)]
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
            cpb.preprocess_formats(bufs[a], offs[a], hw, fmts[a][0] if a != "mixed" else fmts[a], 512, 512, opt.mean,
                                   opt.std, out=out)

    for a, frames in arms.items():          # each arm against the BGR call on the cv2 conversion of its own bytes
        bgr = torch.from_numpy(np.stack([to_bgr(f, m) for f, m in zip(frames, fmts[a])])).to(dev).reshape(-1)
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


def graph_steps(dev, kind, fmt, S, args):
    import cv2
    h, w = args.height, args.width
    det = make_detector(dev, tracking=kind == "track")
    cls = cpb.TrackGraph if kind == "track" else cpb.DetectGraph
    cam = synth.default_camera(w, h)
    g422 = cls(det, slots=S, frame_hw=(h, w), camera_matrix=cam, pixel_format=fmt)
    gbgr = cls(det, slots=S, frame_hw=(h, w), camera_matrix=cam)
    pool = [encode(f, fmt) for f in synth.synthetic_frames(4, h, w, seed=700)]
    total = args.steps + args.warmup
    src = [torch.from_numpy(np.stack([pool[(t + s) % 4] for s in range(S)])).pin_memory() for t in range(4)]
    bgr = [torch.empty((S, h, w, 3), dtype=torch.uint8).pin_memory() for _ in range(2)]
    code = getattr(cv2, yuv422_ref.CV2_CODES[fmt])
    times = {"host-cvt": [], "422": []}
    for t in range(total):
        frames = src[t % 4]
        t0 = time.perf_counter()
        got = g422(frames)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        got = [x.cpu().numpy() for x in got]
        t2 = time.perf_counter()
        dst = bgr[t % 2]
        for s in range(S):
            cv2.cvtColor(frames[s].numpy(), code, dst=dst[s].numpy())
        want = gbgr(dst)
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        want = [x.cpu().numpy() for x in want]
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), (kind, S, t)
        if t >= args.warmup:
            times["422"].append((t1 - t0) * 1e3)
            times["host-cvt"].append((t3 - t2) * 1e3)
    for arm, ms in times.items():
        print(json.dumps({"graph": kind, "cameras": S, "format": fmt, "frame": "%dx%d" % (w, h), "arm": arm,
                          "median_ms": round(float(np.median(ms)), 3), "mean_ms": round(float(np.mean(ms)), 3),
                          "steps": len(ms), "identical": True}))
    del g422, gbgr, det
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
        raise SystemExit("camera_formats.py measures on a CUDA device; none is available")
    import cv2
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_state(), "cv2_threads": cv2.getNumThreads(), "host_cpus": os.cpu_count()}))
    preprocess_calls(dev, args)
    for kind, fmt in (("detect", "uyvy422"), ("track", "yuyv422")):
        for S in args.cameras:
            graph_steps(dev, kind, fmt, S, args)


if __name__ == "__main__":
    main()
