"""Tracking throughput for S independent video streams: python scripts/track_streams.py [--streams 8 32] [--steps 20]

Three workloads per S, all frames device-resident (the network, pre-process, heat-map render and tracker step are
timed; host uploads are not), the tracking dla_34 with seeded weights whose heat-map biases are calibrated to about 4
objects per frame, CUDA events around `--steps` steps after `--warmup` steps:

  uniform-array  run_batch(uint8 [S,512,512,3], track=True): one frame size and camera, every stream steps every time
  uniform-list   run_batch(list of S 512x512 frames, track=True): the same frames through the slot path
  mixed-list     run_batch(list, track=True) with frames of 512x512, 480x640, 640x480, 600x800, 720x960, 375x500, one
                 camera per size, videos of 3..12 frames that restart their slot (new_video) when they end, and every
                 seventh slot idle for one step out of four

One JSON line per (S, workload): frame pairs per second counts the frames that went through the network (idle slots
excluded).  The GPU's power limit and clocks are printed first; they are part of the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import synth  # noqa: E402

SIZES = [(512, 512), (480, 640), (640, 480), (600, 800), (720, 960), (375, 500)]


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], text=True).strip()
    except Exception as e:                   # the numbers below still stand; say that the state is unknown
        return "unknown (%s)" % e


def make_detector(dev):
    opt = cpb.default_opt("dla_34", tracking_task=True)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=0, offset_std=0.3, head_gain=1.0))
    det = cpb.ObjectPoseDetector(opt, model=m)
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(8, 512, 512, seed=500))).to(dev)
    eng = det.model.engine(8, 512, 512, dev)
    z1, z8 = torch.zeros((8, 1, 512, 512), device=dev), torch.zeros((8, 8, 512, 512), device=dev)
    synth.calibrate_head_bias(det.model, eng.forward(x, x, z1, z8), 4)
    return det


def mixed_schedule(S, steps, rng):
    """Per step: per slot (size index, new_video) or None (idle)."""
    size = [s % len(SIZES) for s in range(S)]
    left = [0] * S
    out = []
    for t in range(steps):
        row = []
        for s in range(S):
            if s % 7 == 6 and t % 4 == 3:
                row.append(None)
                continue
            new = left[s] == 0
            if new:
                left[s] = int(rng.integers(3, 13))
                size[s] = int(rng.integers(0, len(SIZES)))
            left[s] -= 1
            row.append((size[s], new))
        out.append(row)
    return out


def timed(fn, steps, warmup):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        fn(warmup + i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("track_streams.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_state()}))
    det = make_detector(dev)
    pool = {hw: [torch.from_numpy(synth.synthetic_frames(1, hw[0], hw[1], seed=700 + 10 * i + k)[0]).to(dev)
                 for k in range(4)] for i, hw in enumerate(SIZES)}
    cams = {hw: synth.default_camera(hw[1], hw[0]) for hw in SIZES}
    total = args.steps + args.warmup
    for S in args.streams:
        cam = cams[(512, 512)]
        uni = [torch.stack([pool[(512, 512)][(s + k) % 4] for s in range(S)]) for k in range(4)]
        det.reset_tracking()
        ms = timed(lambda i: det.run_batch(uni[i % 4], cam, track=True, to_host=False), args.steps, args.warmup)
        print(json.dumps({"streams": S, "workload": "uniform-array", "ms_per_step": ms, "frame_pairs_per_s": S / ms * 1e3}))
        det.reset_tracking()
        ms = timed(lambda i: det.run_batch(list(uni[i % 4]), cam, track=True, to_host=False), args.steps, args.warmup)
        print(json.dumps({"streams": S, "workload": "uniform-list", "ms_per_step": ms, "frame_pairs_per_s": S / ms * 1e3}))
        sched = mixed_schedule(S, total, np.random.default_rng(S))
        steps = []
        for t, row in enumerate(sched):
            frames = [pool[SIZES[e[0]]][(t + s) % 4] if e is not None else None for s, e in enumerate(row)]
            slot_cams = np.stack([cams[SIZES[e[0]]] if e is not None else cam for e in row])
            steps.append((frames, slot_cams, [e is not None and e[1] for e in row]))
        det.reset_tracking()
        ms = timed(lambda i: det.run_batch(steps[i][0], steps[i][1], track=True, to_host=False, new_video=steps[i][2]),
                   args.steps, args.warmup)
        live = np.mean([sum(f is not None for f in st[0]) for st in steps[args.warmup:]])
        print(json.dumps({"streams": S, "workload": "mixed-list", "ms_per_step": ms, "live_per_step": float(live),
                          "frame_pairs_per_s": live / ms * 1e3}))


if __name__ == "__main__":
    main()
