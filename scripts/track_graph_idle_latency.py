"""Live-video tracking with idle slots: TrackGraph(idle_slots=True) against run_batch(list, track=True), at 512 x 512 in
tf32x3.

    python scripts/track_graph_idle_latency.py [--steps 20] [--warmup 5] [--runs 2] [--out results/track_graph_idle.json]

For S = 4 and 8 slots and BGR and NV12 frames (480 x 640, from pinned host memory) both arms track the same synthetic
video with the same seeded drop pattern: every slot is idle on about 25 % of the steps, slot 1 starts late and the last
slot ends two thirds of the way through.  The arms alternate step by step on one seeded, calibrated detector, and
their tracks are checked identical at every step (time_arms of scripts/track_graph_latency.py, which also defines the
columns).  Then, with every slot live, the idle-capable graph against the default TrackGraph: the cost of the per-slot
previous-frame store, the row maps and the gathers.  Last, the build time and the device memory (free memory before and
after, so the plan, the captured graphs and the buffers) of both graphs at S = 8 and 32.  The GPU's name, power limit
and clocks are read in the same run and written beside the numbers."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import synth  # noqa: E402
from track_graph_latency import H, W, detector, gpu_conditions, time_arms, video  # noqa: E402


def drop_pattern(S, n, seed=7):
    """live[k][i]: slot i has a frame at step k.  About 25 % idle per slot, slot 1 starts late, slot S-1 ends."""
    live = np.random.default_rng(seed).random((n, S)) >= 0.25
    live[:n // 4, 1] = False
    live[2 * n // 3:, S - 1] = False
    return live


def measure(S, fmt, steps, warmup, runs):
    det = detector()
    cam = synth.default_camera(W, H)
    n = warmup + steps
    frames = video(S, fmt, n)                                # pinned [S, ...] per step
    live = drop_pattern(S, n)
    lists = [[f[i] if live[k, i] else None for i in range(S)] for k, f in enumerate(frames)]
    ig = cpb.TrackGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam, pixel_format=fmt, idle_slots=True)
    arms = {"idle_graph": lambda f: ig(f),
            "run_batch": lambda f: det.run_batch(f, cam, track=True, pixel_format=fmt, to_host=False)}
    idle = time_arms(arms, [ig.reset, det.reset_tracking], lists, warmup, runs, "S=%d %s idle" % (S, fmt))
    tg = cpb.TrackGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam, pixel_format=fmt)
    arms = {"idle_graph": lambda f: ig(f), "graph": lambda f: tg(f)}
    full = time_arms(arms, [ig.reset, tg.reset], frames, warmup, runs, "S=%d %s all live" % (S, fmt))
    return idle, full, float(live.mean())


def build_cost(S, fmt="nv12"):
    """(seconds, bytes of device memory) to build the default and the idle-capable graph of S slots."""
    det = detector()
    cam = synth.default_camera(W, H)
    out = {}
    for name, idle in (("graph", False), ("idle_graph", True)):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        t0 = time.perf_counter()
        g = cpb.TrackGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam, pixel_format=fmt, idle_slots=idle)
        torch.cuda.synchronize()
        out[name] = {"build_s": time.perf_counter() - t0, "device_bytes": free0 - torch.cuda.mem_get_info()[0]}
        del g
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("track_graph_idle_latency.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    cond = gpu_conditions()
    print(json.dumps(cond), flush=True)
    rows = []
    for S in (4, 8):
        for fmt in ("bgr", "nv12"):
            idle, full, frac = measure(S, fmt, a.steps, a.warmup, a.runs)
            rows.append({"slots": S, "pixel_format": fmt, "live_fraction": frac, "idle": idle, "all_live": full})
            for what, r in (("idle slots (%.0f %% live)" % (100 * frac), idle), ("all live", full)):
                for arm, x in r.items():
                    print("S=%d %-4s %-22s %-10s step %7.3f ms  gpu %7.3f ms  busy %7.3f ms  launch+host %6.3f ms"
                          % (S, fmt, what, arm, x["step_ms"]["median"], x["gpu_ms"]["median"], x["busy_ms"],
                             x["step_ms"]["median"] - x["busy_ms"]), flush=True)
    builds = {}
    for S in (8, 32):
        builds[S] = build_cost(S)
        for name, b in builds[S].items():
            print("S=%d %-10s build %6.2f s  device memory %7.1f MB" % (S, name, b["build_s"], b["device_bytes"] / 2**20),
                  flush=True)
    cond.update(frame="%dx%d" % (W, H), input="512x512", precision="tf32x3", steps=a.steps, warmup=a.warmup, runs=a.runs)
    print(json.dumps(cond))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fp:
            json.dump({"conditions": cond, "rows": rows, "builds": builds}, fp, indent=1)


if __name__ == "__main__":
    main()
