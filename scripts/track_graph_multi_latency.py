"""Live-video tracking steps of several categories and of slots of different frame sizes: MultiCategoryTrackGraph against
MultiCategoryTracker.run_batch, and TrackGraph with one frame_hw per slot against run_batch(list, track=True), at
512 x 512 in tf32x3.

    python scripts/track_graph_multi_latency.py [--steps 20] [--warmup 5] [--runs 2] [--out results/track_graph_multi.json]

Configurations (frames from pinned host memory):
  * M = 3 and M = 9 categories, 1 slot of 480 x 640, BGR and NV12 frames;
  * 1 category, 2 slots of 480 x 640 and 720 x 1280, BGR frames.
Every category's checkpoint is seeded and its heat-map biases calibrated to about 4 objects per frame.  Both arms track
the same synthetic video, alternating step by step, and their tracks are checked bit for bit every step.  The columns
are those of track_graph_latency.py (step_ms: host clock of a step; busy_ms: the device's busy time in a profiled run of
its own).  The plan bytes of each multi-category graph (cp_plan_memory) and the GPU's name, power limit and clocks, read
in the same run, are written beside the numbers."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import synth  # noqa: E402
import track_graph_latency as tgl  # noqa: E402

H, W = tgl.H, tgl.W
CATEGORIES = ["chair", "cup", "laptop", "bike", "book", "bottle", "camera", "cereal_box", "shoe"]


def tracker(M, ckpt_dir):
    """A MultiCategoryTracker of the first M categories, one seeded, calibrated checkpoint each."""
    opt = cpb.default_opt("dla_34", tracking_task=True)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, 512, 512, seed=5))).cuda()
    z = torch.zeros((2, 1, 512, 512), device="cuda")
    paths = {}
    for i, c in enumerate(CATEGORIES[:M]):
        paths[c] = os.path.join(ckpt_dir, c + ".pth")
        if not os.path.exists(paths[c]):
            m.load_state_dict(synth.seeded_state_dict(m, seed=31 + i, offset_std=0.3))
            with torch.no_grad():
                synth.calibrate_head_bias(m, m(x, x, z, z.repeat(1, 8, 1, 1))[-1], target=4)
            cpb.save_model(paths[c], 1, m)
    return cpb.MultiCategoryTracker(opt, paths)


def measure_multi(M, fmt, a, ckpt_dir):
    trk = tracker(M, ckpt_dir)
    cam = synth.default_camera(W, H)
    tg = cpb.MultiCategoryTrackGraph(trk, slots=1, frame_hw=(H, W), camera_matrix=cam, pixel_format=fmt)
    arms = {"graph": lambda f: tg(f),
            "run_batch": lambda f: trk.run_batch(f, cam, pixel_format=fmt, to_host=False)}
    r = tgl.time_arms(arms, [tg.reset, trk.reset_tracking], tgl.video(1, fmt, a.warmup + a.steps), a.warmup, a.runs,
                      "M=%d %s" % (M, fmt), a.traces and os.path.join(a.traces, "track_graph_multi_%%s_M%d_%s.json" % (M, fmt)))
    r["plan_memory"] = tg.eng.memory
    r["plan_bytes"] = tg.eng.plan_bytes
    return r


def ragged_video(sizes, n):
    bases = [synth.synthetic_frames(1, h, w, seed=21 + i)[0] for i, (h, w) in enumerate(sizes)]
    return [[torch.from_numpy(np.ascontiguousarray(np.roll(b, (2 * k, 3 * k), axis=(0, 1)))).pin_memory() for b in bases]
            for k in range(n)]


def measure_ragged(a):
    sizes = [(480, 640), (720, 1280)]
    det = tgl.detector()
    cams = np.stack([synth.default_camera(w, h) for h, w in sizes])
    tg = cpb.TrackGraph(det, slots=2, frame_hw=sizes, camera_matrix=cams)
    arms = {"graph": lambda f: tg(f),
            "run_batch": lambda f: det.run_batch(f, cams, track=True, to_host=False)}
    return tgl.time_arms(arms, [tg.reset, det.reset_tracking], ragged_video(sizes, a.warmup + a.steps), a.warmup,
                         a.runs, "per-slot sizes", a.traces and os.path.join(a.traces, "track_graph_ragged_%s.json"))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default="")
    ap.add_argument("--traces", default="", help="directory for the profiler traces (none when empty)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("track_graph_multi_latency.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    cond = tgl.gpu_conditions()
    rows = []
    with tempfile.TemporaryDirectory() as ckpt_dir:
        configs = [("M=%d S=1 480x640" % M, fmt, lambda M=M, fmt=fmt: measure_multi(M, fmt, a, ckpt_dir))
                   for M in (3, 9) for fmt in ("bgr", "nv12")]
        configs.append(("M=1 S=2 480x640+720x1280", "bgr", lambda: measure_ragged(a)))
        for label, fmt, fn in configs:
            r = fn()
            rows.append({"config": label, "pixel_format": fmt, **r})
            g, h = r["graph"], r["run_batch"]
            for arm in ("graph", "run_batch"):
                x = r[arm]
                print("%-26s %-4s %-9s step %7.3f ms  gpu %7.3f ms  kernel sum %7.3f ms (%d)  busy %7.3f ms  "
                      "launch+host %6.3f ms" % (label, fmt, arm, x["step_ms"]["median"], x["gpu_ms"]["median"],
                                                x["kernel_sum_ms"], x["kernels_per_step"], x["busy_ms"],
                                                x["step_ms"]["median"] - x["busy_ms"]), flush=True)
            print("%-26s %-4s speed-up %.2fx%s" % (label, fmt, h["step_ms"]["median"] / g["step_ms"]["median"],
                                                   ("  plan bytes %d (%s)" % (r["plan_bytes"], r["plan_memory"]))
                                                   if "plan_bytes" in r else ""), flush=True)
    cond.update(input="512x512", precision="tf32x3", steps=a.steps, warmup=a.warmup, runs=a.runs)
    print(json.dumps(cond))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fp:
            json.dump({"conditions": cond, "rows": rows}, fp, indent=1)


if __name__ == "__main__":
    main()
