"""One live-video detection step, DetectGraph against run_batch, at 512 x 512 in tf32x3.

    python scripts/detect_graph_latency.py [--steps 20] [--warmup 5] [--runs 2] [--out results/detect_graph.json]

Configurations (frames from pinned host memory, 480 x 640 unless stated):
  * S = 1 and 8 cameras, BGR and NV12 frames (run_batch's array form);
  * two cameras of 480 x 640 and 720 x 1280, BGR (run_batch(list));
  * S = 4 cameras, BGR, with the seeded drop pattern of track_graph_idle_latency.py (about 25 % idle per camera, a late
    start, an end): DetectGraph(idle_slots=True) against run_batch(list) of the live frames, whose rows the arm scatters
    to the slots on the device (a zero fill and one index copy per output);
  * M = 3 categories (MultiCategoryDetectGraph against MultiCategoryDetector.run_batch) at S = 1, BGR.
Every checkpoint is seeded and its heat-map biases calibrated to about 4 objects per frame.  Both arms run the same
frames, alternating step by step, and their poses and n_valid are checked identical at every step.  The detector's plan
is made at S frames first, so run_batch runs on a plan of the graph's capacity (split-K follows the plan's workspace).
The columns are those of track_graph_latency.py (time_arms): step_ms is the host clock from the call to the outputs
ready on the device, busy_ms the time the device has a kernel or copy running, in a profiled run of its own.  Also per
configuration: the graph's build time and the drop in free device memory it costs.  The GPU's name, power limit and
clocks are read in the same run and written beside the numbers."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import synth  # noqa: E402
from track_graph_idle_latency import drop_pattern  # noqa: E402
from track_graph_latency import H, W, gpu_conditions, time_arms, video  # noqa: E402
from track_graph_multi_latency import ragged_video  # noqa: E402

CATEGORIES = ["chair", "cup", "laptop"]


def calibrated(opt, seed):
    """A seeded model calibrated on one frame: its plan holds one frame until the configuration makes it hold S."""
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    m.load_state_dict(synth.seeded_state_dict(m, seed=seed, offset_std=0.3))
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(1, 512, 512, seed=5))).cuda()
    with torch.no_grad():
        synth.calibrate_head_bias(m, m(x)[-1], target=4)
    return m


def detector():
    opt = cpb.default_opt("dla_34")
    return cpb.ObjectPoseDetector(opt, model=calibrated(opt, 31))


def multi_detector(ckpt_dir):
    opt = cpb.default_opt("dla_34")
    paths = {}
    for i, c in enumerate(CATEGORIES):
        paths[c] = os.path.join(ckpt_dir, c + ".pth")
        cpb.save_model(paths[c], 1, calibrated(opt, 31 + i))
    return cpb.MultiCategoryDetector(opt, paths)


def build(make):
    """(graph, seconds to build it, bytes of free device memory it took)."""
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    g = make()
    torch.cuda.synchronize()
    return g, time.perf_counter() - t0, free0 - torch.cuda.mem_get_info()[0]


def scattered(run, S):
    """A run_batch arm for a list with idle slots: run on the live frames, the rows scattered to the slots."""
    def arm(fs):
        live = [i for i, f in enumerate(fs) if f is not None]
        poses = torch.zeros((S, 100, cpb._lib.CP_POSE_RECORD), dtype=torch.float32, device="cuda")
        n = torch.zeros((S,), dtype=torch.int32, device="cuda")
        if live:
            p, c = run([fs[i] for i in live], live)
            idx = torch.tensor(live, device="cuda")
            poses.index_copy_(0, idx, p)
            n.index_copy_(0, idx, c)
        return poses, n
    return arm


def measure(label, a, ckpt_dir):
    n = a.warmup + a.steps
    if label.startswith("M=3"):
        det, S = multi_detector(ckpt_dir), 1
        cam = synth.default_camera(W, H)
        det.engine(S, det.opt.input_h, det.opt.input_w)
        g, build_s, nbytes = build(lambda: cpb.MultiCategoryDetectGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam))
        frames = video(S, "bgr", n)
        ref = lambda f: det.run_batch(f, cam, to_host=False)  # noqa: E731
        fmt = "bgr"
    else:
        det = detector()
        if label.startswith("2 cameras"):
            sizes, S, fmt = [(480, 640), (720, 1280)], 2, "bgr"
            cam = np.stack([synth.default_camera(w, h) for h, w in sizes])
            det.model.engine(S, det.opt.input_h, det.opt.input_w)
            g, build_s, nbytes = build(lambda: cpb.DetectGraph(det, slots=S, frame_hw=sizes, camera_matrix=cam))
            frames = ragged_video(sizes, n)
            ref = lambda f: det.run_batch(f, cam, to_host=False)  # noqa: E731
        elif label.startswith("idle"):
            S, fmt = 4, "bgr"
            cam = np.stack([synth.default_camera(W, H)] * S)
            det.model.engine(S, det.opt.input_h, det.opt.input_w)
            g, build_s, nbytes = build(lambda: cpb.DetectGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam,
                                                               idle_slots=True))
            live = drop_pattern(S, n)
            frames = [[f[i] if live[k, i] else None for i in range(S)] for k, f in enumerate(video(S, fmt, n))]
            ref = scattered(lambda fs, ids: det.run_batch(fs, cam[ids], to_host=False), S)
        else:
            S, fmt = int(label.split()[0][2:]), label.split()[1]
            cam = synth.default_camera(W, H)
            det.model.engine(S, det.opt.input_h, det.opt.input_w)
            g, build_s, nbytes = build(lambda: cpb.DetectGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam,
                                                               pixel_format=fmt))
            frames = video(S, fmt, n)
            ref = lambda f: det.run_batch(f, cam, pixel_format=fmt, to_host=False)  # noqa: E731
    r = time_arms({"graph": lambda f: g(f), "run_batch": ref}, [], frames, a.warmup, a.runs, label)
    r.update(slots=S, pixel_format=fmt, build_s=build_s, device_bytes=nbytes)
    return r


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("detect_graph_latency.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    cond = gpu_conditions()
    print(json.dumps(cond), flush=True)
    rows = []
    labels = ["S=1 bgr", "S=1 nv12", "S=8 bgr", "S=8 nv12", "2 cameras 480x640+720x1280 bgr", "idle S=4 bgr",
              "M=3 S=1 bgr"]
    with tempfile.TemporaryDirectory() as ckpt_dir:
        for label in labels:
            r = measure(label, a, ckpt_dir)
            rows.append({"config": label, **r})
            for arm in ("graph", "run_batch"):
                x = r[arm]
                print("%-32s %-9s step %7.3f ms  gpu %7.3f ms  kernel sum %7.3f ms (%d)  busy %7.3f ms  "
                      "launch+host %6.3f ms" % (label, arm, x["step_ms"]["median"], x["gpu_ms"]["median"],
                                                x["kernel_sum_ms"], x["kernels_per_step"], x["busy_ms"],
                                                x["step_ms"]["median"] - x["busy_ms"]), flush=True)
            print("%-32s speed-up %.2fx  build %.2f s  device memory %.1f MB"
                  % (label, r["run_batch"]["step_ms"]["median"] / r["graph"]["step_ms"]["median"], r["build_s"],
                     r["device_bytes"] / 2**20), flush=True)
    cond.update(frame="%dx%d" % (W, H), input="512x512", precision="tf32x3", steps=a.steps, warmup=a.warmup, runs=a.runs)
    print(json.dumps(cond))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fp:
            json.dump({"conditions": cond, "rows": rows}, fp, indent=1)


if __name__ == "__main__":
    main()
