"""One live-video tracking step, TrackGraph against run_batch(track=True), at 512 x 512 in tf32x3.

    python scripts/track_graph_latency.py [--steps 20] [--warmup 5] [--runs 2] [--out results/track_graph_latency.json]

For S = 1 and 8 slots and BGR and NV12 frames (480 x 640, from pinned host memory) both arms track the same synthetic
video on one seeded, calibrated detector, alternating step by step.  Per arm and configuration it reports:
  * step_ms: host clock from the call with the frames on the host to the tracks ready (a device synchronise);
  * gpu_ms: CUDA events around the same call (the device's span of the step, copies included);
  * kernel_sum_ms / copy_ms: the sum of the step's kernel (and copy) durations from torch.profiler, in a separate run;
    kernels launched with programmatic dependent launch start before their predecessor ends, so this sum counts the
    overlap twice and can exceed the step;
  * busy_ms: the time the device has a kernel or copy running (the union of those intervals) in the same run.
step_ms - busy_ms is the launch and host share of a step: the device idles while the host issues work.  Medians over
steps; the runs are repeats of the whole alternation.  Both arms' tracks are checked bit for bit every step.  The
GPU's name, power limit and clocks are read in the same run and written beside the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import synth  # noqa: E402

H, W = 480, 640


def gpu_conditions():
    q = "name,power.limit,clocks.max.sm,clocks.sm,temperature.gpu"
    try:
        row = subprocess.check_output(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], text=True)
        return dict(zip(q.split(","), [v.strip() for v in row.splitlines()[0].split(",")]))
    except (OSError, subprocess.CalledProcessError):
        return {"name": torch.cuda.get_device_name(0)}


def detector():
    opt = cpb.default_opt("dla_34", tracking_task=True)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    m.load_state_dict(synth.seeded_state_dict(m, seed=31, offset_std=0.3))
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, 512, 512, seed=5))).cuda()
    z = torch.zeros((2, 1, 512, 512), device="cuda")
    with torch.no_grad():
        synth.calibrate_head_bias(m, m(x, x, z, z.repeat(1, 8, 1, 1))[-1], target=4)
    return cpb.ObjectPoseDetector(opt, model=m)


def to_nv12(bgr):
    import cv2
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    c = i420[H:].reshape(-1)
    n = H * W // 4
    return np.concatenate([i420[:H], np.stack([c[:n], c[n:]], axis=-1).reshape(H // 2, W)])


def video(S, fmt, n):
    base = synth.synthetic_frames(S, H, W, seed=11 + S)
    out = []
    for k in range(n):
        f = np.roll(base, (2 * k, 3 * k), axis=(1, 2))
        f = f if fmt == "bgr" else np.stack([to_nv12(g) for g in f])
        out.append(torch.from_numpy(f).pin_memory())
    return out


def measure(S, fmt, steps, warmup, runs, prof_dir):
    det = detector()
    cam = synth.default_camera(W, H)
    tg = cpb.TrackGraph(det, slots=S, frame_hw=(H, W), camera_matrix=cam, pixel_format=fmt)
    arms = {"graph": lambda f: tg(f),
            "run_batch": lambda f: det.run_batch(f, cam, track=True, pixel_format=fmt, to_host=False)}
    return time_arms(arms, [tg.reset, det.reset_tracking], video(S, fmt, warmup + steps), warmup, runs,
                     "S=%d %s" % (S, fmt), prof_dir and os.path.join(prof_dir, "track_graph_%%s_S%d_%s.json" % (S, fmt)))


def time_arms(arms, resets, frames, warmup, runs, label, trace=None):
    """Both arms over the same frames, alternating step by step, after calling every reset; their outputs are checked
    identical at every step.  trace: a path pattern with one %s (the arm) for the profiler traces, or None."""
    res = {a: {"step_ms": [], "gpu_ms": []} for a in arms}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(runs):
        for r in resets:
            r()
        for k, f in enumerate(frames):
            outs = {}
            for a, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ev0.record()
                t, n = fn(f)
                ev1.record()
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                outs[a] = (t.cpu().numpy(), n.cpu().numpy())
                if k >= warmup:
                    res[a]["step_ms"].append((t1 - t0) * 1e3)
                    res[a]["gpu_ms"].append(ev0.elapsed_time(ev1))
            g, r = outs["graph"], outs["run_batch"]
            if not (np.array_equal(g[0], r[0]) and np.array_equal(g[1], r[1])):
                raise SystemExit("%s step %d: the graph and run_batch disagree" % (label, k))
    # kernel and copy sums per step, profiled in a run of their own
    from torch.autograd import DeviceType
    n_prof = 5
    for a, fn in arms.items():
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                                torch.profiler.ProfilerActivity.CUDA]) as prof:
            for f in frames[:n_prof]:
                fn(f)
            torch.cuda.synchronize()
        dev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
        copies = [e for e in dev if e.name.startswith(("Memcpy", "Memset"))]
        kern = [e for e in dev if not e.name.startswith(("Memcpy", "Memset"))]
        res[a]["kernel_sum_ms"] = sum(e.time_range.elapsed_us() for e in kern) / 1e3 / n_prof
        res[a]["copy_ms"] = sum(e.time_range.elapsed_us() for e in copies) / 1e3 / n_prof
        busy, end = 0.0, -1.0
        for s0, s1 in sorted((e.time_range.start, e.time_range.end) for e in dev):
            busy += max(0.0, s1 - max(s0, end))
            end = max(end, s1)
        res[a]["busy_ms"] = busy / 1e3 / n_prof
        res[a]["kernels_per_step"] = len(kern) / n_prof
        if trace:
            prof.export_chrome_trace(trace % a)
    for a in arms:
        for k in ("step_ms", "gpu_ms"):
            v = np.array(res[a][k])
            res[a][k] = {"median": float(np.median(v)), "p10": float(np.percentile(v, 10)),
                         "p90": float(np.percentile(v, 90)), "n": int(v.size)}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default="")
    ap.add_argument("--traces", default="", help="directory for the profiler traces (none when empty)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("track_graph_latency.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    cond = gpu_conditions()
    rows = []
    for S in (1, 8):
        for fmt in ("bgr", "nv12"):
            r = measure(S, fmt, a.steps, a.warmup, a.runs, a.traces)
            rows.append({"slots": S, "pixel_format": fmt, **r})
            for arm in ("graph", "run_batch"):
                x = r[arm]
                print("S=%d %-4s %-9s step %7.3f ms  gpu %7.3f ms  kernel sum %7.3f ms (%d)  copies %6.3f ms  "
                      "busy %7.3f ms  launch+host %6.3f ms"
                      % (S, fmt, arm, x["step_ms"]["median"], x["gpu_ms"]["median"], x["kernel_sum_ms"],
                         x["kernels_per_step"], x["copy_ms"], x["busy_ms"], x["step_ms"]["median"] - x["busy_ms"]),
                      flush=True)
    cond.update(frame="%dx%d" % (W, H), input="512x512", precision="tf32x3", steps=a.steps, warmup=a.warmup,
                runs=a.runs)
    print(json.dumps(cond))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fp:
            json.dump({"conditions": cond, "rows": rows}, fp, indent=1)


if __name__ == "__main__":
    main()
