"""ObjectPoseDetector.run() per call, device pre-process against the host one:
    python scripts/run_latency.py [--calls 20] [--warmup 5] [--rounds 2]

Two arms, alternated call by call (their order swaps every call), `--rounds` times:
  host    run() with the host pre_process (cv2.resize, cv2.warpAffine, the float64 normalisation, the fp32 upload):
          the device pre-process is replaced in this script only, on that arm's own detector
  device  run() as built: the uint8 frame uploaded once, resized and warped on the device
Workloads, on 1920x1440 and 640x480 frames: fix_res at test_scales [1], test_scales [0.75], and a CenterPoseTrack run()
sequence (both arms' detectors see the same frames in the same order).  Seeded dla_34 weights (tf32x3) with heat-map
biases calibrated to about 4 objects per frame; both arms' detectors hold the same weights, and their results (the
`results` records and the `output` maps) are checked to be identical at every call.

Per arm and round: the median over `--calls` calls after `--warmup` of the wall time of a call (a host clock around
run(), which ends in a device synchronise) and of run()'s own `pre` / `net` / `dec` / `tot` stamps, in ms.  The card
name, power limit and maximum SM clock are printed first, in the same run; they are part of the numbers.  Prints JSON
lines.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centerpose_b200 import synth  # noqa: E402
from scripts.yuv_input import gpu_state, make_detector  # noqa: E402

SIZES = [(1440, 1920), (480, 640)]
WORKLOADS = [("fix_res", [1.0], False), ("scale_0.75", [0.75], False), ("track", [1.0], True)]
STAMPS = ("pre", "net", "dec", "tot")


def same_bits(a, b):
    if isinstance(b, torch.Tensor):
        a, b = a.cpu().numpy(), b.cpu().numpy()
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def same_run(a, b):
    """run() results equal bit for bit: every result record field, the box tuples and the output maps."""
    if len(a["results"]) != len(b["results"]) or len(a["boxes"]) != len(b["boxes"]):
        return False
    for x, y in zip(a["results"], b["results"]):
        if sorted(x) != sorted(y) or not all(same_bits(x[k], y[k]) for k in y):
            return False
    for x, y in zip(a["boxes"], b["boxes"]):
        if not all(same_bits(x[i], y[i]) for i in range(4)):
            return False
    return all((v is None and a["output"][k] is None) or same_bits(a["output"][k], v) for k, v in b["output"].items())


def run_pair(dev, name, scales, tracking, h, w, args):
    arms = {}
    for arm in ("host", "device"):
        det = make_detector(dev, tracking)
        det.opt.test_scales = det.scales = scales
        if arm == "host":
            det._device_frame = lambda image: None
        arms[arm] = det
    frames = synth.synthetic_frames(4, h, w, seed=900)
    cam = synth.default_camera(w, h)
    for r in range(args.rounds):
        stats = {arm: {k: [] for k in ("wall",) + STAMPS} for arm in arms}
        found = []
        for det in arms.values():
            if tracking:
                det.reset_tracking()
        for t in range(args.warmup + args.calls):
            meta = {"camera_matrix": cam, "id": t}
            rets = {}
            for arm in (("host", "device") if t % 2 else ("device", "host")):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rets[arm] = arms[arm].run(frames[t % 4], meta_inp=meta)
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                if t >= args.warmup:
                    stats[arm]["wall"].append(wall * 1e3)
                    for k in STAMPS:
                        stats[arm][k].append(rets[arm][k] * 1e3)
            if not same_run(rets["device"], rets["host"]):
                raise SystemExit("run_latency: %s %dx%d call %d: the arms' results differ" % (name, w, h, t))
            found.append(len(rets["device"]["results"]))
        for arm, s in stats.items():
            row = {"workload": name, "frame": "%dx%d" % (w, h), "arm": arm, "round": r, "calls": args.calls,
                   "identical": True, "results_per_call": round(float(np.mean(found)), 2)}
            row.update({k + "_ms": round(float(np.median(v)), 3) for k, v in s.items()})
            print(json.dumps(row), flush=True)
    del arms
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("run_latency.py measures on a CUDA device; none is available")
    import cv2
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_state(), "cv2_threads": cv2.getNumThreads(), "host_cpus": os.cpu_count()}), flush=True)
    for h, w in SIZES:
        for name, scales, tracking in WORKLOADS:
            run_pair(dev, name, scales, tracking, h, w, args)


if __name__ == "__main__":
    main()
