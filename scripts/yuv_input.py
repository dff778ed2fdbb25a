"""YUV 4:2:0 input against host conversion: python scripts/yuv_input.py [--slots 8 32] [--batch 32] [--steps 20]

A video source gives NV12 frames (1920x1440, Objectron's native size, pinned host memory).  Two arms feed them to the
same pipeline, alternated within one run, `--rounds` times each:

  host-cvt  today's path: cv2.cvtColor(COLOR_YUV2BGR_NV12) on the host, per frame, into pinned BGR buffers, and the BGR
            frames (3 B/px) are submitted
  nv12      the NV12 frames (1.5 B/px) are submitted as they are (pixel_format="nv12"); the conversion runs inside the
            pre-process kernel

Workloads, 512x512 network input, tf32x3, seeded dla_34 weights whose heat-map biases are calibrated to about 4 objects
per frame: TrackPipeline with `--slots` video slots (one frame per slot per step), BatchPipeline at `--batch`.  Every
step's results of the two arms are compared (they must be identical).  Per arm: the wall time per step over `--steps`
steps after `--warmup` (a host clock around submit / collect, ending in a device synchronise), frame pairs (tracking) or
images per second, host ms per step spent in cv2.cvtColor, and the host-to-device bytes of the frames per step.

Then the pre-process calls alone on 32 device-resident frames (CUDA events, `--reps` calls, alternated): the BGR
cp_preprocess_ragged against cp_preprocess_yuv420 in NV12 and I420.

The card name, power limit and maximum SM clock are printed first, in the same run; they are part of the numbers.
"""
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


def gpu_state():
    q = "name,power.limit,clocks.max.sm"
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], text=True).strip()
    except Exception as e:                   # the numbers below still stand; say that the state is unknown
        return "unknown (%s)" % e


def nv12_frames(n, h, w, seed):
    """n synthetic frames encoded by cv2 as I420 and re-packed as NV12: uint8 [3h/2, w] each."""
    import cv2
    out = []
    for f in synth.synthetic_frames(n, h, w, seed=seed):
        i420 = cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420)
        c = i420[h:].reshape(-1)
        q = h * w // 4
        out.append(np.concatenate([i420[:h], np.stack([c[:q], c[q:]], axis=-1).reshape(h // 2, w)]))
    return out


def make_detector(dev, tracking):
    opt = cpb.default_opt("dla_34", tracking_task=tracking)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=0, offset_std=0.3, head_gain=1.0))
    det = cpb.ObjectPoseDetector(opt, model=m)
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(8, 512, 512, seed=500))).to(dev)
    eng = det.model.engine(8, 512, 512, dev)
    if tracking:
        z1, z8 = torch.zeros((8, 1, 512, 512), device=dev), torch.zeros((8, 8, 512, 512), device=dev)
        synth.calibrate_head_bias(det.model, eng.forward(x, x, z1, z8), 4)
    else:
        synth.calibrate_head_bias(det.model, eng.forward(x), 4)
    return det


class HostConvert(object):
    """cv2.cvtColor(NV12 -> BGR) into rotating pinned BGR buffers: `depth` + 1 sets, so a buffer is rewritten only after
    the pipeline has collected the step that uploaded it.  A list of frames gives a list, a stacked batch a batch."""

    def __init__(self, n, h, w, depth):
        self.sets = [torch.empty((n, h, w, 3), dtype=torch.uint8).pin_memory() for _ in range(depth + 1)]
        self.k = 0
        self.seconds = 0.0

    def __call__(self, frames):
        import cv2
        dst = self.sets[self.k % len(self.sets)]
        self.k += 1
        t = time.perf_counter()
        for i, f in enumerate(frames):
            cv2.cvtColor(f.numpy(), cv2.COLOR_YUV2BGR_NV12, dst=dst[i].numpy())
        self.seconds += time.perf_counter() - t
        return list(dst) if isinstance(frames, list) else dst


def run_arm(pipe, step_frames, convert, steps, warmup, submit):
    """Drive the pipeline over warmup + steps steps -> (ms per step, host cvtColor ms per step, every step's results)."""
    results, t0 = [], None
    for i, frames in enumerate(step_frames[:warmup + steps]):
        if i == warmup:
            torch.cuda.synchronize()
            if convert is not None:
                convert.seconds = 0.0
            t0 = time.perf_counter()
        if convert is not None:
            frames = convert(frames)
        if pipe.in_flight == pipe.depth:
            results.append([np.array(a) for a in pipe.collect()])
        submit(pipe, frames, i)
    while pipe.in_flight:
        results.append([np.array(a) for a in pipe.collect()])
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) / steps * 1e3
    return ms, (convert.seconds / steps * 1e3 if convert is not None else 0.0), results


def workload(name, det, make_pipe, submit, step_frames, n, h, w, args):
    rows = {"host-cvt": [], "nv12": []}
    same = True
    for r in range(args.rounds):
        res = {}
        for arm in ("host-cvt", "nv12"):
            if getattr(det.opt, "tracking_task", False):
                det.reset_tracking()
            pipe = make_pipe("bgr" if arm == "host-cvt" else "nv12")
            conv = HostConvert(n, h, w, pipe.depth) if arm == "host-cvt" else None
            ms, host_ms, res[arm] = run_arm(pipe, step_frames, conv, args.steps, args.warmup, submit)
            rows[arm].append((ms, host_ms))
        same = same and all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
                            for a, b in zip(res["host-cvt"], res["nv12"]))
    for arm, v in rows.items():
        ms = [m for m, _ in v]
        bpp = 3 if arm == "host-cvt" else 1.5
        print(json.dumps({"workload": name, "arm": arm, "ms_per_step": ms, "per_s_best": n / min(ms) * 1e3,
                          "host_cvtcolor_ms_per_step": [hm for _, hm in v], "h2d_bytes_per_step": int(n * h * w * bpp),
                          "identical_results": bool(same)}))


def kernel_times(dev, h, w, args):
    """CUDA-event time per pre-process call on 32 device-resident frames, BGR against NV12 / I420, alternated."""
    import cv2
    B = 32
    nv = nv12_frames(4, h, w, seed=900)
    nv = [nv[b % 4] for b in range(B)]
    i420 = []
    for f in nv:
        c = f[h:].reshape(h // 2, w // 2, 2)
        i420.append(np.concatenate([f[:h].reshape(-1), c[..., 0].reshape(-1), c[..., 1].reshape(-1)]))
    bgr = [cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) for f in nv]
    hw = np.array([(h, w)] * B, np.int32)
    bufs = {"bgr": torch.from_numpy(np.concatenate([f.reshape(-1) for f in bgr])).to(dev),
            "nv12": torch.from_numpy(np.concatenate([f.reshape(-1) for f in nv])).to(dev),
            "i420": torch.from_numpy(np.concatenate(i420)).to(dev)}
    out = torch.empty((B, 3, 512, 512), dtype=torch.float32, device=dev)
    opt = cpb.default_opt("dla_34")

    def call(fmt):
        buf = bufs[fmt]
        offs = np.arange(B, dtype=np.int64) * (buf.numel() // B)
        if fmt == "bgr":
            cpb.preprocess_ragged(buf, offs, hw, 512, 512, opt.mean, opt.std, out=out)
        else:
            cpb.preprocess_yuv420(buf, offs, hw, fmt, 512, 512, opt.mean, opt.std, out=out)

    outs = {}
    for fmt in bufs:
        call(fmt)
        outs[fmt] = out.clone()
    assert torch.equal(outs["bgr"], outs["nv12"]) and torch.equal(outs["bgr"], outs["i420"])
    times = {f: [] for f in bufs}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for fmt in bufs:
            for _ in range(5):
                call(fmt)
            a.record()
            for _ in range(args.reps):
                call(fmt)
            b.record()
            torch.cuda.synchronize()
            times[fmt].append(a.elapsed_time(b) / args.reps * 1e3)
    for fmt, us in times.items():
        print(json.dumps({"preprocess_call": fmt, "frames": B, "src": "%dx%d" % (w, h), "dst": "512x512",
                          "us_per_call": us, "source_bytes": int(bufs[fmt].numel())}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--height", type=int, default=1440)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--cv2-threads", type=int, default=-1, help="cv2.setNumThreads (-1: cv2's default)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("yuv_input.py measures on a CUDA device; none is available")
    import cv2
    if args.cv2_threads >= 0:
        cv2.setNumThreads(args.cv2_threads)
    dev = torch.device("cuda")
    h, w = args.height, args.width
    print(json.dumps({"gpu": gpu_state(), "cv2_threads": cv2.getNumThreads(), "host_cpus": os.cpu_count()}))
    pool = [torch.from_numpy(f).pin_memory() for f in nv12_frames(4, h, w, seed=800)]
    total = args.steps + args.warmup

    det = make_detector(dev, tracking=True)
    cam = synth.default_camera(w, h)
    for S in args.slots:
        steps = [[pool[(t + s) % 4] for s in range(S)] for t in range(total)]
        workload("track-%d" % S, det,
                 lambda pf: cpb.TrackPipeline(det, slots=S, camera_matrix=cam, pixel_format=pf),
                 lambda pipe, frames, i: pipe.submit(list(frames), new_video=[i == 0] * S),
                 steps, S, h, w, args)
    del det

    det = make_detector(dev, tracking=False)
    B = args.batch
    batches = [torch.stack([pool[(t + b) % 4] for b in range(B)]).pin_memory() for t in range(4)]
    workload("batch-%d" % B, det,
             lambda pf: cpb.BatchPipeline(det, batch=B, height=h, width=w, camera_matrix=cam, pixel_format=pf),
             lambda pipe, frames, i: pipe.submit(frames), [batches[t % 4] for t in range(total)], B, h, w, args)
    kernel_times(dev, h, w, args)


if __name__ == "__main__":
    main()
