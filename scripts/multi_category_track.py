"""Multi-category tracking: one MultiCategoryTracker step against M ObjectPoseDetector tracking steps back to back, and
one cp_tracker_step over M x S streams against M calls of S streams.

    python scripts/multi_category_track.py [--out table.json]

512 x 512, tf32x3, seeded and calibrated CenterPoseTrack checkpoints, uint8 frames resident on the device, M in {1, 3, 9}
categories x S in {1, 8} slots; CUDA events around 20 steps after 5 warm-up steps.  A whole step is pre-process, render,
network + decode + PnP and the tracker step (run_batch(track=True, to_host=False)).  The tracker-only rows step ~10
tracks per stream (scripts/track_step_time.py's records).  Prints the card, its power limit and max SM clock (read in the
same run).  A configuration that does not fit is reported as not measured.  Checkpoints go to a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import synth  # noqa: E402
from track_step_time import records  # noqa: E402

CATS = ["chair", "cup", "laptop", "bottle", "book", "camera", "bike", "shoe", "cereal_box"]
WARMUP, STEPS, H, W = 5, 20, 512, 512


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def _time(step):
    for _ in range(WARMUP):
        step()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(STEPS):
        step()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / STEPS


def _checkpoints(opt, tmp):
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, H, W, seed=3))).cuda()
    z = torch.zeros((2, 1, H, W), device="cuda")
    paths = {}
    for i, c in enumerate(CATS):
        m.load_state_dict(synth.seeded_state_dict(m, seed=100 + i, offset_std=0.3))
        synth.calibrate_head_bias(m, m(x, x, z, z.repeat(1, 8, 1, 1))[-1], target=4)
        paths[c] = os.path.join(tmp, c + ".pth")
        cpb.save_model(paths[c], 1, m)
    return paths


def _oom(e):
    return isinstance(e, torch.cuda.OutOfMemoryError) or "out of memory" in str(e).lower()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = _card()
    print("card:", card)
    opt = cpb.default_opt("dla_34", tracking_task=True)
    tmp = tempfile.mkdtemp(prefix="cp_mct_")
    paths = _checkpoints(opt, tmp)
    cam = synth.default_camera(W, H)
    rows = []
    print("%2s %2s | %12s %12s %7s | %12s %12s %7s" % ("M", "S", "step multi", "step M x 1", "speedup",
                                                       "trk multi", "trk M x 1", "speedup"))
    for M in (1, 3, 9):
        cats = CATS[:M]
        for S in (1, 8):
            frames = torch.from_numpy(synth.synthetic_frames(S, H, W, seed=11)).cuda()
            row = dict(M=M, S=S)
            try:
                multi = cpb.MultiCategoryTracker(opt, {c: paths[c] for c in cats})
                row["step_multi_ms"] = _time(lambda: multi.run_batch(frames, cam, to_host=False))
                del multi
                singles = [cpb.ObjectPoseDetector(cpb.default_opt("dla_34", tracking_task=True, c=c, load_model=paths[c]))
                           for c in cats]
                row["step_singles_ms"] = _time(lambda: [d.run_batch(frames, cam, track=True, to_host=False)
                                                        for d in singles])
                del singles
            except RuntimeError as e:
                if not _oom(e):
                    raise
                row["step_multi_ms"] = row["step_singles_ms"] = None
            torch.cuda.empty_cache()
            # the tracker alone: M x S streams in one cp_tracker_step against M calls of S streams
            rng = np.random.default_rng(0)
            meta = cpb.make_meta(M * S, np.array([256., 256.], np.float32), 512.0, 512, 512, cam).cuda()
            recs = [torch.from_numpy(records(rng, M * S, 10)).cuda() for _ in range(4)]
            nv = torch.full((M * S,), 10, dtype=torch.int32, device="cuda")
            tm = cpb.Tracker(opt, streams=S, categories=cats)
            ts = [cpb.Tracker(opt, streams=S) for _ in cats]
            it = [0]

            def multi_step():
                tm.step_records(recs[it[0] % 4], nv, meta)
                it[0] += 1

            def single_steps():
                r = recs[it[0] % 4]
                for m, t in enumerate(ts):
                    t.step_records(r[m * S:(m + 1) * S], nv[m * S:(m + 1) * S], meta[m * S:(m + 1) * S])
                it[0] += 1
            row["trk_multi_ms"] = _time(multi_step)
            it[0] = 0
            row["trk_singles_ms"] = _time(single_steps)
            del tm, ts
            rows.append(row)
            f = lambda v: "not measured" if v is None else "%.3f ms" % v      # noqa: E731
            sp = lambda a, b: "-" if a is None or b is None else "%.2fx" % (b / a)      # noqa: E731
            print("%2d %2d | %12s %12s %7s | %12s %12s %7s" % (
                M, S, f(row["step_multi_ms"]), f(row["step_singles_ms"]), sp(row["step_multi_ms"], row["step_singles_ms"]),
                f(row["trk_multi_ms"]), f(row["trk_singles_ms"]), sp(row["trk_multi_ms"], row["trk_singles_ms"])),
                flush=True)
    if args.out:
        with open(args.out, "w") as fp:
            json.dump({"card": card, "rows": rows}, fp, indent=1)


if __name__ == "__main__":
    main()
