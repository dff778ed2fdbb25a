"""Time cp_tracker_step (CUDA events) at 8 streams with ~10 and ~100 tracks per stream, greedy vs hungarian
association, default CenterPoseTrack options (filter, scale pool, second PnP).  Prints one JSON line per case with the
card name and power limit.

    python scripts/track_step_time.py [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import centerpose_b200 as cpb                      # noqa: E402
from centerpose_b200 import _lib as L              # noqa: E402


def records(rng, B, n, K=128):
    """n detections per stream on a jittered grid: each frame's detection i is near track i of the previous frame."""
    r = np.zeros((B, K, L.CP_POSE_RECORD), np.float32)
    g = np.stack(np.meshgrid(np.arange(12), np.arange(12)), -1).reshape(-1, 2)[:n] * 40.0 + 30.0
    for b in range(B):
        c = g + rng.normal(size=g.shape) * 2.0
        r[b, :n, L.P_SCORE] = 0.9
        r[b, :n, L.P_CT:L.P_CT + 2] = c
        r[b, :n, L.P_BBOX:L.P_BBOX + 2] = c - 15
        r[b, :n, L.P_BBOX + 2:L.P_BBOX + 4] = c + 15
        kp = c[:, None, :] + rng.normal(size=(n, 8, 2)) * 10
        for off in (L.P_KPS, L.P_KPS_DISP_MEAN, L.P_KPS_HM_MEAN):
            r[b, :n, off:off + 16] = kp.reshape(n, 16)
        r[b, :n, L.P_KPS_DISP_STD:L.P_KPS_DISP_STD + 16] = 2.0
        r[b, :n, L.P_KPS_HM_STD:L.P_KPS_HM_STD + 16] = 1.0
        r[b, :n, L.P_OBJ_SCALE:L.P_OBJ_SCALE + 3] = [0.8, 1.0, 0.6]
        r[b, :n, L.P_OBJ_SCALE_UNC:L.P_OBJ_SCALE_UNC + 3] = 0.1
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    rng = np.random.default_rng(0)
    B = 8
    meta = cpb.make_meta(B, np.array([256., 256.], np.float32), 512.0, 512, 512, np.array(
        [[615.0, 0, 256.0], [0, 615.0, 256.0], [0, 0, 1]])).cuda()
    for n in (10, 100):
        frames = [torch.from_numpy(records(rng, B, n)).cuda() for _ in range(4)]
        nv = torch.full((B,), n, dtype=torch.int32, device="cuda")
        for hung in (False, True):
            opt = cpb.default_opt("dla_34", tracking_task=True)
            opt.hungarian = hung
            trk = cpb.Tracker(opt, streams=B)
            for f in range(10):
                tr, nt = trk.step_records(frames[f % 4], nv, meta)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for f in range(args.iters):
                trk.step_records(frames[f % 4], nv, meta, out=(tr, nt))
            e1.record()
            torch.cuda.synchronize()
            print(json.dumps({"streams": B, "tracks_per_stream": int(nt.float().mean().item()),
                              "association": "hungarian" if hung else "greedy",
                              "step_ms": round(e0.elapsed_time(e1) / args.iters, 4), "card": card}), flush=True)
            trk.close()


if __name__ == "__main__":
    main()
