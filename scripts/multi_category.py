"""Multi-category inference: one multi-model plan against M single-model plans called back to back on one stream.

    python scripts/multi_category.py [--out table.json]

512 x 512, tf32x3, M in {1, 3, 9} categories x per-category batch in {1, 4, 8}; forward + decode + PnP (cp_infer /
cp_infer_multi) of seeded, calibrated checkpoints over the same frames; CUDA events around 20 steps after 5 warm-up
steps.  Prints the card, its power limit and max SM clock (read in the same run) and one row per configuration:
images/s counts M x batch category-images per step.  A configuration whose plans do not fit is reported as not
measured."""
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
from centerpose_b200.engine import Engine  # noqa: E402

CATS = ["chair", "cup", "laptop", "bottle", "book", "camera", "bike", "shoe", "cereal_box"]
WARMUP, STEPS, H, W, PREC = 5, 20, 512, 512, "tf32x3"


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = _card()
    print("card:", card)
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    x1 = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(8, H, W, seed=3))).cuda()
    sds = []
    for i in range(len(CATS)):
        m.load_state_dict(synth.seeded_state_dict(m, seed=100 + i, offset_std=0.3))
        synth.calibrate_head_bias(m, m(x1)[-1], target=4)
        sds.append({k: v.detach().clone() for k, v in m.state_dict().items()})
    cam = synth.default_camera(W, H)
    rows = []
    print("%3s %5s | %10s %9s %12s | %10s %9s %12s | %7s" % ("M", "batch", "multi img/s", "ms/step", "plan bytes",
                                                             "M x 1 img/s", "ms/step", "plan bytes", "speedup"))
    for M in (1, 3, 9):
        prms = [cpb.decode_params(opt, c=c) for c in CATS[:M]]
        for B in (1, 4, 8):
            x = x1[:B]
            meta = cpb.make_meta(B, np.array([W / 2., H / 2.], np.float32), float(W), W, H, cam, device="cuda")
            row = dict(M=M, batch=B)
            engs = []
            try:
                multi = Engine("dla_34", m.heads, m.head_conv, B, H, W, 0, precision=PREC, models=M)
                engs.append(multi)
                for i in range(M):
                    multi.load_state_dict(sds[i], model=i)
                po = torch.empty((M, B, opt.K, 192), device="cuda")
                nv = torch.empty((M, B), dtype=torch.int32, device="cuda")
                ms = _time(lambda: multi.infer(x, meta, prms if M > 1 else prms[0], poses=po if M > 1 else po[0],
                                               n_valid=nv if M > 1 else nv[0]))
                row.update(multi_ms=ms, multi_ips=M * B * 1e3 / ms, multi_bytes=multi.plan_bytes)
                singles = []
                for i in range(M):
                    e = Engine("dla_34", m.heads, m.head_conv, B, H, W, 0, precision=PREC)
                    e.load_state_dict(sds[i])
                    singles.append(e)
                    engs.append(e)

                def seq():
                    for i, e in enumerate(singles):
                        e.infer(x, meta, prms[i], poses=po[i], n_valid=nv[i])
                ms = _time(seq)
                row.update(seq_ms=ms, seq_ips=M * B * 1e3 / ms, seq_bytes=sum(e.plan_bytes for e in singles))
                print("%3d %5d | %10.1f %9.3f %12d | %10.1f %9.3f %12d | %6.2fx" % (
                    M, B, row["multi_ips"], row["multi_ms"], row["multi_bytes"], row["seq_ips"], row["seq_ms"],
                    row["seq_bytes"], row["seq_ms"] / row["multi_ms"]))
            except (RuntimeError, torch.cuda.OutOfMemoryError) as ex:
                row["not_measured"] = str(ex)[:200]
                print("%3d %5d | not measured: %s" % (M, B, row["not_measured"]))
            for e in engs:
                e.close()
            torch.cuda.empty_cache()
            rows.append(row)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=card, precision=PREC, height=H, width=W, warmup=WARMUP, steps=STEPS, rows=rows), f,
                      indent=1)


if __name__ == "__main__":
    main()
