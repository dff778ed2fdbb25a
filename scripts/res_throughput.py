"""Network throughput of the ResNet backbones next to dla_34, on the GPU (the table in README.md "ResNet backbones").

    python scripts/res_throughput.py [--batch 32] [--size 512] [--warmup 5] [--steps 20]

For res_18, res_50, res_101 and dla_34, in tf32x3 and tf32, at batch 32 and 512 x 512 (seeded weights, default heads,
head_conv 64 for the ResNets and 256 for DLA as opts.py:344-345 sets them):
  * images/s of the network forward (cp_forward), timed with CUDA events over `--steps` calls after `--warmup`;
  * the share of the forward's per-launch time (one cp_plan_profile, events between the launches) spent in the three
    transposed convs and in the stem (the 7x7 convs and the 3x3/2 max-pool; DLA: its 7x7 stem);
  * the fraction of the tf32x3 compute bound: algorithmic GFLOP/img x images/s over 495 / 3 TFLOP/s (the H100 SXM
    data sheet's dense TF32 rate; tf32x3 issues three tf32 products per fp32 product).
GFLOP/img is 2 x MAC at 512 x 512 with head_conv 64 as counted with hooks on the reference module (a transposed conv
counts 16 Hin Win Cin Cout MACs): 64.66 / 91.63 / 130.42 for res_18 / res_50 / res_101; dla_34 (which has no such count)
takes the plan's own count of its launches (cp_op_stat.flops), printed in the same column.  The card's name, power
limit and maximum SM clock are printed with the table.  Needs a CUDA device; there is no CPU fallback.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import centerpose_b200 as cpb          # noqa: E402
from centerpose_b200 import synth       # noqa: E402
from centerpose_b200.engine import Engine     # noqa: E402

TF32X3_PEAK = 495e12 / 3
GFLOP_512 = {"res_18": 64.66, "res_50": 91.63, "res_101": 130.42}
ARCHS = ["res_18", "res_50", "res_101", "dla_34"]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:      # the numbers still stand; the card is named by torch
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def measure(arch, prec, B, S, warmup, steps):
    opt = cpb.default_opt(arch)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    eng = Engine(m._arch(), m.heads, m.head_conv, B, S, S, 0, precision=prec, reuse_activations=True)
    eng.load_state_dict(synth.seeded_state_dict(m, seed=7, offset_std=0.3))
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(B, S, S, seed=317))).cuda()
    out = {n: torch.empty((B, c, S // 4, S // 4), device="cuda") for n, c in m.heads.items()}
    for _ in range(warmup):
        eng.forward(x, out=out)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0.record()
    for _ in range(steps):
        eng.forward(x, out=out)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / steps
    prof = eng.profile(x)
    total = sum(p["ms"] for p in prof)
    deconv = sum(p["ms"] for p in prof if p["kind"] == 3)
    stem = sum(p["ms"] for p in prof if p["kind"] == 0 or p["kind"] == 11)
    gflop = sum(p["flops"] for p in prof) / B / 1e9
    if arch in GFLOP_512 and S == 512:
        gflop = GFLOP_512[arch]
    eng.close()
    ips = B * 1e3 / ms
    return dict(arch=arch, prec=prec, ms=ms, ips=ips, deconv=deconv / total, stem=stem / total, gflop=gflop,
                bound=gflop * 1e9 * ips / TF32X3_PEAK)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("res_throughput: needs a CUDA device")
    torch.cuda.set_device(0)
    print("card: %s" % card())
    print("batch %d, %dx%d, %d warm-up + %d timed forwards per row (CUDA events)" % (a.batch, a.size, a.size, a.warmup,
                                                                                 a.steps))
    print("| arch | precision | ms / batch | images/s | transposed convs | stem | GFLOP/img | of tf32x3 bound |")
    print("|---|---|---|---|---|---|---|---|")
    for arch in ARCHS:
        for prec in ("tf32x3", "tf32"):
            r = measure(arch, prec, a.batch, a.size, a.warmup, a.steps)
            print("| %s | %s | %.2f | %.1f | %s | %.1f %% | %.2f | %.1f %% |" % (
                r["arch"], r["prec"], r["ms"], r["ips"], "%.1f %%" % (100 * r["deconv"]) if arch != "dla_34" else "-",
                100 * r["stem"], r["gflop"], 100 * r["bound"]))
            sys.stdout.flush()


if __name__ == "__main__":
    main()
