"""Device memory of a plan with the full activation arena and with the liveness-packed one (CP_PLAN_REUSE_ACTIVATIONS).

    python scripts/plan_memory.py            # byte tables, on the host (cp_plan_memory), no GPU needed
    python scripts/plan_memory.py --time     # + the timings below, on cuda:0

The tables cover dla_34, dlav1_34 and dla_34 tracking at 512 x 512 in tf32x3, batch 1 / 8 / 32 and M = 1 / 3 / 9 models.
--time times, full against reuse in alternation (three rounds each, CUDA events around 20 cp_infer calls after 5
warm-up calls): dla_34 512 x 512 tf32x3 at batch 1 and 32; then one MultiCategoryTracker step (run_batch, to_host=False)
of M = 9 seeded tracking checkpoints over S = 32 slots, which fits only with reuse: the full-arena step is reported as
not measured with its dry-run bytes.  Prints the card, its power limit and max SM clock, read in the same run.
Checkpoints go to a temporary directory."""
import argparse
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200.engine import plan_memory  # noqa: E402

CATS = ["chair", "cup", "laptop", "bottle", "book", "camera", "bike", "shoe", "cereal_box"]
ARCHS = [("dla_34", False), ("dlav1_34", False), ("dla_34", True)]
H = W = 512
GB = 1e9


def _mem(arch, trk, B, M, reuse):
    opt = cpb.default_opt(arch, tracking_task=trk)
    return plan_memory(arch, opt.heads, opt.head_conv, B, H, W, tracking=trk, tracking_task_gru=arch == "dlav1_34" and trk,
                       precision="tf32x3", models=M, reuse_activations=reuse)


def tables():
    print("%-14s %2s %3s | %10s %10s | %10s %10s | %8s %8s %9s" % (
        "arch", "M", "B", "act full", "act reuse", "all full", "all reuse", "weights", "tiles", "workspace"))
    for arch, trk in ARCHS:
        for M in (1, 3, 9):
            for B in (1, 8, 32):
                f, r = _mem(arch, trk, B, M, False), _mem(arch, trk, B, M, True)
                print("%-14s %2d %3d | %8.2f GB %8.2f GB | %8.2f GB %8.2f GB | %5.2f GB %5.2f GB %6.2f GB" % (
                    arch + ("+trk" if trk else ""), M, B, f["activation"] / GB, r["activation"] / GB, f["total"] / GB,
                    r["total"] / GB, f["weights"] / GB, f["tiles"] / GB, f["workspace"] / GB))


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown card"


def _time(step, warmup=5, steps=20):
    import torch
    for _ in range(warmup):
        step()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(steps):
        step()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / steps


def timings():
    import torch
    from centerpose_b200 import synth
    from centerpose_b200.engine import Engine
    print("card:", _card())
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sd = synth.seeded_state_dict(m, seed=1, offset_std=0.3)
    prm = cpb.decode_params(opt)
    for B in (1, 32):
        engs = {}
        for reuse in (False, True):
            engs[reuse] = Engine("dla_34", m.heads, m.head_conv, B, H, W, 0, precision="tf32x3", reuse_activations=reuse)
            engs[reuse].load_state_dict(sd)
        x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(B, H, W, seed=2))).cuda()
        meta = cpb.make_meta(B, [W / 2, H / 2], float(W), W, H, synth.default_camera(W, H), device="cuda")
        ms = {False: [], True: []}
        for _ in range(3):
            for reuse in (False, True):
                ms[reuse].append(_time(lambda: engs[reuse].infer(x, meta, prm)))
        for reuse in (False, True):
            e = engs[reuse]
            print("dla_34 tf32x3 B=%2d %-5s arena %7.1f MB: cp_infer %s ms" % (
                B, "reuse" if reuse else "full", e.memory["activation"] / 1e6, " / ".join("%.3f" % v for v in ms[reuse])))
        del engs
        torch.cuda.empty_cache()
    # one MultiCategoryTracker step, M = 9 categories x S = 32 slots
    M, S = 9, 32
    topt = cpb.default_opt("dla_34", tracking_task=True)
    full = _mem("dla_34", True, S, M, False)
    print("MultiCategoryTracker M=%d S=%d full arena: %.1f GB in all (dry run), does not fit: not measured" % (
        M, S, full["total"] / GB))
    tm = cpb.create_model(topt.arch, topt.heads, topt.head_conv, topt).cuda()
    x2 = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, H, W, seed=3))).cuda()
    z = torch.zeros((2, 1, H, W), device="cuda")
    tmp = tempfile.mkdtemp(prefix="cp_planmem_")
    paths = {}
    for i, c in enumerate(CATS[:M]):
        tm.load_state_dict(synth.seeded_state_dict(tm, seed=100 + i, offset_std=0.3))
        synth.calibrate_head_bias(tm, tm(x2, x2, z, z.repeat(1, 8, 1, 1))[-1], target=4)
        paths[c] = os.path.join(tmp, c + ".pth")
        cpb.save_model(paths[c], 1, tm)
    del tm
    torch.cuda.empty_cache()
    det = cpb.MultiCategoryTracker(topt, paths)
    frames = torch.from_numpy(synth.synthetic_frames(S, H, W, seed=11)).cuda()
    cam = synth.default_camera(W, H)
    ms = [_time(lambda: det.run_batch(frames, cam, to_host=False), warmup=3, steps=10) for _ in range(3)]
    print("MultiCategoryTracker M=%d S=%d reuse arena %.1f GB (%.1f GB in all): step %s ms, peak allocated by torch "
          "%.1f GB" % (M, S, det._eng.memory["activation"] / GB, det._eng.memory["total"] / GB,
                       " / ".join("%.1f" % v for v in ms), torch.cuda.max_memory_allocated() / GB))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--time", action="store_true", help="also time full against reuse on cuda:0")
    args = ap.parse_args()
    tables()
    if args.time:
        timings()


if __name__ == "__main__":
    main()
