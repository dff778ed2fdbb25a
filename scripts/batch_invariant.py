"""What batch invariance costs: dla_34 at 512 x 512, tf32x3, the forward of an Engine with frames resident on the
device, at batches 1 .. 32, in three arms alternated call block by call block:
  default     the default plan (split-K chosen per launch from its tiles and the SM count)
  invariant   a CP_PLAN_BATCH_INVARIANT plan (fixed K segments: split or fold)
  nosplitk    the default plan with CP_NO_SPLITK=1 (one CTA per tile over the whole K)
Each arm runs 20 calls after 5 warm-ups per round, two rounds; the median ms per call is reported.  Then, per
split-capable launch of the invariant plan, its G, the path it took, its grid and its time at each batch
(cp_plan_run_ops stepped from op 0, CUDA events around each op).

    python scripts/batch_invariant.py [--out FILE.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import centerpose_b200 as cpb  # noqa: E402
from centerpose_b200 import _lib, synth  # noqa: E402
from centerpose_b200.engine import Engine  # noqa: E402

BATCHES = (1, 2, 4, 8, 16, 32)
PATH = {_lib.KPATH_ONE: "one", _lib.KPATH_SPLIT: "split", _lib.KPATH_FOLD: "fold", _lib.KPATH_NONE: "-"}


def _time(eng, x, n):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
    ev[0].record()
    for i in range(n):
        eng.forward(x)
        ev[i + 1].record()
    torch.cuda.synchronize()
    return [ev[i].elapsed_time(ev[i + 1]) for i in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sd = synth.seeded_state_dict(m, seed=11, offset_std=0.3)
    engs = {}
    for name, inv in (("default", False), ("invariant", True)):
        e = Engine(m._arch(), m.heads, m.head_conv, 32, 512, 512, 0, precision="tf32x3", reuse_activations=True,
                   batch_invariant=inv)
        e.load_state_dict(sd)
        engs[name] = e
    x32 = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(32, 512, 512, seed=3))).cuda()
    props = torch.cuda.get_device_properties(0)
    res = dict(device=props.name, sms=props.multi_processor_count, batches={})
    for B in BATCHES:
        x = x32[:B].contiguous()
        t = {"default": [], "invariant": [], "nosplitk": []}
        for _ in range(2):
            for arm in ("default", "invariant", "nosplitk"):
                eng = engs["invariant" if arm == "invariant" else "default"]
                if arm == "nosplitk":
                    os.environ["CP_NO_SPLITK"] = "1"
                _time(eng, x, 5)
                t[arm] += _time(eng, x, 20)
                os.environ.pop("CP_NO_SPLITK", None)
        med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
        res["batches"][B] = med
        print("batch %2d  default %.3f ms  invariant %.3f ms (%+.1f %%)  nosplitk %.3f ms" % (
            B, med["default"], med["invariant"], 100 * (med["invariant"] / med["default"] - 1), med["nosplitk"]),
            flush=True)
    # per-launch table of the split-capable launches of the invariant plan
    eng = engs["invariant"]
    n_ops = int(eng.L.cp_plan_num_ops(eng.plan))
    descs = eng.op_descs()
    rows = {}
    for B in BATCHES:
        x = x32[:B].contiguous()
        out = {k: torch.empty((B, c, 128, 128), device="cuda") for k, c in eng.heads.items()}
        eng.run_ops(x, 0, n_ops, out)          # warm-up
        for i in range(n_ops):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            li = eng.run_ops(x, i, i + 1, out)[0]
            e.record()
            torch.cuda.synchronize()
            k = eng.op_ksegments(i)
            if k["segments"] > 1:
                rows.setdefault(descs[i]["name"], dict(G=k["segments"]))[B] = dict(
                    path=PATH[k["last_path"]], grid=li["grid"], us=1000 * s.elapsed_time(e))
    print("\nlayer                               G   " + "  ".join("b%-2d path grid    us" % B for B in BATCHES))
    for name, r in rows.items():
        cells = []
        for B in BATCHES:
            c = r[B]
            cells.append("%-5s %4d %6.1f" % (c["path"], c["grid"], c["us"]))
        print("%-34s %3d   %s" % (name[:34], r["G"], "  ".join(cells)))
    res["launches"] = rows
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    for e in engs.values():
        e.close()


if __name__ == "__main__":
    main()
