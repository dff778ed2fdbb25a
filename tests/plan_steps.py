"""Stepping the plan one op at a time and scoring each op against its fp64 reference (tests/layer_ref.py), shared by
tests/test_gpu_plan_layers.py (the benched shapes) and tests/test_gpu_plan_geometry.py (the keep_res / fix_short
shapes and the benched batch of 32)."""
import os

import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib, synth
from centerpose_b200.engine import Engine, _device_view
from tests import layer_ref
from tests.util import LAYER_CEIL

FAM = _lib.FAMILY_NAMES
TC_FAMILIES = (_lib.FAM_IGEMM_UMMA, _lib.FAM_CONV_TMA, _lib.FAM_DCN_TMA)


def _engine(arch, trk, H, W, max_batch, prec, sd=None, wseed=11):
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    if sd is None:
        sd = synth.seeded_state_dict(m, seed=wseed, offset_std=0.3)
    eng = Engine(m._arch(), m.heads, m.head_conv, max_batch, H, W, 0, tracking=m.tracking_inputs,
                 tracking_task_gru=m.use_convGRU and m.tracking_task, precision=prec)
    eng.load_state_dict(sd)
    return eng, opt, sd


def _inputs(eng, batch, seed=317):
    H, W = eng.height, eng.width
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(batch, H, W, seed=seed))).cuda()
    if not eng.tracking:
        return x, [x, None, None, None]
    g = torch.Generator(device="cuda").manual_seed(seed)
    pre_img = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(batch, H, W, seed=seed + 1))).cuda()
    pre_hm = torch.rand((batch, 1, H, W), device="cuda", generator=g)
    pre_hm_hp = torch.rand((batch, 8, H, W), device="cuda", generator=g)
    return x, [x, pre_img, pre_hm, pre_hm_hp]


def _heads(eng, batch):
    return {n: torch.full((batch, c, eng.height // 4, eng.width // 4), float("nan"), device="cuda")
            for n, c in eng.heads.items()}


def _fetch(ptr, n):
    return _device_view(ptr, n, torch.device("cuda", 0))


def _ceiling(d, prec):
    """LAYER_CEIL key of the arithmetic op `d` runs in."""
    if d["family"] == _lib.FAM_MAXPOOL:
        return "exact"
    if d["family"] in TC_FAMILIES and not d["x3"]:
        return "bf16" if prec == "bf16" else "tf32"
    return "fp32"


def _exact_bn(sd):
    """BatchNorm parameters whose fold is exact in fp32 and fp64 alike (mean 0, var 2^40, gamma 2^20: scale 1, shift
    beta), and no conv bias in front of a BatchNorm, so the plan's packed matrices are the state dict's weights."""
    out = dict(sd)
    for k in sd:
        if k.endswith(".running_mean"):
            p = k[:-len(".running_mean")]
            out[k] = torch.zeros_like(sd[k])
            out[p + ".running_var"] = torch.full_like(sd[k], 2.0 ** 40)
            out[p + ".weight"] = torch.full_like(sd[k], 2.0 ** 20)
            cb = p.replace(".actf.0", ".conv.bias")
            if cb != p and cb in sd:
                out[cb] = torch.zeros_like(sd[cb])
    return out


class _env(object):
    """Set the environment switches `env` ({name: value}) for the duration of a with block, then restore them."""

    def __init__(self, env):
        self.env = dict(env or {})

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.env}
        os.environ.update({k: str(v) for k, v in self.env.items()})

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        return False


def step_and_score(arch, trk, H, W, batch, max_batch, prec, env=None, label=None):
    """Run the schedule op by op; returns one record per op (name, family, BN, ksplit, grid, K, r, ceiling key and the
    op's geometry).  env: environment switches ({name: value}) set while the plan is created, where the plan reads
    them (CP_NO_DCN_TMA).  label: the record's config name (default: arch, size, batch, prec)."""
    with _env(env):
        eng, opt, _ = _engine(arch, trk, H, W, max_batch, prec)
    descs = eng.op_descs()
    x, ext = _inputs(eng, batch)
    heads = _heads(eng, batch)
    rd = layer_ref.ActReader(eng.arena(), ext, sorted({0, batch - 1}), max_batch)
    frames = rd.frames
    names = eng.head_names
    config = label or "%s%s %dx%d b%d/%d %s" % (arch, "+trk" if trk else "", H, W, batch, max_batch, prec)
    recs = []
    for i, d in enumerate(descs):
        with torch.no_grad():
            want = layer_ref.op_ref(d, rd, _fetch, descs)
        li = eng.run_ops(x, i, i + 1, heads, *ext[1:])[0]
        torch.cuda.synchronize()
        if d["fused_away"]:
            assert li["family"] == _lib.FAM_NONE
            continue
        assert li["family"] == d["family"], (d["name"], li, d["family"])
        r = 0.0
        for (kind, tgt), ref, S in want:
            got = rd.get(tgt) if kind == "act" else heads[names[tgt]][frames].double()
            if d["family"] == _lib.FAM_MAXPOOL:
                r = max(r, 0.0 if torch.equal(got, ref) else float("inf"))
            else:
                r = max(r, layer_ref.score(got, ref, S))
        K = d["kh"] * d["kh"] * d["Cin"] if d["kind"] in (0, 1, 2) else 0
        src = d["src"][0]
        out = d["out"] if d["out_head"] < 0 else dict(H=H // 4, W=W // 4)
        recs.append(dict(config=config, prec=prec, batch=batch, index=i, name=d["name"], family=d["family"],
                         x3=d["x3"], kind=d["kind"], BN=li["BN"], ksplit=li["ksplit"], grid=li["grid"], K=K, r=r,
                         ceil=_ceiling(d, prec), nsrc=d["nsrc"], has_res=d["has_res"],
                         res_after_relu=d["res_after_relu"], out_head=d["out_head"], fuse_heads=d["fuse_heads"],
                         has_skip=d["has_skip"], first_step=d["first_step"], kh=d["kh"], stride=d["stride"],
                         Cin=d["Cin"], Cout=d["Cout"], CoutPad=d["CoutPad"], n_children=d["n_children"],
                         srcH=src["H"], srcW=src["W"], outH=out["H"], outW=out["W"]))
    eng.close()
    return recs


def chained_heads(eng, ext, B):
    """The fp64 per-op references chained through the schedule (no teacher forcing, an fp64 arena) from the external
    inputs `ext` (four NCHW float64 tensors or None) of B frames: {head name: [B,C,H/4,W/4] float64}."""
    arena64 = torch.zeros(eng.arena().numel(), dtype=torch.float64, device="cuda")
    rd = layer_ref.ActReader(arena64, ext, range(B), B)
    descs = eng.op_descs()
    heads = {}
    with torch.no_grad():
        for d in descs:
            for (kind, tgt), ref, _ in layer_ref.op_ref(d, rd, _fetch, descs, fp32_pos=False):
                if kind == "act":
                    rd.put(tgt, ref)
                else:
                    heads[eng.head_names[tgt]] = ref
    return heads


def print_records(recs):
    """The per-op table and the worst r per ceiling (run pytest with -s)."""
    print("\n%-36s %-42s %-11s %3s %4s %3s %10s %9s" % ("config", "op", "family", "x3", "BN", "ks", "r", "ceiling"))
    for q in recs:
        print("%-36s %-42s %-11s %3d %4d %3d %10.3e %9.1e" % (q["config"], q["name"][:42], FAM[q["family"]], q["x3"],
                                                            q["BN"], q["ksplit"], q["r"], LAYER_CEIL[q["ceil"]]))
    print_worst(recs)


def print_worst(recs, title=""):
    """The worst r per ceiling over `recs`."""
    worst = {}
    for q in recs:
        if q["r"] >= worst.get(q["ceil"], {"r": -1.0})["r"]:
            worst[q["ceil"]] = q
    for k, q in sorted(worst.items()):
        print("%sworst r, ceiling %-5s: %.3e (ceiling %.1e) at %s %s (%s)" % (title, k, q["r"], LAYER_CEIL[k], q["config"],
                                                                            q["name"], FAM[q["family"]]))


def over_ceiling(recs):
    """Failure lines of the ops whose r exceeds their ceiling (empty when every op is under it)."""
    return ["%s op %d %s (%s BN %d ksplit %d): r %.3e > %.1e" % (
        q["config"], q["index"], q["name"], FAM[q["family"]], q["BN"], q["ksplit"], q["r"], LAYER_CEIL[q["ceil"]])
        for q in recs if not q["r"] <= LAYER_CEIL[q["ceil"]]]


def weak_discrimination(recs, floor):
    """Single-pass tf32 tensor-core launches with K >= 288 (fused heads left out, see test_gpu_plan_layers) and the
    ones among them scoring under `floor`: (candidates, weak)."""
    tf = [q for q in recs if q["prec"] == "tf32" and q["family"] in TC_FAMILIES and not q["x3"]
          and q["K"] >= 288 and not q["fuse_heads"]]
    return tf, [q for q in tf if q["r"] < floor]
