"""Per-layer fp64 parity of every launch the plan makes, teacher-forced, at the benched shapes and in all four precisions.

The whole-network tests compare heads after ~50 layers and 16 deformable samplings, which amplify rounding ~2000x, so
their bars cannot see a subtle error in one launch.  Here the plan is stepped one op at a time (cp_plan_run_ops): before
an op runs its inputs are read from the arena exactly as the plan produced them, the op is evaluated in fp64 from those
inputs (tests/layer_ref.py), the op runs, and its output is scored against that reference with the per-element metric
r = max |got - ref| / S.  Frames are independent, so references are taken for the first and the last frame only.
Run with -s for the per-op table (op, family, BN, ksplit, r).
"""
import os

import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib, synth
from centerpose_b200.engine import Engine, _device_view
from tests import layer_ref
from tests.util import LAYER_CEIL, LAYER_DISCRIMINATION, golden, net_case_inputs

pytestmark = pytest.mark.gpu

# (arch, tracking_task, H, W, batch, max_batch, precisions)
CONFIGS = [
    ("dla_34", False, 512, 512, 1, 4, ("fp32", "tf32x3", "tf32", "bf16")),
    ("dla_34", False, 512, 512, 3, 4, ("fp32", "tf32x3", "tf32", "bf16")),
    ("dla_34", True, 256, 256, 2, 2, ("fp32", "tf32x3")),
    ("dlav1_34", True, 128, 160, 2, 2, ("fp32", "tf32x3", "tf32")),
]
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


def step_and_score(arch, trk, H, W, batch, max_batch, prec):
    """Run the schedule op by op; returns one record per op (name, family, BN, ksplit, K, r, ceiling key)."""
    eng, opt, _ = _engine(arch, trk, H, W, max_batch, prec)
    descs = eng.op_descs()
    x, ext = _inputs(eng, batch)
    heads = _heads(eng, batch)
    rd = layer_ref.ActReader(eng.arena(), ext, sorted({0, batch - 1}), max_batch)
    frames = rd.frames
    names = eng.head_names
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
        recs.append(dict(config="%s%s %dx%d b%d/%d %s" % (arch, "+trk" if trk else "", H, W, batch, max_batch, prec),
                         prec=prec, index=i, name=d["name"], family=d["family"], x3=d["x3"], kind=d["kind"],
                         BN=li["BN"], ksplit=li["ksplit"], grid=li["grid"], K=K, r=r, ceil=_ceiling(d, prec),
                         nsrc=d["nsrc"], has_res=d["has_res"], res_after_relu=d["res_after_relu"],
                         out_head=d["out_head"], fuse_heads=d["fuse_heads"], has_skip=d["has_skip"],
                         first_step=d["first_step"]))
    eng.close()
    return recs


@pytest.fixture(scope="module")
def layer_records(cplib):
    recs = []
    for arch, trk, H, W, b, mb, precs in CONFIGS:
        for prec in precs:
            recs += step_and_score(arch, trk, H, W, b, mb, prec)
    print("\n%-36s %-42s %-11s %3s %4s %3s %10s %9s" % ("config", "op", "family", "x3", "BN", "ks", "r", "ceiling"))
    for q in recs:
        print("%-36s %-42s %-11s %3d %4d %3d %10.3e %9.1e" % (q["config"], q["name"][:42], FAM[q["family"]], q["x3"],
                                                            q["BN"], q["ksplit"], q["r"], LAYER_CEIL[q["ceil"]]))
    worst = {}
    for q in recs:
        if q["r"] >= worst.get(q["ceil"], {"r": -1.0})["r"]:
            worst[q["ceil"]] = q
    for k, q in sorted(worst.items()):
        print("worst r, ceiling %-5s: %.3e (ceiling %.1e) at %s %s (%s)" % (k, q["r"], LAYER_CEIL[k], q["config"],
                                                                          q["name"], FAM[q["family"]]))
    return recs


def test_every_op_under_its_ceiling(layer_records):
    bad = [q for q in layer_records if not q["r"] <= LAYER_CEIL[q["ceil"]]]
    assert not bad, "\n".join("%s op %d %s (%s BN %d ksplit %d): r %.3e > %.1e" % (
        q["config"], q["index"], q["name"], FAM[q["family"]], q["BN"], q["ksplit"], q["r"], LAYER_CEIL[q["ceil"]])
        for q in bad)


def test_bound_discriminates_tf32_from_tf32x3(layer_records):
    """Single-pass tf32 must score far above the fp32 / tf32x3 ceiling on every tensor-core op with K >= 288: a tf32x3
    kernel that lost its lo terms on some tile would fail that ceiling.  The fused-heads conv is left out: its heads
    are scored through the 1x1 with |W1| (S_hidden + |hidden|), which does not let the random-sign hidden errors
    cancel, so single-pass tf32 scores only ~3 fp32 ceilings there."""
    tf = [q for q in layer_records if q["prec"] == "tf32" and q["family"] in TC_FAMILIES and not q["x3"]
          and q["K"] >= 288 and not q["fuse_heads"]]
    assert tf
    factor = min(q["r"] for q in tf) / LAYER_CEIL["fp32"]
    print("tf32-vs-tf32x3 discrimination: min r(tf32) / fp32 ceiling = %.1f over %d launches" % (factor, len(tf)))
    weak = [q for q in tf if q["r"] < LAYER_DISCRIMINATION * LAYER_CEIL["fp32"]]
    assert not weak, ["%s %s r %.3e" % (q["config"], q["name"], q["r"]) for q in weak]


def test_launch_coverage(layer_records):
    """The configurations reach every kernel path the plan has (upsampling always carries a skip in this network); a
    schedule change that stops reaching one fails here instead of leaving the per-op assertions vacuous."""
    R = layer_records
    have = set()
    for q in R:
        f, p = q["family"], q["prec"]
        if f == _lib.FAM_CONV_TMA:
            have.add(("conv_tma", q["x3"], q["BN"]))
            if q["fuse_heads"]:
                have.add(("fused_heads", p))
            if q["ksplit"] > 1:
                have.add("conv_tma ksplit")
        if f == _lib.FAM_DCN_TMA:
            have.add(("dcn_tma", q["x3"]))
            if q["ksplit"] > 1:
                have.add("dcn_tma ksplit")
        if f == _lib.FAM_IGEMM_UMMA:
            have.add(("igemm_umma", "bf16" if p == "bf16" else ("x3" if q["x3"] else "tf32"), q["kind"]))
        if f in (_lib.FAM_STEM, _lib.FAM_CONV3_C16, _lib.FAM_IGEMM_FP32, _lib.FAM_GN_RELU):
            have.add(FAM[f])
        if q["nsrc"] > 1:
            have.add("multi-source")
        if q["has_res"]:
            have.add("residual after relu" if q["res_after_relu"] else "residual before relu")
        if q["out_head"] >= 0:
            have.add("nchw head")
        if f == _lib.FAM_UPADD:
            have.add("upsample+skip" if q["has_skip"] else "upsample")
        if f == _lib.FAM_GRU:
            have.add("gru first step" if q["first_step"] else "gru later step")
    need = {("conv_tma", x3, bn) for x3 in (0, 1) for bn in (32, 64, 128)}
    need |= {("fused_heads", "tf32"), ("fused_heads", "tf32x3"), "conv_tma ksplit", "dcn_tma ksplit",
             ("dcn_tma", 0), ("dcn_tma", 1), ("igemm_umma", "bf16", 1), ("igemm_umma", "bf16", 2),
             ("igemm_umma", "x3", 1), ("igemm_umma", "x3", 2), "stem", "conv3_c16", "igemm_fp32", "gn_relu",
             "multi-source", "residual after relu", "residual before relu", "nchw head", "upsample+skip",
             "gru first step", "gru later step"}
    print("coverage: %s" % sorted(map(str, have)))
    assert not (need - have), "paths no configuration reaches: %s" % sorted(map(str, need - have))


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


@pytest.mark.parametrize("name", ["net_dla34_b2_96x128", "net_dlav1_b1_64x64", "net_dla34track_b1_64x96"])
def test_chained_op_references_are_the_network(name, cplib):
    """The op descriptors mean the network: the fp64 per-op references chained through the schedule (no teacher
    forcing, an fp64 arena) reproduce the fp64 oracle network, so concat order, strides, residual placement, the GRU
    routing and the head mapping are read as the plan runs them."""
    from oracle import net_ref
    g = golden(name)
    arch, trk, B, H, W = str(g["arch"]), bool(int(g["tracking"])), int(g["batch"]), int(g["H"]), int(g["W"])
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sd = _exact_bn(synth.seeded_state_dict(m, seed=int(g["wseed"]), offset_std=float(g["offset_std"])))
    eng, _, _ = _engine(arch, trk, H, W, B, "fp32", sd=sd)
    x, extra = net_case_inputs(g)
    ext = [torch.from_numpy(x).cuda().double()] + [
        torch.from_numpy(extra[k]).cuda().double() if k in extra else None for k in ("pre_img", "pre_hm", "pre_hm_hp")]
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
        sd64 = {k: v.double().cuda() if v.dtype.is_floating_point else v for k, v in sd.items()}
        want = net_ref.forward(ext[0], sd64, opt.heads, arch, pre_img=ext[1], pre_hm=ext[2], pre_hm_hp=ext[3],
                               tracking_task=trk)
    eng.close()
    assert sorted(heads) == sorted(want)
    for h in want:
        e = float((heads[h] - want[h]).abs().max()) / max(1e-30, float(want[h].abs().max()))
        print("%s head %-18s chained-vs-oracle %.2e" % (name, h, e))
        assert e <= 1e-10, (h, e)


@pytest.mark.parametrize("pdl", ["CP_NO_PDL", "CP_PDL"])
def test_stepping_is_the_forward(pdl, cplib):
    """cp_plan_run_ops over the whole schedule computes what cp_forward computes, bit for bit, with PDL off or on."""
    old = {k: os.environ.pop(k, None) for k in ("CP_NO_PDL", "CP_PDL")}
    os.environ[pdl] = "1"
    try:
        eng, _, _ = _engine("dla_34", False, 512, 512, 4, "tf32x3")
        x, ext = _inputs(eng, 2)
        a = eng.forward(x)
        b = _heads(eng, 2)
        recs = eng.run_ops(x, 0, len(eng.op_descs()), b)
        torch.cuda.synchronize()
        eng.close()
    finally:
        os.environ.pop(pdl, None)
        for k, v in old.items():
            if v is not None:
                os.environ[k] = v
    assert len(recs) > 0
    for h in a:
        assert torch.equal(a[h], b[h]), h
