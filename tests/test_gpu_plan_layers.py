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
from tests.plan_steps import (FAM, TC_FAMILIES, _engine, _exact_bn, _heads, _inputs, chained_heads, over_ceiling,
                              print_records, step_and_score)
from tests.util import LAYER_CEIL, LAYER_DISCRIMINATION, golden, net_case_inputs

pytestmark = pytest.mark.gpu

# (arch, tracking_task, H, W, batch, max_batch, precisions)
CONFIGS = [
    ("dla_34", False, 512, 512, 1, 4, ("fp32", "tf32x3", "tf32", "bf16")),
    ("dla_34", False, 512, 512, 3, 4, ("fp32", "tf32x3", "tf32", "bf16")),
    ("dla_34", True, 256, 256, 2, 2, ("fp32", "tf32x3")),
    ("dlav1_34", True, 128, 160, 2, 2, ("fp32", "tf32x3", "tf32")),
]


@pytest.fixture(scope="module")
def layer_records(cplib):
    recs = []
    for arch, trk, H, W, b, mb, precs in CONFIGS:
        for prec in precs:
            recs += step_and_score(arch, trk, H, W, b, mb, prec)
    print_records(recs)
    return recs


def test_every_op_under_its_ceiling(layer_records):
    bad = over_ceiling(layer_records)
    assert not bad, "\n".join(bad)


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
    heads = chained_heads(eng, ext, B)
    with torch.no_grad():
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
