"""Per-layer fp64 parity (tests/test_gpu_plan_layers.py) at the input sizes run() builds in the keep_res and fix_short
modes, and at the benched batch of 32.

The plan picks each op's kernel from its shape, so these sizes take paths the 512 x 512 configurations never reach:
  * keep_res, an 800 x 600 (h x w) portrait frame -> 832 x 608: maps 208 x 152 ... 26 x 19.  No deformable conv fits
    dcn_tma (maps <= 128 x 128 with H % 8 == 0 and W % 16 == 0), so all of them run on the igemm_umma gather kernel,
    which in both tf32 plans runs the three-pass tf32x3 arithmetic; odd 1/32 map and partial M tiles.
  * fix_short 512, a 1920 x 1440 portrait frame -> 704 x 512: the 176 x 128 and 44 x 32 / 22 x 16 deformable convs
    (H > 128, H % 8 != 0) on the gather kernel next to dcn_tma on the non-square 88 x 64 map.
  * fix_short 512, a 1080 x 1920 landscape frame -> 512 x 960: conv_tma 3 x 3 at its widest slab (W + 2 = 242, in
    tf32x3 with 16-channel slabs) and the fused heads epilogue on a 128 x 240 map.
  * keep_res, a 720 x 1280 frame -> 736 x 1312: the 184 x 328 maps are too wide for conv_tma's 3 x 3 slab, so the
    merged-heads 3 x 3 runs on the gather kernel and the per-head 1 x 1 convs run as separate conv_tma launches.
  * the benched batch (32 of 32) at 512 x 512: the persistent conv_tma / dcn_tma kernels loop over many tiles per CTA.
  * 512 x 512 with CP_NO_DCN_TMA=1: the 128 x 128 deformable convs on the gather kernel in tf32x3.
Every op is scored against LAYER_CEIL exactly as at the benched shapes.  Run with -s for the per-op table.
"""
import time

import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib, synth
from tests.plan_steps import (FAM, _engine, _exact_bn, chained_heads, over_ceiling, print_records, print_worst,
                              step_and_score, weak_discrimination)
from tests.util import LAYER_CEIL, LAYER_DISCRIMINATION

pytestmark = pytest.mark.gpu

# (name, H, W, batch, max_batch, precisions, environment switches at plan creation)
GEOMETRIES = [
    ("keep_res 832x608", 832, 608, 2, 2, ("fp32", "tf32x3", "tf32", "bf16"), None),
    ("fix_short 704x512", 704, 512, 2, 2, ("fp32", "tf32x3", "tf32"), None),
    ("fix_short 512x960", 512, 960, 2, 2, ("tf32x3", "tf32"), None),
    ("keep_res 736x1312", 736, 1312, 2, 2, ("tf32x3", "tf32"), None),
    ("batch 32", 512, 512, 32, 32, ("tf32x3", "tf32"), None),
    ("no dcn_tma", 512, 512, 2, 2, ("tf32x3",), {"CP_NO_DCN_TMA": "1"}),
]
TC = ("tf32x3", "tf32")
# the paths each geometry exists to reach (see the module docstring), per precision
NEED = {("keep_res 832x608", p, k) for p in TC for k in ("every dcn on gather", "gather dcn W>128", "gather dcn W%16")}
NEED |= {("keep_res 832x608", p, "26x19 map") for p in ("fp32", "tf32x3", "tf32", "bf16")}
NEED |= {("fix_short 704x512", p, k) for p in TC for k in ("gather dcn H>128", "gather dcn H%8", "dcn_tma non-square")}
NEED |= {("fix_short 512x960", p, k) for p in TC for k in ("conv_tma 3x3 W+2=242", "fused heads 128x240")}
NEED |= {("keep_res 736x1312", p, k) for p in TC for k in ("merged heads on gather", "unfused head 1x1 on conv_tma")}
NEED |= {("batch 32", p, k) for p in TC for k in ("conv_tma >= 4 tiles per CTA", "dcn_tma >= 4 tiles per CTA")}
NEED |= {("no dcn_tma", "tf32x3", k) for k in ("every dcn on gather", "gather dcn 128x128")}


@pytest.fixture(scope="module")
def geometry_records(cplib):
    recs = []
    for name, H, W, b, mb, precs, env in GEOMETRIES:
        for prec in precs:
            t0 = time.time()
            got = step_and_score("dla_34", False, H, W, b, mb, prec, env=env,
                                 label="%s b%d/%d %s" % (name, b, mb, prec))
            for q in got:
                q["geom"] = name
            recs += got
            print("%s %s: %d ops in %.1f s" % (name, prec, len(got), time.time() - t0))
    print_records(recs)
    for name, *_ in GEOMETRIES:
        print_worst([q for q in recs if q["geom"] == name], "%s: " % name)
    return recs


def test_every_op_under_its_ceiling(geometry_records):
    bad = over_ceiling(geometry_records)
    assert not bad, "\n".join(bad)


def test_bound_discriminates_tf32_from_tf32x3(geometry_records):
    """Single-pass tf32 scores at least LAYER_DISCRIMINATION fp32 ceilings on every single-pass tensor-core launch with
    K >= 288 at these sizes too (conv_tma and dcn_tma; the gather kernel runs tf32x3 arithmetic in both tf32 plans, so
    its launches meet the fp32 ceiling instead)."""
    tf, weak = weak_discrimination(geometry_records, LAYER_DISCRIMINATION * LAYER_CEIL["fp32"])
    assert tf
    print("tf32-vs-tf32x3 discrimination: min r(tf32) / fp32 ceiling = %.1f over %d launches"
          % (min(q["r"] for q in tf) / LAYER_CEIL["fp32"], len(tf)))
    assert not weak, ["%s %s r %.3e" % (q["config"], q["name"], q["r"]) for q in weak]


def _tiles(q):
    """Output tiles of a conv_tma / dcn_tma launch: 128-position M tiles (a lower bound for the 3 x 3 conv_tma, whose
    tiles also cover the two padding columns) times the N tiles of width BN, times the split-K factor."""
    m = -(-q["batch"] * q["outH"] * q["outW"] // 128)
    return m * (q["CoutPad"] // q["BN"]) * q["ksplit"]


def _paths(recs):
    """Coverage keys (geometry, precision, path) judged from the op records."""
    have, dcn_fams = set(), {}
    for q in recs:
        g, p, f = q["geom"], q["prec"], q["family"]
        key = lambda k: have.add((g, p, k))       # noqa: E731
        if q["kind"] == 2:
            dcn_fams.setdefault((g, p), set()).add(f)
            if f == _lib.FAM_IGEMM_UMMA and q["x3"]:
                if q["srcW"] > 128:
                    key("gather dcn W>128")
                if q["srcH"] > 128:
                    key("gather dcn H>128")
                if q["srcW"] % 16:
                    key("gather dcn W%16")
                if q["srcH"] % 8:
                    key("gather dcn H%8")
                if (q["srcH"], q["srcW"]) == (128, 128):
                    key("gather dcn 128x128")
            if f == _lib.FAM_DCN_TMA and q["srcH"] != q["srcW"]:
                key("dcn_tma non-square")
        if (q["srcH"], q["srcW"]) == (26, 19):
            key("26x19 map")
        x3_ok = bool(q["x3"]) == (p == "tf32x3")
        if f == _lib.FAM_CONV_TMA and x3_ok:
            if q["kh"] == 3 and q["srcW"] + 2 == 242:
                key("conv_tma 3x3 W+2=242")
            if q["fuse_heads"] and (q["srcH"], q["srcW"]) == (128, 240):
                key("fused heads 128x240")
            if q["out_head"] >= 0 and q["kh"] == 1:
                key("unfused head 1x1 on conv_tma")
        if f == _lib.FAM_IGEMM_UMMA and q["n_children"] > 0 and q["kh"] == 3 and not q["fuse_heads"]:
            key("merged heads on gather")
        if f in (_lib.FAM_CONV_TMA, _lib.FAM_DCN_TMA) and x3_ok and _tiles(q) >= 4 * q["grid"]:
            key("%s >= 4 tiles per CTA" % FAM[f])
    for (g, p), fams in dcn_fams.items():
        if fams == {_lib.FAM_IGEMM_UMMA}:
            have.add((g, p, "every dcn on gather"))
    return have


def test_launch_coverage(geometry_records):
    """Each geometry reaches the paths it is here for; a schedule change that moves an op off one fails here instead
    of leaving the per-op assertions vacuous."""
    have = _paths(geometry_records)
    print("coverage: %s" % sorted(map(str, have & NEED)))
    assert not (NEED - have), "paths no configuration reaches: %s" % sorted(map(str, NEED - have))


def test_chained_op_references_are_the_network_at_832x608(cplib):
    """The op descriptors mean the network at an odd size (1/32 map 26 x 19, odd up-sampling): the fp64 per-op
    references chained through the schedule reproduce the fp64 oracle network, both computed on the device."""
    from oracle import net_ref
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sd = _exact_bn(synth.seeded_state_dict(m, seed=5, offset_std=0.3))
    H, W = 832, 608
    eng, _, _ = _engine("dla_34", False, H, W, 1, "fp32", sd=sd)
    g = torch.Generator(device="cuda").manual_seed(832)
    x = torch.randn((1, 3, H, W), generator=g, device="cuda", dtype=torch.float64)
    heads = chained_heads(eng, [x, None, None, None], 1)
    eng.close()
    with torch.no_grad():
        sd64 = {k: v.double().cuda() if v.dtype.is_floating_point else v for k, v in sd.items()}
        want = net_ref.forward(x, sd64, opt.heads, "dla_34")
    assert sorted(heads) == sorted(want)
    for h in want:
        assert heads[h].shape == want[h].shape == (1, opt.heads[h], H // 4, W // 4)
        e = float((heads[h] - want[h]).abs().max()) / max(1e-30, float(want[h].abs().max()))
        print("832x608 head %-18s chained-vs-oracle %.2e" % (h, e))
        assert e <= 1e-10, (h, e)
