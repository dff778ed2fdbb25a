"""Deformable convolution at its sampling edges: every DCN kernel, stand-alone and in the plan, against fp64 on the
crafted fields of tests/dcn_positions.py (integers, the bounds -1 and H, just inside them, half-integers at the border,
the dcn_tma slab thresholds, far-out samples; masks 0, 1, 0.5 or logits -30, 0, +30).

  * stand-alone launches (cp_dcn_v2_forward_ex) in fp32, tf32x3, tf32 and bf16 at shapes that reach each kernel at its
    limits: dcn_tma with one patch, with image coordinates up to 127 in both 7-bit record fields, H = 128 with one patch
    column, a partial N tile, 16 slabs on two tiles; the gather kernel at H > 128, W > 128 and odd H, C and Co padded.
    fp32 runs every shape on igemm_fp32 and bf16 on the gather kernel.  Stand-alone launches never split K (no
    workspace); the plans below do.  Outputs are pre-filled with NaN, so an unwritten element scores inf;
  * the zero-offset identity (every sample on an integer, the border taps exactly on -1 and H) in every precision;
  * every DCN launch of dla_34 plans, teacher-forced (tests/plan_steps.py): before each DCN op its offset / mask input
    is overwritten with a crafted field (mask as logits) for every frame and its output with NaN, then the op runs and
    is scored against layer_ref.op_ref.  The coverage assertion lists every DCN path these plans must reach, from the
    launch records and the field's classes (tests/dcn_positions.classify), so the per-op assertion cannot pass vacuously.

Scores are r = max |got - ref| / S (tests/layer_ref.py) under LAYER_CEIL.  Run with -s for the tables.
"""
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib, synth
from centerpose_b200.engine import Engine, _stream
from oracle.net_ref import dcn_v2_forward_ref
from tests import dcn_positions as dp
from tests import layer_ref
from tests.plan_steps import FAM, _ceiling, _env, _fetch, _inputs, over_ceiling, print_records, print_worst
from tests.util import LAYER_CEIL

pytestmark = pytest.mark.gpu

CEIL = {"fp32": "fp32", "tf32x3": "fp32", "tf32": "tf32", "bf16": "bf16"}


def _dcn_into_nan(x, w, b, off, mask, prec):
    """cp_dcn_v2_forward_ex into an output pre-filled with NaN."""
    B, C, H, W = x.shape
    Co = w.shape[0]
    out = torch.full((B, Co, H, W), float("nan"), device="cuda")
    ts = [t.contiguous() for t in (x, w, b, off, mask)]
    rc = _lib.load().cp_dcn_v2_forward_ex(*[ctypes.c_void_p(t.data_ptr()) for t in ts + [out]], B, C, H, W, Co,
                                          _lib.PRECISIONS[prec], _stream())
    _lib.check(rc, "cp_dcn_v2_forward_ex")
    torch.cuda.synchronize()
    return out


def _score_standalone(x, w, b, off, mask, prec):
    got = _dcn_into_nan(x, w, b, off, mask, prec)
    offp = layer_ref.fp32_positions(off.double())
    ref = dcn_v2_forward_ref(x.double(), offp, mask.double(), w.double(), b.double())
    S = dcn_v2_forward_ref(x.double().abs(), offp, mask.double(), w.double().abs(), b.double().abs())
    return layer_ref.score(got, ref, S)


@pytest.mark.parametrize("prec", ["fp32", "tf32x3", "tf32", "bf16"])
def test_standalone_crafted_fields(prec, cplib):
    g = torch.Generator().manual_seed(23)
    bad, worst = [], 0.0
    for i, (B, C, H, W, Co) in enumerate(dp.TMA_SHAPES + dp.GATHER_SHAPES):
        x = torch.randn(B, C, H, W, generator=g).cuda()
        w = (torch.randn(Co, C, 3, 3, generator=g) / np.sqrt(9 * C)).cuda()
        b = (torch.randn(Co, generator=g) * 0.1).cuda()
        off = dp.crafted_offsets(B, H, W, 100 + i).cuda()
        mask = dp.crafted_masks(B, H, W, 200 + i).cuda()
        r = _score_standalone(x, w, b, off, mask, prec)
        kernel = ("igemm_fp32" if prec == "fp32" else "igemm_umma bf16" if prec == "bf16"
                  else "dcn_tma" if dp.dcn_tma_shape(H, W) else "igemm_umma x3")
        print("stand-alone %-6s %-22s %-16s r %.3e (ceiling %.1e)" % (prec, (B, C, H, W, Co), kernel, r,
                                                                       LAYER_CEIL[CEIL[prec]]))
        worst = max(worst, r)
        if not r <= LAYER_CEIL[CEIL[prec]]:
            bad.append(((B, C, H, W, Co), r))
    print("stand-alone %s: worst r %.3e, ceiling %s %.1e" % (prec, worst, CEIL[prec], LAYER_CEIL[CEIL[prec]]))
    assert not bad, (prec, bad)


@pytest.mark.parametrize("prec", ["fp32", "tf32x3", "tf32", "bf16"])
def test_zero_offset_identity_every_precision(prec, cplib):
    """DCNv2/testcuda.py's check_zero_offset with mask 1: the centre tap of an identity weight returns the input."""
    x = torch.randn(2, 64, 16, 16, device="cuda")
    w = torch.zeros(64, 64, 3, 3, device="cuda")
    for c in range(64):
        w[c, c, 1, 1] = 1.0
    off = torch.zeros(2, 18, 16, 16, device="cuda")
    mask = torch.ones(2, 9, 16, 16, device="cuda")
    got = _dcn_into_nan(x, w, torch.zeros(64, device="cuda"), off, mask, prec)
    r = layer_ref.score(got, x.double(), x.double().abs())
    print("zero-offset identity %s: r %.3e" % (prec, r))
    assert r <= LAYER_CEIL[CEIL[prec]], (prec, r)


# (label, precision, H, W, batch, environment at plan creation, batch_invariant, models)
PLANS = [
    ("256 b2", "tf32x3", 256, 256, 2, None, False, 1),
    ("256 b2", "tf32", 256, 256, 2, None, False, 1),
    ("256 b2 no dcn_tma", "tf32x3", 256, 256, 2, {"CP_NO_DCN_TMA": "1"}, False, 1),
    ("256 b2 no dcn_tma", "bf16", 256, 256, 2, {"CP_NO_DCN_TMA": "1"}, False, 1),
    ("256 b2", "fp32", 256, 256, 2, None, False, 1),
    # batch 8 overflows the split-K workspace at the 16 x 16 maps: their fixed K segments are folded in one CTA
    ("256 b8 invariant", "tf32x3", 256, 256, 8, None, True, 1),
    ("256 b2 models=2", "tf32x3", 256, 256, 2, None, False, 2),
    ("512 b1", "tf32x3", 512, 512, 1, None, False, 1),
]


def _step_crafted(label, prec, H, W, batch, env, invariant, models):
    """Step a dla_34 plan op by op; each DCN op runs on a crafted field and is scored (one record per DCN op)."""
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    with _env(env):
        eng = Engine(m._arch(), m.heads, m.head_conv, batch, H, W, 0, precision=prec, models=models,
                     batch_invariant=invariant)
    for i in range(models):
        eng.load_state_dict(synth.seeded_state_dict(m, seed=11 + i, offset_std=0.3), model=i)
    descs = [eng.op_descs(model=i) for i in range(models)]
    x, ext = _inputs(eng, batch)
    heads = {n: torch.full(eng._head_shape(batch, c), float("nan"), device="cuda") for n, c in eng.heads.items()}
    arena = eng.arena()
    every = layer_ref.ActReader(arena, ext, range(batch), batch)
    scored = layer_ref.ActReader(arena, ext, sorted({0, batch - 1}), batch)
    config = "%s %s" % (label, prec)
    recs = []
    for k, d in enumerate(descs[0]):
        dcn = d["kind"] == 2 and not d["fused_away"]
        if dcn:
            h, w = d["om"]["H"], d["om"]["W"]
            wants, counts = [], dict.fromkeys(dp.CLASS_KEYS, 0)
            for i in range(models):
                di = descs[i][k]
                seed = 1000 * k + 10 * i + batch
                off = dp.crafted_offsets(batch, h, w, seed)
                om = torch.cat([off, dp.crafted_masks(batch, h, w, seed + 1, logits=True)], 1).cuda()
                every.put(di["om"], om)
                o = di["out"]
                every.put(o, torch.full((batch, o["C"], o["H"], o["W"]), float("nan"), device="cuda"))
                with torch.no_grad():
                    wants.append(layer_ref.op_ref(di, scored, _fetch, descs[i]))
                for key, v in dp.classify(off, h, w).items():
                    counts[key] += v
        li = eng.run_ops(x, k, k + 1, heads, *ext[1:])[0]
        torch.cuda.synchronize()
        if not dcn:
            continue
        assert li["family"] == d["family"], (d["name"], li, d["family"])
        r = max(layer_ref.score(scored.get(tgt), ref, S) for want in wants for (_, tgt), ref, S in want)
        recs.append(dict(config=config, prec=prec, index=k, name=d["name"], family=d["family"], x3=d["x3"], BN=li["BN"],
                         ksplit=li["ksplit"], path=eng.op_ksegments(k)["last_path"], r=r, ceil=_ceiling(d, prec),
                         H=h, W=w, models=models, counts=counts))
    eng.close()
    return recs


@pytest.fixture(scope="module")
def dcn_records(cplib):
    recs = []
    for plan in PLANS:
        recs += _step_crafted(*plan)
    print_records(recs)
    for q in recs:
        c = q["counts"]
        print("%-28s %-40s %4dx%-4d outside %6d slab %6d global %6d global127 %5d" % (
            q["config"], q["name"][:40], q["H"], q["W"], c["outside"], c["slab"], c["global"], c["global127"]))
    return recs


def test_every_dcn_op_under_its_ceiling(dcn_records):
    print_worst(dcn_records, "plan DCN ops: ")
    bad = over_ceiling(dcn_records)
    assert not bad, "\n".join(bad)


def test_dcn_path_coverage(dcn_records):
    have = set()
    for q in dcn_records:
        f, c = q["family"], q["counts"]
        if f == _lib.FAM_DCN_TMA:
            have.add(("dcn_tma", "x3" if q["x3"] else "tf32"))
            if q["path"] == _lib.KPATH_SPLIT and q["ksplit"] > 1:
                have.add("dcn_tma split-K")
            if q["path"] == _lib.KPATH_FOLD:
                have.add("dcn_tma fold")
            if q["models"] > 1:
                have.add("dcn_tma models=2")
            if c["slab"] > 0 and c["global"] > 0:
                have.add("dcn_tma in-slab and global samples")
            if c["global127"] > 0:
                have.add("dcn_tma row / column 127")
        elif f == _lib.FAM_IGEMM_UMMA:
            have.add(("gather", "bf16" if q["prec"] == "bf16" else "x3" if q["x3"] else "tf32"))
        else:
            have.add(FAM[f])
    need = {("dcn_tma", "x3"), ("dcn_tma", "tf32"), "dcn_tma split-K", "dcn_tma fold", "dcn_tma models=2",
            "dcn_tma in-slab and global samples", "dcn_tma row / column 127", ("gather", "x3"), ("gather", "bf16"),
            "igemm_fp32"}
    print("DCN coverage: %s" % sorted(map(str, have)))
    assert not (need - have), "DCN paths no plan reaches: %s" % sorted(map(str, need - have))
    # the default tf32x3 plan itself runs its 8 x 8 map (width not a multiple of 16) on the gather kernel
    assert any(q["config"] == "256 b2 tf32x3" and q["family"] == _lib.FAM_IGEMM_UMMA for q in dcn_records)
