"""The tf32x3 fused-heads 3x3 runs the per-head 1x1 in a warpgroup of its own, fed relu(conv + bias) through a ring in
shared memory while the consumers run the next tile's MMAs.  That must not change a bit.  For the plans no other test
puts through that launch:
  * the 11-head tracking plan (71 outputs across the heads);
  * a 2-model plan (the model-indexed instance), against each model's own plan;
  * a 64 x 64 input (16 x 16 heads), where every CTA gets one head's tiles or none, so the 1x1 warpgroup drains the
    CTA's last tile with nothing behind it;
every op against fp64 under LAYER_CEIL, and with a fixed K partition (CP_NO_SPLITK=1) frame 0 of the heads is the same
bits at batch 1 and batch 3.
"""
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib, synth
from centerpose_b200.engine import Engine
from tests import layer_ref
from tests.plan_steps import _ceiling, _engine, _fetch, _heads, _inputs, step_and_score
from tests.util import LAYER_CEIL, no_splitk

pytestmark = pytest.mark.gpu

# (label, tracking plan, H, W)
CASES = [("tracking 512", True, 512, 512), ("one unit per CTA 64", False, 64, 64)]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fused_heads_layers_vs_fp64(case):
    _, trk, H, W = case
    recs = step_and_score("dla_34", trk, H, W, 3, 3, "tf32x3")
    assert any(q["family"] == _lib.FAM_CONV_TMA and q["x3"] and q["fuse_heads"] for q in recs), "no fused-heads launch"
    bad = [(q["name"], q["r"], LAYER_CEIL[q["ceil"]]) for q in recs if not q["r"] <= LAYER_CEIL[q["ceil"]]]
    assert not bad, bad


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fused_heads_batch_invariant_bits(case):
    _, trk, H, W = case
    with no_splitk():
        eng, _, _ = _engine("dla_34", trk, H, W, 3, "tf32x3")
        if trk:
            assert len(eng.heads) == 11 and sum(eng.heads.values()) == 71, eng.heads
        n_ops = len(eng.op_descs())
        x, ext = _inputs(eng, 3)
        h3 = _heads(eng, 3)
        eng.run_ops(x, 0, n_ops, h3, *ext[1:])
        h1 = _heads(eng, 1)
        eng.run_ops(x[:1].contiguous(), 0, n_ops, h1, *[None if e is None else e[:1].contiguous() for e in ext[1:]])
        torch.cuda.synchronize()
        for n in h3:
            assert torch.isfinite(h1[n]).all(), n
            assert torch.equal(h1[n][0], h3[n][0]), n
        eng.close()


M = 2
H2, W2 = 256, 256


def _two_models(B):
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sds = [synth.seeded_state_dict(m, seed=s, offset_std=0.3) for s in (21, 22)]
    kw = dict(tracking_task_gru=False, precision="tf32x3")
    multi = Engine(m._arch(), m.heads, m.head_conv, B, H2, W2, 0, models=M, **kw)
    singles = [Engine(m._arch(), m.heads, m.head_conv, B, H2, W2, 0, **kw) for _ in range(M)]
    for i, sd in enumerate(sds):
        multi.load_state_dict(sd, model=i)
        singles[i].load_state_dict(sd)
    return multi, singles


def test_two_models_vs_fp64():
    multi, _ = _two_models(1)
    x, ext = _inputs(multi, 1)
    heads = {n: torch.full((M, 1, c, H2 // 4, W2 // 4), float("nan"), device="cuda") for n, c in multi.heads.items()}
    descs = [multi.op_descs(model=i) for i in range(M)]
    fused = False
    bad = []
    for k in range(len(descs[0])):
        wants = []
        with torch.no_grad():
            for i in range(M):
                rd = layer_ref.ActReader(multi.arena(), ext, [0], 1)
                wants.append((rd, layer_ref.op_ref(descs[i][k], rd, _fetch, descs[i])))
        info = multi.run_ops(x, k, k + 1, heads)[0]
        torch.cuda.synchronize()
        d = descs[0][k]
        if d["fused_away"]:
            continue
        fused |= info["family"] == _lib.FAM_CONV_TMA and d["x3"] and d["fuse_heads"]
        for i, (rd, want) in enumerate(wants):
            r = 0.0
            for (kind, tgt), ref, S in want:
                got = rd.get(tgt) if kind == "act" else heads[multi.head_names[tgt]][i].double()
                r = max(r, (0.0 if torch.equal(got, ref) else float("inf")) if d["family"] == _lib.FAM_MAXPOOL
                        else layer_ref.score(got, ref, S))
            if not r <= LAYER_CEIL[_ceiling(d, "tf32x3")]:
                bad.append((i, k, d["name"], r))
    assert fused, "no fused-heads launch"
    assert not bad, bad


def test_two_models_bits():
    """Each model's slice is its own plan's heads, bit for bit, and frame 0 is the same at batch 1 and batch 3."""
    with no_splitk():
        multi, singles = _two_models(3)
        x, _ = _inputs(multi, 3)
        got3 = {n: t.clone() for n, t in multi.forward(x).items()}
        got1 = {n: t.clone() for n, t in multi.forward(x[:1].contiguous()).items()}
        for i, eng in enumerate(singles):
            want = eng.forward(x)
            for n in want:
                assert torch.isfinite(got3[n][i]).all(), (i, n)
                assert torch.equal(got3[n][i], want[n]), (i, n)
                assert torch.equal(got1[n][i][0], got3[n][i][0]), (i, n)
