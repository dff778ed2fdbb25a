"""The tf32x3 TMA convolution's schedule: an accumulation group's K blocks stay in flight on one accumulator, and the
accumulator is dead through the epilogue.  Neither may change a bit, so:
  * every op of the plan, among them the fused-heads 3x3 and the unfused tf32x3 3x3 convs, against fp64 under
    LAYER_CEIL at a 96 x 160 head map (partial last tile, several tiles per CTA, both N tiles of every head);
  * with a fixed K partition (CP_NO_SPLITK=1) the heads of frame 0 are the same bits at batch 1 and batch 3.
"""
import pytest
import torch

from centerpose_b200 import _lib
from tests.plan_steps import _engine, _heads, _inputs, step_and_score
from tests.util import LAYER_CEIL, no_splitk

pytestmark = pytest.mark.gpu

H, W = 384, 640      # heads at 96 x 160: 96 * 162 positions = 121.5 tiles of 128


def test_conv_tma_x3_layers_vs_fp64():
    recs = step_and_score("dla_34", False, H, W, 3, 3, "tf32x3")
    tma = [q for q in recs if q["family"] == _lib.FAM_CONV_TMA and q["x3"] and q["kh"] == 3]
    assert any(q["fuse_heads"] for q in tma), "no fused-heads conv_tma launch"
    assert any(not q["fuse_heads"] for q in tma), "no unfused tf32x3 conv_tma launch"
    bad = [(q["name"], q["r"], LAYER_CEIL[q["ceil"]]) for q in recs if not q["r"] <= LAYER_CEIL[q["ceil"]]]
    assert not bad, bad


def test_conv_tma_x3_batch_invariant_bits():
    with no_splitk():
        eng, _, _ = _engine("dla_34", False, H, W, 3, "tf32x3")
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
