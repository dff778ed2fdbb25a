"""The crafted deformable sampling fields (tests/dcn_positions.py) on the CPU: their targets are exact in fp32, they
populate every sampling class at every shape tests/test_gpu_dcn_edges.py launches, the fp64 restatement is the oracle's
op, and the two mistakes a kernel could make at these positions (truncation instead of floor, border corners clamped
instead of zeroed) move the output far past the fp32 ceiling."""
import pytest
import torch

from oracle.net_ref import dcn_v2_forward_ref
from tests import dcn_positions as dp
from tests import layer_ref
from tests.util import LAYER_CEIL

TMA_SHAPES, GATHER_SHAPES, PLAN_MAPS = dp.TMA_SHAPES, dp.GATHER_SHAPES, dp.PLAN_MAPS
SHAPES = TMA_SHAPES + GATHER_SHAPES


def _case(B, C, H, W, Co, seed=5):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Co, C, 3, 3, generator=g, dtype=torch.float64) / (9 * C) ** 0.5
    b = torch.randn(Co, generator=g, dtype=torch.float64) * 0.1
    off = dp.crafted_offsets(B, H, W, seed).double()
    mask = dp.crafted_masks(B, H, W, seed).double()
    return x, off, mask, w, b


def test_shapes_reach_both_kernels():
    assert all(dp.dcn_tma_shape(H, W) for _, _, H, W, _ in TMA_SHAPES)
    assert not any(dp.dcn_tma_shape(H, W) for _, _, H, W, _ in GATHER_SHAPES)


@pytest.mark.parametrize("H,W", sorted({(s[2], s[3]) for s in SHAPES} | set(PLAN_MAPS)))
def test_targets_are_fp32_positions(H, W):
    """base + offset rounded to fp32 is the exact sum: the kernels sample where the field aims."""
    off = dp.crafted_offsets(2, H, W, 7).double()
    assert torch.equal(layer_ref.fp32_positions(off), off)
    assert float(off.abs().max()) > 30          # some samples land tens of pixels outside the image


@pytest.mark.parametrize("H,W", sorted({(s[2], s[3]) for s in SHAPES} | set(PLAN_MAPS)))
def test_every_class_populated(H, W):
    B = 2 if H * W < 4096 else 1
    n = dp.classify(dp.crafted_offsets(B, H, W, 7), H, W)
    empty = [k for k in dp.required_classes(H, W) if n[k] == 0]
    assert not empty, (H, W, n)
    if dp.dcn_tma_shape(H, W):
        assert n["slab"] + n["global"] + n["outside"] == n["samples"], n


def test_masks_hit_their_values():
    m = dp.crafted_masks(2, 8, 16, 3)
    for v in (0.0, 1.0, 0.5):
        assert int((m == v).sum()) > 0, v
    lg = dp.crafted_masks(2, 8, 16, 3, logits=True)
    for v in (-30.0, 0.0, 30.0):
        assert int((lg == v).sum()) > 0, v


@pytest.mark.parametrize("shape", SHAPES)
def test_restatement_is_the_oracle_and_mutants_fail(shape):
    x, off, mask, w, b = _case(*shape)
    ref = dcn_v2_forward_ref(x, off, mask, w, b)
    S = dcn_v2_forward_ref(x.abs(), off, mask, w.abs(), b.abs())
    mine = dp.sample_ref(x, off, mask, w, b)
    assert layer_ref.score(mine, ref, S) <= 1e-12
    for variant in ("trunc", "clamp"):
        r = layer_ref.score(dp.sample_ref(x, off, mask, w, b, variant), ref, S)
        print("%s %s: r %.3e" % (shape, variant, r))
        assert r > 10 * LAYER_CEIL["fp32"], (shape, variant, r)
