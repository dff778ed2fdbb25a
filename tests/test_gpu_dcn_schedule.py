"""The TMA-staged deformable convolution's schedule (dcn_tma.cu): each consumer warp releases an A stage once its
fragments are in registers, the x3 instances with BN <= 64 issue an accumulation group's two K blocks under one wait,
and the A ring is 4 stages deep where 3 weight stages still fit beside it (2 for x3 at BN = 128).  None of it may move a
bit or a sample, so:
  * stand-alone launches of every N tile (16 / 32 / 64 / 128) in tf32x3 and tf32, scored against the fp64 restatement
    of dcn_v2_im2col_cuda.cu under LAYER_CEIL: split-K (few tiles), an odd K-block count per segment (a group of one K
    block at its end), several tiles per CTA (more tiles than SMs), and offsets large enough to send most samples
    through the global-memory path (the standard deviation of tests/golden/dcn_edge_big_offsets.npz and twice it;
    that golden's own 6 x 5 map is not a dcn_tma shape).  A single A stage is never chosen at these tile sizes;
  * every DCN op of a batch-invariant plan against fp64 at batches 2 and 4 (fixed K segments, split or folded);
  * with a fixed K partition (CP_NO_SPLITK=1) the heads of frame 0 are the same bits at batch 1 and batch 3.
"""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.engine import Engine
from centerpose_b200 import synth
from oracle.net_ref import dcn_v2_forward_ref
from tests import layer_ref
from tests.plan_steps import _engine, _heads, _inputs
from tests.util import LAYER_CEIL, golden, no_splitk

pytestmark = pytest.mark.gpu

BIG_OFF = float(golden("dcn_edge_big_offsets")["off_std"])

# (B, Cin, H, W, Cout): N tile 16 / 32 / 64 / 128 (Cout 256: two N tiles), split-K at 1-4 tiles, 3 slabs (27 K blocks:
# the last accumulation group of a segment is one K block), 256 and 512 tiles > 132 CTAs
SHAPES = [(1, 64, 16, 16, 16), (2, 48, 16, 32, 32), (1, 256, 16, 16, 64), (1, 128, 16, 32, 256),
          (4, 48, 64, 128, 64), (2, 64, 128, 128, 32), (3, 64, 32, 32, 128)]


@pytest.mark.parametrize("prec", ["tf32x3", "tf32"])
@pytest.mark.parametrize("off_std", [0.5, BIG_OFF, 2 * BIG_OFF])
def test_dcn_tma_launches_vs_fp64(prec, off_std):
    g = torch.Generator().manual_seed(41)
    ceil = LAYER_CEIL["fp32" if prec == "tf32x3" else "tf32"]
    bad = []
    for (B, C, H, W, Co) in SHAPES:
        x = torch.randn(B, C, H, W, generator=g)
        off = torch.randn(B, 18, H, W, generator=g) * off_std
        mask = torch.rand(B, 9, H, W, generator=g)
        w = torch.randn(Co, C, 3, 3, generator=g) / np.sqrt(C * 9)
        b = torch.randn(Co, generator=g) * 0.1
        got = cpb.dcn_v2_forward(x.cuda(), w.cuda(), b.cuda(), off.cuda(), mask.cuda(), precision=prec).cpu()
        offp = layer_ref.fp32_positions(off.double())
        ref = dcn_v2_forward_ref(x.double(), offp, mask.double(), w.double(), b.double())
        S = dcn_v2_forward_ref(x.double().abs(), offp, mask.double(), w.double().abs(), b.double().abs())
        r = layer_ref.score(got, ref, S)
        print("dcn_tma %s %s off_std %.1f: r %.3e" % ((B, C, H, W, Co), prec, off_std, r))
        if not r <= ceil:
            bad.append(((B, C, H, W, Co), r))
    assert not bad, (prec, off_std, ceil, bad)


@pytest.mark.parametrize("batch", [2, 4])
def test_dcn_batch_invariant_plan_vs_fp64(batch):
    """Batch-invariant plan at 256 x 256 (DCN maps 64 x 64 down to 16 x 16): its fixed K segments run split, or folded in
    one CTA per tile where the partial sums do not fit the workspace; every DCN op is scored."""
    from tests.plan_steps import _fetch
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sd = synth.seeded_state_dict(m, seed=11, offset_std=0.3)
    eng = Engine(m._arch(), m.heads, m.head_conv, batch, 256, 256, 0, precision="tf32x3", batch_invariant=True)
    eng.load_state_dict(sd)
    descs = eng.op_descs()
    x, ext = _inputs(eng, batch)
    heads = _heads(eng, batch)
    rd = layer_ref.ActReader(eng.arena(), ext, sorted({0, batch - 1}), batch)
    paths, bad = set(), []
    for i, d in enumerate(descs):
        with torch.no_grad():
            want = layer_ref.op_ref(d, rd, _fetch, descs) if d["family"] == _lib.FAM_DCN_TMA else None
        li = eng.run_ops(x, i, i + 1, heads, *ext[1:])[0]
        torch.cuda.synchronize()
        if want is None:
            continue
        paths.add(eng.op_ksegments(i)["last_path"])
        r = max(layer_ref.score(rd.get(tgt), ref, S) for (kind, tgt), ref, S in want)
        if not r <= LAYER_CEIL["fp32"]:
            bad.append((d["name"], li["BN"], li["ksplit"], r))
    eng.close()
    print("batch %d: K paths of the DCN launches %s" % (batch, sorted(paths)))
    assert paths & {_lib.KPATH_SPLIT, _lib.KPATH_FOLD}, paths
    assert not bad, bad


def test_dcn_frame_bits_batch_1_vs_3():
    with no_splitk():
        eng, _, _ = _engine("dla_34", False, 256, 256, 3, "tf32x3")
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
