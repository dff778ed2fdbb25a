"""Network parity on the GPU: CUDA plan (through the C ABI) vs the reference's
golden head tensors and vs the CPU oracle on the same seeded inputs."""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import synth
from tests.util import TOL_HEAD_REL, dcn_case_inputs, golden, net_case_inputs

pytestmark = pytest.mark.gpu

CASES = ["net_dla34_b2_96x128", "net_dlav1_b1_64x64", "net_dla34track_b1_64x96"]


def _model(arch, trk, wseed, offset_std=0.3, precision="fp32"):
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.precision = precision
    sd = synth.seeded_state_dict(m, seed=wseed, offset_std=offset_std)
    m.load_state_dict(sd)
    return m.cuda().eval(), opt, sd


def _check(out, want, rel=TOL_HEAD_REL, truth=None, truth_factor=4.0):
    """Stage-B bar (tests/util.py): max|gpu - ref_fp32| <= TOL_HEAD_REL * max|head|.  When the fp64 evaluation
    of the same graph (`truth`) is given, additionally: the CUDA heads may not be further from the fp64 truth
    than `truth_factor` x the reference's own fp32 CPU path is (+3e-5) -- i.e. the kernel is fp32-equivalent."""
    worst = 0.0
    for h, w in want.items():
        got = out[h].float().cpu().numpy()
        assert got.shape == w.shape, (h, got.shape, w.shape)
        assert np.isfinite(got).all(), h
        mag = max(1e-6, np.abs(w).max())
        e = np.abs(got - w).max() / mag
        worst = max(worst, e)
        assert e <= rel, "head %s: max-abs error %.3e of max|ref| (tolerance %.1e)" % (h, e, rel)
        if truth is not None:
            t = truth[h]
            e_ref = np.abs(w.astype(np.float64) - t).max() / mag
            e_gpu = np.abs(got.astype(np.float64) - t).max() / mag
            print("head %-18s gpu-vs-ref %.2e  gpu-vs-fp64 %.2e  ref-fp32-vs-fp64 %.2e" % (h, e, e_gpu, e_ref))
            assert e_gpu <= truth_factor * e_ref + 3e-5, \
                "head %s: gpu-vs-fp64 %.3e, reference-fp32-vs-fp64 %.3e" % (h, e_gpu, e_ref)
    return worst


def _truth(x, sd, heads, arch, extra=None, tracking_task=False):
    """fp64 CPU evaluation of the oracle graph."""
    from oracle import net_ref
    sd64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in sd.items()}
    kw = {k: torch.from_numpy(v).double() for k, v in (extra or {}).items()}
    out = net_ref.forward(torch.from_numpy(x).double(), sd64, heads, arch, tracking_task=tracking_task, **kw)
    return {h: v.numpy() for h, v in out.items()}


@pytest.mark.parametrize("name", CASES)
def test_forward_matches_reference_golden(name, cplib):
    g = golden(name)
    arch, trk = str(g["arch"]), bool(int(g["tracking"]))
    m, opt, sd = _model(arch, trk, int(g["wseed"]), float(g["offset_std"]))
    x, extra = net_case_inputs(g)
    kw = {k: torch.from_numpy(v).cuda() for k, v in extra.items()}
    out = m(torch.from_numpy(x).cuda(), **kw)[-1]
    assert list(out) == list(opt.heads)
    _check(out, {h: g["head_" + h] for h in opt.heads}, truth=_truth(x, sd, opt.heads, arch, extra))


def test_forward_512_matches_oracle(cplib):
    """BASELINE config 2 shape (batch 1, 512x512, dla_34) against the CPU oracle.  (Weights with DCN offset
    std 0.3: with 1.5 the graph is numerically chaotic on noise frames -- the reference's own fp32 CPU heads
    are then 16-23 % away from the fp64 evaluation, see DESIGN.md section 5.)"""
    from oracle import net_ref
    m, opt, sd = _model("dla_34", False, 12)
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(1, 512, 512, seed=317)))
    want = net_ref.forward(x, sd, opt.heads, "dla_34")
    out = m(x.cuda())[-1]
    # at 512 x 512 the fp32 floor is higher (the reference's fp32 heads are 1.2e-4 .. 2.6e-4 from the fp64 truth)
    _check(out, {h: v.numpy() for h, v in want.items()}, rel=1e-3, truth=_truth(x.numpy(), sd, opt.heads, "dla_34"))


def test_batch_invariance_and_replay(cplib):
    """Frames are independent (SURVEY.md 8e): a frame's heads do not depend on its batch neighbours
    or on the plan's max_batch, and the plan is re-entrant."""
    m, opt, _ = _model("dla_34", False, 5)
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(3, 128, 160, seed=1))).cuda()
    full = m(x)[-1]
    again = m(x)[-1]
    single = m(x[1:2].contiguous())[-1]
    for h in full:
        assert torch.equal(full[h], again[h])
        assert torch.equal(full[h][1:2], single[h]), h


@pytest.mark.parametrize("arch,trk", [("dlav1_34", False), ("dla_34", True)])
def test_batch_invariance_and_replay_gn_and_tracking(arch, trk, cplib):
    """The same for the dlav1 plan (convGRU, GroupNorm heads: the GroupNorm statistics are summed in a fixed order)
    and for the tracking plan (pre_img / pre_hm / pre_hm_hp stems): bit-identical on replay and independent of the
    batch neighbours."""
    m, opt, _ = _model(arch, trk, 5)
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(3, 128, 160, seed=1))).cuda()
    kw = {}
    if trk:
        g = torch.Generator(device="cuda").manual_seed(2)
        kw = dict(pre_img=torch.randn(3, 3, 128, 160, device="cuda", generator=g),
                  pre_hm=torch.rand(3, 1, 128, 160, device="cuda", generator=g),
                  pre_hm_hp=torch.rand(3, 8, 128, 160, device="cuda", generator=g))
    full = m(x, **kw)[-1]
    again = m(x, **kw)[-1]
    single = m(x[1:2].contiguous(), **{k: v[1:2].contiguous() for k, v in kw.items()})[-1]
    for h in full:
        assert torch.equal(full[h], again[h]), h
        assert torch.equal(full[h][1:2], single[h]), h


def test_weight_reload_is_picked_up(cplib):
    m, opt, sd = _model("dla_34", False, 6)
    x = torch.randn(1, 3, 64, 64, device="cuda")
    a = m(x)[-1]["hm"].clone()
    with torch.no_grad():
        m.hm[2].bias.add_(1.0)
    b = m(x)[-1]["hm"]
    assert torch.allclose(b, a + 1.0, atol=1e-5)


def test_missing_and_misshaped_weights_are_reported(cplib):
    from centerpose_b200.engine import Engine
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    eng = Engine("dla_34", opt.heads, 256, 1, 64, 64, 0)
    sd = {k: v for k, v in m.state_dict().items() if k != "ida_up.node_1.conv.weight"}
    with pytest.raises(RuntimeError, match="ida_up.node_1.conv.weight"):
        eng.load_state_dict(sd)
    with pytest.raises(RuntimeError, match="load_weights"):
        eng.forward(torch.zeros(1, 3, 64, 64, device="cuda"))
    sd = dict(m.state_dict())
    sd["hm.2.weight"] = torch.zeros(2, 256, 1, 1)
    with pytest.raises(RuntimeError, match="hm.2.weight"):
        eng.load_state_dict(sd)
    eng.close()


@pytest.mark.parametrize("name", ["dcn_small", "dcn_edge_big_offsets"])
def test_dcn_ext_matches_reference_cpp(name, cplib):
    """cp_dcn_v2_forward (the `_ext.dcn_v2_forward` replacement) vs the reference's own C++ CPU op."""
    g = golden(name)
    x, off, mask, w, bias = [torch.from_numpy(a).cuda() for a in dcn_case_inputs(g)]
    out = cpb.dcn_v2_forward(x, w, bias, off, mask, 3, 3, 1, 1, 1, 1, 1, 1, 1).cpu().numpy()
    assert np.abs(out - g["out"]).max() <= 2e-5


def test_dcn_zero_offset_identity(cplib):
    """DCNv2/testcuda.py:32-67 check_zero_offset."""
    x = torch.randn(2, 64, 16, 16, device="cuda")
    w = torch.zeros(64, 64, 3, 3, device="cuda")
    for c in range(64):
        w[c, c, 1, 1] = 1.0
    out = cpb.dcn_v2_forward(x, w, torch.zeros(64, device="cuda"), torch.zeros(2, 18, 16, 16, device="cuda"),
                             torch.full((2, 9, 16, 16), 0.5, device="cuda"))
    assert (2 * out - x).abs().max().item() <= 1e-6


def test_dcn_ext_matches_oracle_odd_channels(cplib):
    """Channel counts that are not multiples of 16 (DCNv2/testcuda.py uses C=2) go through zero padding."""
    from oracle import net_ref
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 6, 10, 7, generator=g)
    off = torch.randn(1, 18, 10, 7, generator=g) * 3
    mask = torch.rand(1, 9, 10, 7, generator=g)
    w = torch.randn(5, 6, 3, 3, generator=g) * 0.2
    b = torch.randn(5, generator=g)
    want = net_ref.dcn_v2_forward_ref(x, off, mask, w, b)
    got = cpb.dcn_v2_forward(x.cuda(), w.cuda(), b.cuda(), off.cuda(), mask.cuda()).cpu()
    assert (got - want).abs().max().item() <= 2e-5
