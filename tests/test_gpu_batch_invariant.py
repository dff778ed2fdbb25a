"""Batch-invariant plans (CP_PLAN_BATCH_INVARIANT) on the device, with split-K left on: a frame's heads are the same
bits at any batch, in any row, with one or several models, on either K path (split at small batches, fold at large
ones), and equal to a default plan's batch-1 heads on a 132-SM H100."""
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib, synth
from centerpose_b200.engine import Engine

pytestmark = pytest.mark.gpu

NETS = [("dla_34", False), ("dlav1_34", False), ("res_18", False), ("dla_34", True)]
SHAPES = [(512, 512), (96, 128)]
# (batch, first frame): frame f + r sits in row r of the batch
BATCHES = [(2, 30), (3, 4), (8, 24), (32, 0)]


def _model(arch, trk, wseed=11):
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    return m, synth.seeded_state_dict(m, seed=wseed, offset_std=0.3)


def _engine(m, sds, H, W, max_batch, prec, invariant=True):
    eng = Engine(m._arch(), m.heads, m.head_conv, max_batch, H, W, 0, tracking=m.tracking_inputs,
                 tracking_task_gru=m.use_convGRU and m.tracking_task, precision=prec, models=len(sds),
                 batch_invariant=invariant)
    for i, sd in enumerate(sds):
        eng.load_state_dict(sd, model=i)
    return eng


def _inputs(eng, n, seed=317):
    H, W = eng.height, eng.width
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(n, H, W, seed=seed))).cuda()
    if not eng.tracking:
        return [x, None, None, None]
    g = torch.Generator(device="cuda").manual_seed(seed)
    pre_img = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(n, H, W, seed=seed + 1))).cuda()
    return [x, pre_img, torch.rand((n, 1, H, W), device="cuda", generator=g),
            torch.rand((n, 8, H, W), device="cuda", generator=g)]


def _forward(eng, xs, a, b):
    s = [None if t is None else t[a:b].contiguous() for t in xs]
    out = eng.forward(s[0], pre_img=s[1], pre_hm=s[2], pre_hm_hp=s[3])
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


def _paths(eng):
    return [eng.op_ksegments(i) for i in range(eng.L.cp_plan_num_ops(eng.plan))]


def _assert_rows_equal(got, refs, first, what):
    for n in got:
        for r in range(got[n].shape[-4]):
            assert torch.equal(got[n][..., r, :, :, :], refs[first + r][n][..., 0, :, :, :]), \
                "%s: head %s of frame %d differs from its batch-1 bits" % (what, n, first + r)


@pytest.mark.parametrize("prec", ["tf32x3", "tf32"])
@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("arch,trk", NETS)
def test_heads_same_bits_at_every_batch(arch, trk, H, W, prec):
    m, sd = _model(arch, trk)
    eng = _engine(m, [sd], H, W, 32, prec)
    xs = _inputs(eng, 32)
    refs = [_forward(eng, xs, f, f + 1) for f in range(32)]
    one = _paths(eng)
    split = [p for p in one if p["segments"] > 1]
    for p in one:
        if p["segments"] > 1:
            assert p["last_segments"] == p["segments"] and p["last_path"] == _lib.KPATH_SPLIT, p
    for B, f in BATCHES:
        got = _forward(eng, xs, f, f + B)
        _assert_rows_equal(got, refs, f, "%s%s %dx%d %s batch %d" % (arch, " tracking" if trk else "", H, W, prec, B))
        for p in _paths(eng):
            if p["segments"] > 1:
                assert p["last_segments"] == p["segments"] and p["last_path"] in (_lib.KPATH_SPLIT, _lib.KPATH_FOLD), p
    if H == 512 and split:
        # batch 32 at 512 x 512 overflows the split-K workspace in at least one launch: the fold ran and matched
        assert any(p["last_path"] == _lib.KPATH_FOLD for p in _paths(eng))
    eng.close()


@pytest.mark.parametrize("prec", ["tf32x3", "tf32"])
@pytest.mark.parametrize("H,W", SHAPES)
def test_three_models_match_one(H, W, prec):
    m, sd = _model("dla_34", False)
    _, sd1 = _model("dla_34", False, wseed=12)
    _, sd2 = _model("dla_34", False, wseed=13)
    one = _engine(m, [sd], H, W, 8, prec)
    three = _engine(m, [sd, sd1, sd2], H, W, 8, prec)
    xs = _inputs(one, 8)
    refs = [_forward(one, xs, f, f + 1) for f in range(8)]
    for B, f in ((1, 3), (3, 2), (8, 0)):
        got = _forward(three, xs, f, f + B)
        _assert_rows_equal({k: v[0] for k, v in got.items()}, refs, f, "model 0 of 3, batch %d" % B)
    if H == 512:
        # 3 models x 8 frames overflow the split-K workspace: the MULTI fold instances ran (dcn_tma in tf32 and tf32x3,
        # conv_tma in tf32x3)
        paths = _paths(three)
        assert any(p["last_path"] == _lib.KPATH_FOLD for p in paths)
        fams = {d["family"] for d, p in zip(three.op_descs(), paths) if p["last_path"] == _lib.KPATH_FOLD}
        assert _lib.FAM_DCN_TMA in fams and (prec == "tf32" or _lib.FAM_CONV_TMA in fams), fams
    one.close()
    three.close()


@pytest.mark.parametrize("arch,trk", NETS)
def test_batch32_is_the_default_plans_batch1_bits(arch, trk):
    """On a 132-SM H100 the fixed segments are the ones a default plan picks at batch 1: invariant heads at batch 32
    equal default heads at batch 1, frame by frame."""
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("a default plan's batch-1 split equals the fixed one on a 132-SM device only")
    m, sd = _model(arch, trk)
    inv = _engine(m, [sd], 512, 512, 32, "tf32x3")
    dflt = _engine(m, [sd], 512, 512, 1, "tf32x3", invariant=False)
    xs = _inputs(inv, 32)
    got = _forward(inv, xs, 0, 32)
    assert any(p["last_path"] == _lib.KPATH_FOLD for p in _paths(inv))
    refs = [_forward(dflt, xs, f, f + 1) for f in range(32)]
    _assert_rows_equal(got, refs, 0, "%s%s invariant batch 32 against default batch 1" % (arch, " tracking" if trk else ""))
    inv.close()
    dflt.close()


def test_network_module_and_default_bits():
    """The network's own forward (the plan every single-category product path builds through model.engine) carries the
    flag; on a 132-SM device its bits at batch 8 are a default plan's batch-1 bits."""
    opt = cpb.default_opt("dla_34", batch_invariant=True)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    assert m.batch_invariant
    sd = synth.seeded_state_dict(m, seed=11, offset_std=0.3)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(8, 512, 512, seed=5))).cuda()
    with torch.no_grad():
        refs = [{k: v.clone() for k, v in m(x[i:i + 1])[-1].items()} for i in range(8)]
        got = {k: v.clone() for k, v in m(x)[-1].items()}
    _assert_rows_equal(got, refs, 0, "model forward, batch 8")
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the batch-1 bits of a default plan equal the invariant ones on a 132-SM device only")
    dflt = _engine(m, [sd], 512, 512, 1, "tf32x3", invariant=False)
    for i in range(8):
        want = _forward(dflt, [x, None, None, None], i, i + 1)
        for n in want:
            assert torch.equal(got[n][i:i + 1], want[n]), "frame %d head %s: not the default plan's batch-1 bits" % (i, n)
    dflt.close()


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_fp32_bf16_accept_the_flag_unchanged(prec):
    m, sd = _model("dla_34", False)
    inv = _engine(m, [sd], 96, 128, 3, prec)
    dflt = _engine(m, [sd], 96, 128, 3, prec, invariant=False)
    xs = _inputs(inv, 3)
    a, b = _forward(inv, xs, 0, 3), _forward(dflt, xs, 0, 3)
    for n in a:
        assert torch.equal(a[n], b[n]), n
    assert all(p["segments"] == 1 for p in _paths(inv))
    inv.close()
    dflt.close()
