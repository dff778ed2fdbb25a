"""wgmma tensor-core kernels (igemm_umma.cu, conv_tma.cu, dcn_tma.cu) against a plain PyTorch fp32 reference of the same op and
against the fp32 CUDA-core kernel: layer level (cp_conv2d, cp_dcn_v2_forward_ex) and whole network
(precision = tf32x3 -- fp32-equivalent -- and bf16 -- fast mode, looser stated tolerance)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import centerpose_b200 as cpb
from centerpose_b200 import synth
from tests.util import TOL_HEAD_REL, golden, net_case_inputs

pytestmark = pytest.mark.gpu

TOL = {"fp32": 2e-5, "tf32x3": 5e-5, "bf16": 1.5e-2, "tf32": 4e-3}     # max-abs error / max|ref| of one layer


def _conv_case(B, H, W, Cin, Cout, k, stride, pad, relu, res, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / np.sqrt(Cin * k * k)
    b = torch.randn(Cout, generator=g) * 0.1
    want = F.conv2d(x.double(), w.double(), b.double(), stride, pad)
    r = None
    if res:
        r = torch.randn(want.shape, generator=g)
        want = want + r.double()
    if relu:
        want = F.relu(want)
    return x, w, b, r, want.float()


CONV_SHAPES = [
    # B, H, W, Cin, Cout, k, stride, pad, relu, residual
    (1, 8, 16, 64, 64, 1, 1, 0, False, False),        # exactly one 128 x 64 tile, one K block (bf16)
    (2, 16, 16, 64, 64, 3, 1, 1, True, True),         # BasicBlock conv2 shape
    (1, 20, 24, 16, 32, 3, 2, 1, True, False),        # level1: Cin 16, stride 2, K blocks straddle taps
    (1, 12, 20, 128, 256, 1, 1, 0, False, False),     # BN = 256
    (1, 9, 7, 64, 16, 1, 1, 0, False, False),         # N = 16, M = 63 (< one tile)
    (3, 16, 16, 64, 512, 3, 1, 1, True, False),       # 2 N tiles of 256, merged-heads-like
    (1, 8, 8, 512, 256, 3, 1, 1, True, False),        # long K (72 / 144 K blocks)
    (2, 24, 40, 16, 16, 3, 1, 1, True, False),        # level0: 16 -> 16 (64-byte rows / SWIZZLE_64B on the TMA path)
    (1, 20, 150, 16, 16, 3, 1, 1, False, False),      # level0 over several 64 x 16 tiles of the direct kernel (fp32 leg)
    (2, 16, 16, 128, 128, 3, 1, 1, True, True),       # BasicBlock conv2 with residual through the coalesced loader
    (1, 32, 32, 192, 64, 1, 1, 0, True, False),       # root-like 1x1 over a wide input
]


@pytest.mark.parametrize("prec", ["tf32x3", "bf16", "tf32"])
@pytest.mark.parametrize("shape", CONV_SHAPES)
def test_conv2d_tensor_core(shape, prec, cplib):
    B, H, W, Cin, Cout, k, stride, pad, relu, res = shape
    x, w, b, r, want = _conv_case(B, H, W, Cin, Cout, k, stride, pad, relu, res, seed=sum(shape))
    xh = x.permute(0, 2, 3, 1).contiguous().cuda()
    rh = r.permute(0, 2, 3, 1).contiguous().cuda() if r is not None else None
    got = cpb.conv2d_nhwc(xh, w.cuda(), b.cuda(), rh, stride=stride, pad=pad, relu=relu, precision=prec)
    torch.cuda.synchronize()
    got = got.permute(0, 3, 1, 2).cpu()
    ref32 = cpb.conv2d_nhwc(xh, w.cuda(), b.cuda(), rh, stride=stride, pad=pad, relu=relu, precision="fp32")
    ref32 = ref32.permute(0, 3, 1, 2).cpu()
    mag = want.abs().max().item()
    assert (ref32 - want).abs().max().item() / mag <= TOL["fp32"]
    err = (got - want).abs().max().item() / mag
    print("conv %s %s: rel err %.3e" % (shape, prec, err))
    assert err <= TOL[prec], "wgmma %s conv off by %.3e (tolerance %.1e)" % (prec, err, TOL[prec])


@pytest.mark.parametrize("prec", ["tf32x3", "bf16"])
def test_dcn_tensor_core(prec, cplib):
    from oracle import net_ref
    g = torch.Generator().manual_seed(11)
    for (B, C, H, W, Co) in ((2, 64, 12, 10, 64), (1, 128, 9, 16, 256)):
        x = torch.randn(B, C, H, W, generator=g)
        off = torch.randn(B, 18, H, W, generator=g) * 2.0
        mask = torch.rand(B, 9, H, W, generator=g)
        w = torch.randn(Co, C, 3, 3, generator=g) / np.sqrt(C * 9)
        b = torch.randn(Co, generator=g) * 0.1
        want = net_ref.dcn_v2_forward_ref(x.double(), off.double(), mask.double(), w.double(), b.double()).float()
        got = cpb.dcn_v2_forward(x.cuda(), w.cuda(), b.cuda(), off.cuda(), mask.cuda(), precision=prec).cpu()
        err = (got - want).abs().max().item() / want.abs().max().item()
        print("dcn %s %s: rel err %.3e" % ((B, C, H, W, Co), prec, err))
        assert err <= TOL[prec]


@pytest.mark.parametrize("prec", ["tf32x3", "tf32"])
@pytest.mark.parametrize("off_std", [0.5, 6.0])
def test_dcn_tma_staged(prec, off_std, cplib):
    """Shapes the TMA-staged deformable kernel (dcn_tma.cu) takes: H % 8 == 0, W % 16 == 0, both <= 128.
    off_std 0.5 keeps the corners inside the staged slab, 6.0 sends a large share through the global-memory path;
    both must match the fp64 restatement of dcn_v2_im2col_cuda.cu."""
    from oracle import net_ref
    g = torch.Generator().manual_seed(23)
    for (B, C, H, W, Co) in ((2, 64, 16, 16, 64), (1, 32, 8, 32, 48), (1, 128, 8, 64, 128), (1, 16, 8, 128, 16),
                             (2, 64, 24, 48, 64), (3, 64, 32, 32, 256),
                             (4, 48, 64, 128, 32)):     # 256 tiles > 132 CTAs with an odd number of K blocks
        x = torch.randn(B, C, H, W, generator=g)
        off = torch.randn(B, 18, H, W, generator=g) * off_std
        mask = torch.rand(B, 9, H, W, generator=g)
        w = torch.randn(Co, C, 3, 3, generator=g) / np.sqrt(C * 9)
        b = torch.randn(Co, generator=g) * 0.1
        want = net_ref.dcn_v2_forward_ref(x.double(), off.double(), mask.double(), w.double(), b.double()).float()
        got = cpb.dcn_v2_forward(x.cuda(), w.cuda(), b.cuda(), off.cuda(), mask.cuda(), precision=prec).cpu()
        err = (got - want).abs().max().item() / want.abs().max().item()
        print("dcn_tma %s %s off_std %.1f: rel err %.3e" % ((B, C, H, W, Co), prec, off_std, err))
        assert err <= TOL[prec], "dcn_tma %s %s off by %.3e" % ((B, C, H, W, Co), prec, err)


def _net(arch, trk, wseed, prec):
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.precision = prec
    m.load_state_dict(synth.seeded_state_dict(m, seed=wseed, offset_std=0.3))
    return m.cuda().eval(), opt


@pytest.mark.parametrize("name", ["net_dla34_b2_96x128", "net_dlav1_b1_64x64", "net_dla34track_b1_64x96"])
def test_network_tf32x3_is_fp32_equivalent(name, cplib):
    """The parity-mode tensor-core plan must meet the same stage-B bar as the fp32 CUDA-core plan."""
    g = golden(name)
    m, opt = _net(str(g["arch"]), bool(int(g["tracking"])), int(g["wseed"]), "tf32x3")
    x, extra = net_case_inputs(g)
    out = m(torch.from_numpy(x).cuda(), **{k: torch.from_numpy(v).cuda() for k, v in extra.items()})[-1]
    for h in opt.heads:
        want = g["head_" + h]
        err = np.abs(out[h].cpu().numpy() - want).max() / np.abs(want).max()
        print("tf32x3 %s %s %.3e" % (name, h, err))
        assert err <= TOL_HEAD_REL, (h, err)


def test_network_tf32_drift_is_bounded(cplib):
    """TMA-fed single-pass tf32 plan (the math of PyTorch's default cuDNN convs): report drift, bound it at 5e-2."""
    g = golden("net_dla34_b2_96x128")
    m, opt = _net("dla_34", False, int(g["wseed"]), "tf32")
    x, _ = net_case_inputs(g)
    out = m(torch.from_numpy(x).cuda())[-1]
    for h in opt.heads:
        want = g["head_" + h]
        err = np.abs(out[h].cpu().numpy() - want).max() / np.abs(want).max()
        print("tf32 %s %.3e" % (h, err))
        assert err <= 5e-2, (h, err)


def test_network_bf16_drift_is_bounded(cplib):
    """Fast mode: report the drift.  bf16 operand rounding (4e-3 per layer) is amplified by the deformable sampling of
    the seeded random network to ~0.1 of max|head| -- this mode is a throughput option, not a parity mode; the bound
    below only guards against gross breakage."""
    g = golden("net_dla34_b2_96x128")
    m, opt = _net("dla_34", False, int(g["wseed"]), "bf16")
    x, _ = net_case_inputs(g)
    out = m(torch.from_numpy(x).cuda())[-1]
    for h in opt.heads:
        want = g["head_" + h]
        err = np.abs(out[h].cpu().numpy() - want).max() / np.abs(want).max()
        print("bf16 %s %.3e" % (h, err))
        assert err <= 0.3, (h, err)
