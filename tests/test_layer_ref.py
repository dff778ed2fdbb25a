"""The per-layer checker (tests/layer_ref.py) can fail: synthetic "kernel outputs" made on the CPU with the defects a
tensor-core launch could have must score above the ceilings of tests/util.py, and a correct fp32 evaluation under
them.  Needs no GPU."""
import torch
import torch.nn.functional as F

from oracle import net_ref
from tests import layer_ref
from tests.util import LAYER_CEIL

G = torch.Generator().manual_seed(7)


def _tf32(t):
    """Round to tf32 (10 explicit mantissa bits), nearest-even on the 13 dropped bits."""
    i = t.float().contiguous().view(torch.int32).to(torch.int64)
    i = (i + 0xFFF + ((i >> 13) & 1)) & ~0x1FFF
    return i.to(torch.int32).view(torch.float32)


def _conv_case(B=2, Cin=256, Cout=64, H=12, W=12):
    x = torch.randn(B, Cin, H, W, generator=G)
    w = torch.randn(Cout, Cin, 3, 3, generator=G) / (Cin * 9) ** 0.5
    b = torch.randn(Cout, generator=G) * 0.1
    ref, S = layer_ref.conv_ref(x.double(), w.double(), b.double(), 1, 1, False)
    return x, w, b, ref, S


def _r(got, ref, S):
    return layer_ref.score(got, ref, S)


def test_correct_fp32_conv_passes():
    x, w, b, ref, S = _conv_case()
    assert _r(F.conv2d(x, w, b, 1, 1), ref, S) <= LAYER_CEIL["fp32"]


def test_tf32_operands_fail_the_fp32_ceiling():
    x, w, b, ref, S = _conv_case()
    got = F.conv2d(_tf32(x).double(), _tf32(w).double(), b.double(), 1, 1).float()
    r = _r(got, ref, S)
    assert r > LAYER_CEIL["fp32"] * 10, r
    assert r <= LAYER_CEIL["tf32"], r


def test_dropped_k_slab_fails_every_ceiling():
    x, w, b, ref, S = _conv_case()
    x2 = x.clone()
    x2[:, 96:128] = 0          # one 32-channel slab of the K loop never accumulated
    r = _r(F.conv2d(x2, w, b, 1, 1), ref, S)
    assert r > max(LAYER_CEIL.values()), r


def test_tile_without_bias_fails():
    x, w, b, ref, S = _conv_case()
    got = F.conv2d(x, w, b, 1, 1)
    nhwc = got.permute(0, 2, 3, 1).reshape(-1, got.shape[1])
    nhwc[128:256] -= b         # the second 128-row M tile lost its bias
    got = nhwc.reshape(got.shape[0], got.shape[2], got.shape[3], -1).permute(0, 3, 1, 2)
    assert _r(got, ref, S) > max(LAYER_CEIL.values())


def test_dcn_mask_without_sigmoid_fails():
    B, C, H, W, Co = 1, 32, 10, 12, 16
    x = torch.randn(B, C, H, W, generator=G).double()
    om = torch.randn(B, 27, H, W, generator=G).double()
    om[:, :18] *= 1.5
    w = torch.randn(Co, C, 3, 3, generator=G).double() / (C * 9) ** 0.5
    b = torch.randn(Co, generator=G).double() * 0.1
    ref, S = layer_ref.dcn_ref(x, om, w, b, relu=True)
    good = net_ref.dcn_v2_forward_ref(x.float(), om[:, :18].float(), torch.sigmoid(om[:, 18:]).float(), w.float(),
                                      b.float()).clamp_min(0)
    assert _r(good, ref, S) <= LAYER_CEIL["fp32"]
    mask = torch.sigmoid(om[:, 18:])
    mask[:, 4] = om[:, 18 + 4]  # the centre tap's logit used as the mask
    bad = net_ref.dcn_v2_forward_ref(x, om[:, :18], mask, w, b).clamp_min(0)
    assert _r(bad, ref, S) > max(LAYER_CEIL.values())


def test_fused_head_reading_wrong_hidden_half_fails():
    B, H, W, hid = 1, 8, 8, 256
    hidden = torch.randn(B, 2 * hid, H, W, generator=G).double().clamp_min(0)
    S_hidden = hidden.abs() * 1.0
    W1 = torch.randn(16, hid, 1, 1, generator=G).double() / hid ** 0.5
    b1 = torch.randn(16, generator=G).double() * 0.1
    ref, S = layer_ref.fused_head_ref(hidden[:, :hid], S_hidden[:, :hid], W1, b1)
    good = F.conv2d(hidden[:, :hid].float(), W1.float(), b1.float())
    assert _r(good, ref, S) <= LAYER_CEIL["fp32"]
    # the first 128 hidden channels are read from the other head's tile
    wrong = torch.cat([hidden[:, hid:hid + 128], hidden[:, 128:hid]], 1)
    bad = F.conv2d(wrong.float(), W1.float(), b1.float())
    assert _r(bad, ref, S) > max(LAYER_CEIL.values())


def test_elementwise_references_match_torch():
    x = torch.randn(2, 64, 8, 10, generator=G).double()
    gamma, beta = torch.rand(64, generator=G) + 0.5, torch.randn(64, generator=G)
    ref, S = layer_ref.gn_relu_ref(x, gamma, beta, 32)
    assert torch.allclose(ref, F.relu(F.group_norm(x, 32, gamma.double(), beta.double(), 1e-5)), atol=1e-12)
    assert (S >= ref.abs()).all()
    gx = torch.randn(2, 192, 4, 4, generator=G).double()
    gh = torch.randn(2, 192, 4, 4, generator=G).double()
    h = torch.randn(2, 64, 4, 4, generator=G).double()
    ref, S = layer_ref.gru_ref(gx, gh, h)
    r = torch.sigmoid(gx[:, :64] + gh[:, :64])
    z = torch.sigmoid(gx[:, 64:128] + gh[:, 64:128])
    n = torch.tanh(gx[:, 128:] + r * gh[:, 128:])
    assert torch.allclose(ref, (1 - z) * n + z * h, atol=1e-14)
    ref0, _ = layer_ref.gru_ref(gx, None, None)
    z0 = torch.sigmoid(gx[:, 64:128])
    assert torch.allclose(ref0, (1 - z0) * torch.tanh(gx[:, 128:]), atol=1e-14)
