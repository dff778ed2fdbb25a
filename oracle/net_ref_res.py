"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference PoseResNet
forward (res_18 .. res_152, with the optional tracking stems), the ResNet
counterpart of oracle/net_ref.py.

Never imported by the product path (`centerpose_b200/`).  Pure functions over
a flat `state_dict` with the reference's key names, so it is also the
specification of the weights the CUDA plan ingests.  Evaluates in the dtype of
the state_dict (fp64 for the truth the GPU tests compare against).

Parity status: PINNED -- `tests/test_res_cpu.py` checks it against the golden
head tensors `tests/golden/net_res*.npz` made by `oracle/make_golden_res.py`
from the unmodified reference, and against the live reference when present.

Reference lines followed (relative to /root/reference/src/lib/models/networks/msra_resnet.py):
  :35-64    BasicBlock.forward            -> _basic
  :67-105   Bottleneck.forward            -> _bottleneck
  :178-193  _make_layer (downsample)      -> _layer
  :208-233  _make_deconv_layer            -> features (ConvTranspose2d 4x4/2/1, BN, ReLU)
  :116-147, 235-254  PoseResNet.forward   -> features
  :157-174, 255-257  heads                -> forward
  :300-304  resnet_spec                   -> RESNET_SPEC
"""
import torch
import torch.nn.functional as F

from oracle.net_ref import _bn

RESNET_SPEC = {18: (False, [2, 2, 2, 2]), 34: (False, [3, 4, 6, 3]), 50: (True, [3, 4, 6, 3]),
               101: (True, [3, 4, 23, 3]), 152: (True, [3, 8, 36, 3])}


def _conv_bn(x, sd, p, bn, stride=1, pad=0):
    return _bn(F.conv2d(x, sd[p + ".weight"], None, stride, pad), sd, bn)


def _residual(x, sd, p, stride):
    if (p + ".downsample.0.weight") in sd:
        return _conv_bn(x, sd, p + ".downsample.0", p + ".downsample.1", stride, 0)
    return x


def _basic(x, sd, p, stride):
    y = F.relu(_conv_bn(x, sd, p + ".conv1", p + ".bn1", stride, 1))
    y = _conv_bn(y, sd, p + ".conv2", p + ".bn2", 1, 1)
    return F.relu(y + _residual(x, sd, p, stride))


def _bottleneck(x, sd, p, stride):
    y = F.relu(_conv_bn(x, sd, p + ".conv1", p + ".bn1"))
    y = F.relu(_conv_bn(y, sd, p + ".conv2", p + ".bn2", stride, 1))
    y = _conv_bn(y, sd, p + ".conv3", p + ".bn3")
    return F.relu(y + _residual(x, sd, p, stride))


def _stem(x, sd, conv, bn):
    y = F.relu(_bn(F.conv2d(x, sd[conv], None, 2, 3), sd, bn))
    return F.max_pool2d(y, 3, 2, 1)


def depth_of(arch):
    return int(arch.split("_")[1])


def features(x, sd, arch, pre_img=None, pre_hm=None, pre_hm_hp=None):
    """PoseResNet.forward up to the 256-channel stride-4 feature (msra_resnet.py:235-254)."""
    bottleneck, blocks = RESNET_SPEC[depth_of(arch)]
    x = _stem(x, sd, "conv1.weight", "bn1")
    for t, k in ((pre_img, "pre_img_layer"), (pre_hm, "pre_hm_layer"), (pre_hm_hp, "pre_hm_hp_layer")):
        if t is not None:
            x = x + _stem(t, sd, k + ".0.weight", k + ".1")
    block = _bottleneck if bottleneck else _basic
    for i, n in enumerate(blocks):
        for j in range(n):
            x = block(x, sd, "layer%d.%d" % (i + 1, j), 2 if (i > 0 and j == 0) else 1)
    for i in range(3):
        y = F.conv_transpose2d(x, sd["deconv_layers.%d.weight" % (3 * i)], None, stride=2, padding=1)
        x = F.relu(_bn(y, sd, "deconv_layers.%d" % (3 * i + 1)))
    return x


def forward(x, sd, heads, arch="res_18", pre_img=None, pre_hm=None, pre_hm_hp=None):
    """{head: NCHW logits} in `heads` order (3x3 -> ReLU -> 1x1, msra_resnet.py:157-165)."""
    with torch.no_grad():
        f = features(x, sd, arch, pre_img, pre_hm, pre_hm_hp)
        out = {}
        for h in heads:
            y = F.relu(F.conv2d(f, sd[h + ".0.weight"], sd[h + ".0.bias"], 1, 1))
            out[h] = F.conv2d(y, sd[h + ".2.weight"], sd[h + ".2.bias"])
        return out
