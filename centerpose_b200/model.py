"""`create_model` / `load_model` / `save_model` for the H100-native CenterPose
network -- the drop-in for /root/reference/src/lib/models/model.py:26-105.

`create_model(arch, heads, head_conv, opt)` returns an `nn.Module` whose
`state_dict()` has exactly the reference's keys and shapes (SURVEY.md
Appendix A: 416 / 439 / 450 keys for dla_34 / dlav1_34 / dla_34-tracking), so
reference checkpoints load unchanged, and whose
`forward(x, pre_img=None, pre_hm=None, pre_hm_hp=None) -> [ {head: logits} ]`
(pose_dla_dcn.py:523-570) runs the hand-written sm_90a plan in
libcenterpose_b200.so.  The sub-modules below only HOLD parameters under the
reference's names; no PyTorch operator ever runs on the hot path and there is
no CPU fallback -- calling forward without CUDA raises.
"""
import ctypes
import math

import torch
from torch import nn

from . import _lib


# ----------------------------------------------------------------------------- parameter holders
def _conv(cin, cout, k, bias=False):
    return nn.Conv2d(cin, cout, k, bias=bias)


def _conv_bn_seq(cin, cout, k):
    return nn.Sequential(_conv(cin, cout, k), nn.BatchNorm2d(cout), nn.ReLU(inplace=True))


class _Holder(nn.Module):
    def forward(self, *a, **k):        # pragma: no cover
        raise RuntimeError("parameter holder: the network runs inside libcenterpose_b200.so")


def _block(cin, cout):
    m = _Holder()
    m.conv1, m.bn1 = _conv(cin, cout, 3), nn.BatchNorm2d(cout)
    m.conv2, m.bn2 = _conv(cout, cout, 3), nn.BatchNorm2d(cout)
    return m


def _root(cin, cout):
    m = _Holder()
    m.conv, m.bn = _conv(cin, cout, 1), nn.BatchNorm2d(cout)
    return m


def _tree(levels, cin, cout, level_root=False, root_dim=0):
    """Parameter skeleton of pose_dla_dcn.py:171-209."""
    m = _Holder()
    if root_dim == 0:
        root_dim = 2 * cout
    if level_root:
        root_dim += cin
    if levels == 1:
        m.tree1, m.tree2 = _block(cin, cout), _block(cout, cout)
        m.root = _root(root_dim, cout)
    else:
        m.tree1 = _tree(levels - 1, cin, cout)
        m.tree2 = _tree(levels - 1, cout, cout, root_dim=root_dim + cout)
    if cin != cout:
        m.project = nn.Sequential(_conv(cin, cout, 1), nn.BatchNorm2d(cout))
    return m


class _DCN(_Holder):
    def __init__(self, cin, cout):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, 3, 3))
        self.bias = nn.Parameter(torch.zeros(cout))
        self.conv_offset_mask = nn.Conv2d(cin, 27, 3, padding=1, bias=True)
        stdv = 1.0 / math.sqrt(cin * 9)
        with torch.no_grad():
            self.weight.uniform_(-stdv, stdv)
            self.conv_offset_mask.weight.zero_()
            self.conv_offset_mask.bias.zero_()


def _deform(cin, cout):
    m = _Holder()
    m.actf = nn.Sequential(nn.BatchNorm2d(cout), nn.ReLU(inplace=True))
    m.conv = _DCN(cin, cout)
    return m


def _ida(o, channels, up_f):
    m = _Holder()
    for i in range(1, len(channels)):
        f = int(up_f[i])
        setattr(m, "proj_%d" % i, _deform(channels[i], o))
        up = nn.ConvTranspose2d(o, o, f * 2, stride=f, padding=f // 2, groups=o, bias=False)
        with torch.no_grad():
            k = f * 2
            fc = math.ceil(k / 2)
            c = (2 * fc - 1 - fc % 2) / (2.0 * fc)
            ax = torch.tensor([1 - abs(i_ / fc - c) for i_ in range(k)])
            up.weight.copy_((ax[:, None] * ax[None, :]).expand(o, 1, k, k))
        setattr(m, "up_%d" % i, up)
        setattr(m, "node_%d" % i, _deform(o, o))
    return m


def _gru_cell(c):
    m = _Holder()
    for n, bias in (("Wir", True), ("Whr", False), ("Wiz", True), ("Whz", False), ("Win", True), ("Whn", False)):
        setattr(m, n, nn.Conv2d(c, c, 3, 1, 1, bias=bias))
    return m


_CH = [16, 32, 64, 128, 256, 512]


def _flag(opt, name):
    return bool(getattr(opt, name, False)) if opt is not None else False


class DLASegB200(nn.Module):
    """H100-native DLASeg (pose_dla_dcn.py:457-570).

    `precision` selects the kernels of the plan (include/centerpose_b200.h cp_precision): "tf32x3" (default: wgmma
    3-term split with promoted accumulation, fp32-equivalent - meets the same parity bar as "fp32"), "fp32" (CUDA-core
    FFMA), "tf32" (wgmma single pass), "bf16"."""

    def __init__(self, heads, head_conv=256, use_convGRU=False, opt=None, precision="tf32x3"):
        super().__init__()
        self.opt = opt
        self.heads = dict(heads)
        self.head_conv = head_conv
        self.use_convGRU = bool(use_convGRU)
        self.tracking_inputs = _flag(opt, "pre_img") or _flag(opt, "pre_hm") or _flag(opt, "pre_hm_hp")
        if self.tracking_inputs and not (_flag(opt, "pre_img") and _flag(opt, "pre_hm") and _flag(opt, "pre_hm_hp")):
            raise ValueError("centerpose_b200 supports the tracking stems only as the full "
                             "pre_img + pre_hm + pre_hm_hp set (demo.py:117-123)")
        self.tracking_task = _flag(opt, "tracking_task")
        self.precision = precision
        if head_conv <= 0:
            raise ValueError("head_conv must be > 0 (the reference's DLA default is 256, opts.py:344-345)")

        base = _Holder()
        base.base_layer = _conv_bn_seq(3, 16, 7)
        base.level0 = _conv_bn_seq(16, 16, 3)
        base.level1 = _conv_bn_seq(16, 32, 3)
        base.level2 = _tree(1, 32, 64)
        base.level3 = _tree(2, 64, 128, level_root=True)
        base.level4 = _tree(2, 128, 256, level_root=True)
        base.level5 = _tree(1, 256, 512, level_root=True)
        if self.tracking_inputs:
            base.pre_img_layer = _conv_bn_seq(3, 16, 7)
            base.pre_hm_layer = _conv_bn_seq(1, 16, 7)
            base.pre_hm_hp_layer = _conv_bn_seq(8, 16, 7)
        base.fc = nn.Conv2d(512, 1000, 1, bias=True)      # created by load_pretrained_model (:332-334); unused
        self.base = base

        dla_up = _Holder()
        channels = _CH[2:]
        in_ch = list(channels)
        scales = [1, 2, 4, 8]
        for i in range(len(channels) - 1):
            j = -i - 2
            setattr(dla_up, "ida_%d" % i, _ida(channels[j], in_ch[j:], [s // scales[j] for s in scales[j:]]))
            scales[j + 1:] = [scales[j]] * len(scales[j + 1:])
            in_ch[j + 1:] = [channels[j]] * len(in_ch[j + 1:])
        self.dla_up = dla_up
        if self.use_convGRU:
            g = _Holder()
            g.cell0 = _gru_cell(64)
            self.convGRU = g
        self.ida_up = _ida(64, _CH[2:5], [1, 2, 4])
        for head, classes in self.heads.items():
            mods = [nn.Conv2d(64, head_conv, 3, padding=1, bias=True)]
            if self.use_convGRU:
                mods.append(nn.GroupNorm(32 if head_conv % 32 == 0 else 16, head_conv))
            mods += [nn.ReLU(inplace=True), nn.Conv2d(head_conv, classes, 1, bias=True)]
            fc = nn.Sequential(*mods)
            with torch.no_grad():
                if "hm" in head:
                    fc[-1].bias.fill_(-2.19)
                else:
                    for m in fc.modules():
                        if isinstance(m, nn.Conv2d) and m.bias is not None:
                            m.bias.zero_()
            setattr(self, head, fc)
        self._engines = {}
        self._weights_sig = None

    # ------------------------------------------------------------------ native plan management
    def _signature(self):
        sig = []
        for t in list(self.parameters()) + list(self.buffers()):
            sig.append((t.data_ptr(), t._version))
        return hash(tuple(sig))

    def engine(self, batch, height, width, device=None):
        """The native engine for this input shape (created on first use).  Its activation arena is packed by liveness
        (Engine reuse_activations): the results are the same bits as a full arena's in a fraction of the memory."""
        from .engine import Engine
        device = device if device is not None else next(self.parameters()).device
        if device.type != "cuda":
            raise RuntimeError("centerpose_b200: the network only runs on CUDA (sm_90a); "
                               "there is no CPU fallback -- move the model with .to('cuda')")
        key = (height, width, device.index if device.index is not None else torch.cuda.current_device(), self.precision)
        eng = self._engines.get(key)
        if eng is None or eng.max_batch < batch:
            if eng is not None:
                eng.close()
            eng = Engine(self._arch(), self.heads, self.head_conv, max(batch, 1), height, width, key[2],
                         tracking=self.tracking_inputs, tracking_task_gru=self.use_convGRU and self.tracking_task,
                         precision=self.precision, reuse_activations=True)
            eng.weights_sig = None
            self._engines[key] = eng
        sig = self._signature()
        if eng.weights_sig != sig:
            eng.load_state_dict(self.state_dict())
            eng.weights_sig = sig
        return eng

    def _arch(self):
        return "dlav1_34" if self.use_convGRU else "dla_34"

    def forward(self, x, pre_img=None, pre_hm=None, pre_hm_hp=None):
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("expected NCHW input with 3 channels")
        if not x.is_cuda:
            raise RuntimeError("centerpose_b200: forward needs a CUDA tensor (no CPU fallback)")
        B, _, H, W = x.shape
        eng = self.engine(B, H, W, x.device)
        with torch.no_grad():
            out = eng.forward(x, pre_img, pre_hm, pre_hm_hp)
        return [out]

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        for e in self._engines.values():
            e.weights_sig = None
        return r


def get_pose_net(num_layers, heads, head_conv=256, down_ratio=4, opt=None):
    """'dla' factory (pose_dla_dcn.py:573-580)."""
    if num_layers != 34 or down_ratio != 4:
        raise ValueError("centerpose_b200 implements dla_34 at down_ratio 4")
    return DLASegB200(heads, head_conv, use_convGRU=False, opt=opt)


def get_dla_dcn_convGRU(num_layers, heads, head_conv=256, down_ratio=4, opt=None):
    """'dlav1' factory (pose_dla_dcn.py:583-590)."""
    if num_layers != 34 or down_ratio != 4:
        raise ValueError("centerpose_b200 implements dlav1_34 at down_ratio 4")
    return DLASegB200(heads, head_conv, use_convGRU=True, opt=opt)


_model_factory = {"dla": get_pose_net, "dlav1": get_dla_dcn_convGRU}


def create_model(arch, heads, head_conv, opt=None):
    """models/model.py:26-31."""
    num_layers = int(arch[arch.find("_") + 1:]) if "_" in arch else 0
    name = arch[:arch.find("_")] if "_" in arch else arch
    if name not in _model_factory:
        raise KeyError("centerpose_b200 implements the 'dla' and 'dlav1' backbones; got '%s'" % arch)
    return _model_factory[name](num_layers=num_layers, heads=heads, head_conv=head_conv, opt=opt)


def _load_checkpoint(model_path):
    """Checkpoints are downloaded files: unpickle with `weights_only=True` (reference checkpoints hold only
    `epoch`, `state_dict` and `optimizer` tensors/ints).  A checkpoint that needs arbitrary pickled classes is only
    loaded when CENTERPOSE_B200_UNSAFE_LOAD=1 is set explicitly."""
    import os
    import warnings
    try:
        return torch.load(model_path, map_location="cpu", weights_only=True)
    except Exception as e:            # pickle.UnpicklingError and friends
        if os.environ.get("CENTERPOSE_B200_UNSAFE_LOAD", "") != "1":
            raise RuntimeError("load_model: %s cannot be read with weights_only=True (%s); set "
                               "CENTERPOSE_B200_UNSAFE_LOAD=1 to unpickle it anyway if you trust the file"
                               % (model_path, e))
        warnings.warn("load_model: unpickling %s with weights_only=False (arbitrary code execution risk)" % model_path)
        return torch.load(model_path, map_location="cpu", weights_only=False)


def load_model(model, model_path, optimizer=None, resume=False, lr=None, lr_step=None):
    """models/model.py:34-87: strips `module.`, tolerates shape mismatches and
    missing keys with the same messages, restores the optimizer on resume."""
    start_epoch = 0
    checkpoint = _load_checkpoint(model_path)
    print("loaded {}, epoch {}".format(model_path, checkpoint["epoch"]))
    state_dict = {}
    for k, v in checkpoint["state_dict"].items():
        if k.startswith("module") and not k.startswith("module_list"):
            state_dict[k[7:]] = v
        else:
            state_dict[k] = v
    own = model.state_dict()
    msg = ("If you see this, your model does not fully load the pre-trained weight. Please make sure you have "
           "correctly specified --arch xxx or set the correct --num_classes for your own dataset.")
    for k in state_dict:
        if k in own:
            if state_dict[k].shape != own[k].shape:
                print("Skip loading parameter {}, required shape{}, loaded shape{}. {}".format(
                    k, own[k].shape, state_dict[k].shape, msg))
                state_dict[k] = own[k]
        else:
            print("Drop parameter {}.".format(k) + msg)
    for k in own:
        if k not in state_dict:
            print("No param {}.".format(k) + msg)
            state_dict[k] = own[k]
    model.load_state_dict(state_dict, strict=False)
    if optimizer is not None and resume:
        if "optimizer" in checkpoint:
            optimizer.load_state_dict(checkpoint["optimizer"])
            start_epoch = checkpoint["epoch"]
            start_lr = lr
            for step in lr_step:
                if start_epoch >= step:
                    start_lr *= 0.1
            for group in optimizer.param_groups:
                group["lr"] = start_lr
            print("Resumed optimizer with start lr", start_lr)
        else:
            print("No optimizer parameters in checkpoint.")
    if optimizer is not None:
        return model, optimizer, start_epoch
    return model


def save_model(path, epoch, model, optimizer=None):
    """models/model.py:90-105 (legacy, non-zip serialisation)."""
    sd = model.module.state_dict() if isinstance(model, torch.nn.DataParallel) else model.state_dict()
    data = {"epoch": epoch, "state_dict": sd}
    if optimizer is not None:
        data["optimizer"] = optimizer.state_dict()
    torch.save(data, path, _use_new_zipfile_serialization=False)
