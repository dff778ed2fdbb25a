"""The ResNet backbones without a GPU: the parameter skeleton against the reference's keys and shapes, the errors of
create_model and of the C ABI, the host-side plan layout (cp_plan_memory / cp_plan_allocations) of every res config,
and the ResNet oracle (oracle/net_ref_res.py) against the goldens the unmodified reference produced."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.engine import _config
from tests.util import GOLD, TOL_HEAD_REL, TOL_HEAD_REL_512, golden, net_case_inputs

INVALID = -1      # CP_ERR_INVALID
DEPTHS = (18, 34, 50, 101, 152)
VARIANTS = [("res_%d" % d, False) for d in DEPTHS] + [("res_18", True), ("res_101", True)]


def _keys():
    with open(os.path.join(GOLD, "state_dict_keys_res.json")) as f:
        return json.load(f)


def _name(arch, trk):
    return arch + ("_tracking" if trk else "")


@pytest.mark.parametrize("arch,trk", VARIANTS)
def test_state_dict_matches_reference_keys(arch, trk):
    want = _keys()[_name(arch, trk)]
    opt = cpb.default_opt(arch, tracking_task=trk)
    assert opt.head_conv == want["head_conv"] == 64
    assert dict(opt.heads) == want["heads"]
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    assert isinstance(m, cpb.PoseResNetB200) and m._arch() == arch
    got = [[k, list(v.shape)] for k, v in m.state_dict().items()]
    assert got == want["keys"]


@pytest.mark.parametrize("arch,trk", [("res_18", False), ("res_101", False), ("res_18", True)])
def test_state_dict_matches_live_reference(arch, trk):
    from oracle import ref_shims
    if not ref_shims.reference_available():
        pytest.skip("reference tree not present")
    ref_shims.install()
    from lib.models.networks.msra_resnet import get_pose_net as ref_get
    ropt = ref_shims.make_opt(arch, tracking_task=trk)
    ref = ref_get(int(arch.split("_")[1]), ropt.heads, ropt.head_conv, opt=ropt)
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == \
        [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]


def test_bad_depth_and_head_conv_raise():
    opt = cpb.default_opt("res_18")
    for arch in ("res_10", "res_26", "res_200"):
        with pytest.raises(ValueError, match="res_18"):
            cpb.create_model(arch, opt.heads, 64, opt)
    for hc in (0, -1):
        with pytest.raises(ValueError, match="head_conv"):
            cpb.create_model("res_18", opt.heads, hc, opt)


@pytest.mark.parametrize("arch", ["resdcn_18", "resdcn_101", "hourglass", "dlav0_34"])
def test_untested_upstream_backbones_still_raise_keyerror(arch):
    opt = cpb.default_opt("dla_34")
    with pytest.raises(KeyError):
        cpb.create_model(arch, opt.heads, 64, opt)


def _cfg(arch, trk, B=1, H=512, W=512, prec="tf32x3", gru=False):
    opt = cpb.default_opt(arch, tracking_task=trk)
    cfg, keep = _config(arch, opt.heads, opt.head_conv, B, H, W, 0, trk, gru, prec)
    cfg._keep = keep
    return cfg


def test_res_with_tracking_task_gru_is_invalid(cplib):
    for arch in ("res_18", "res_101"):
        cfg = _cfg(arch, True, gru=True)
        m = _lib.CpMemoryInfo()
        assert cplib.cp_plan_memory(ctypes.byref(cfg), 1, 0, ctypes.byref(m)) == INVALID
        assert b"tracking_task_gru" in cplib.cp_last_error()
        plan = ctypes.c_void_p()
        for flags in (0, _lib.CP_PLAN_REUSE_ACTIVATIONS, _lib.CP_PLAN_MULTI_TRACK):
            assert cplib.cp_plan_create_ex(ctypes.byref(cfg), 1, flags, ctypes.byref(plan)) == INVALID
        assert cplib.cp_plan_create(ctypes.byref(cfg), ctypes.byref(plan)) == INVALID
        assert cplib.cp_plan_create_multi_track(ctypes.byref(cfg), 2, ctypes.byref(plan)) == INVALID
        assert not plan.value


def test_unknown_arch_value_is_invalid(cplib):
    cfg = _cfg("res_18", False)
    cfg.arch = 7
    m = _lib.CpMemoryInfo()
    assert cplib.cp_plan_memory(ctypes.byref(cfg), 1, 0, ctypes.byref(m)) == INVALID
    assert b"unknown arch" in cplib.cp_last_error()


def _memory(cfg, models, flags):
    m = _lib.CpMemoryInfo()
    _lib.check(_lib.load().cp_plan_memory(ctypes.byref(cfg), models, flags, ctypes.byref(m)), "cp_plan_memory")
    return m


def _allocs(cfg, models, flags):
    n = ctypes.c_int32()
    L = _lib.load()
    _lib.check(L.cp_plan_allocations(ctypes.byref(cfg), models, flags, (_lib.CpActAlloc * 1)(), 0, ctypes.byref(n)),
               "cp_plan_allocations")
    buf = (_lib.CpActAlloc * n.value)()
    _lib.check(L.cp_plan_allocations(ctypes.byref(cfg), models, flags, buf, n.value, ctypes.byref(n)), "cp_plan_allocations")
    return [(a.floats, a.off, a.first, a.last) for a in buf]


@pytest.mark.parametrize("prec", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("arch,trk", VARIANTS)
def test_packed_arena_smaller_for_every_res_config(arch, trk, prec, cplib):
    """Every creator's layout: one model, three models (multi, or multi-track for tracking configs), full and packed."""
    cfg = _cfg(arch, trk, B=2, prec=prec)
    reuse = _lib.CP_PLAN_REUSE_ACTIVATIONS
    for models, base in ((1, 0), (3, _lib.CP_PLAN_MULTI_TRACK if trk else 0)):
        full, packed = _memory(cfg, models, base), _memory(cfg, models, base | reuse)
        assert 0 < packed.activation_bytes < full.activation_bytes, (models, packed.activation_bytes, full.activation_bytes)
        assert packed.weight_bytes == full.weight_bytes > 0
        fa, pa = _allocs(cfg, models, base), _allocs(cfg, models, base | reuse)
        assert len(fa) == len(pa)
        # the full layout is the bump allocation; the packed one never overlaps two allocations live at once
        off = 0
        for floats, o, first, last in fa:
            assert o == off
            off += floats
        assert off * 4 == full.activation_bytes
        live = [(o, o + f, a, b) for f, o, a, b in pa if f > 0]
        for i, (o0, e0, a0, b0) in enumerate(live):
            assert e0 * 4 <= packed.activation_bytes
            for o1, e1, a1, b1 in live[i + 1:]:
                if a0 <= b1 and a1 <= b0:
                    assert e0 <= o1 or e1 <= o0


def test_res_tile_and_weight_bytes(cplib):
    """The transposed convs own four phase tile sets in the tensor-core precisions, none in fp32."""
    assert _memory(_cfg("res_18", False, prec="fp32"), 1, 0).tile_bytes < _memory(_cfg("res_18", False), 1, 0).tile_bytes
    w18 = _memory(_cfg("res_18", False), 1, 0).weight_bytes
    w50 = _memory(_cfg("res_50", False), 1, 0).weight_bytes
    assert w18 > 4 * (512 * 256 * 16 + 2 * 256 * 256 * 16) and w50 > w18


@pytest.mark.parametrize("name", ["net_res18_b2_96x128", "net_res50_b1_64x64", "net_res18track_b1_64x96",
                                  "net_res101_b1_512"])
def test_oracle_matches_reference_golden(name):
    from oracle import net_ref_res
    from centerpose_b200 import synth
    g = golden(name)
    arch, trk = str(g["arch"]), bool(int(g["tracking"]))
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sd = synth.seeded_state_dict(m, seed=int(g["wseed"]), offset_std=float(g["offset_std"]))
    x, extra = net_case_inputs(g)
    out = net_ref_res.forward(torch.from_numpy(x), sd, opt.heads, arch,
                              **{k: torch.from_numpy(v) for k, v in extra.items()})
    assert list(out) == list(opt.heads)
    rel = TOL_HEAD_REL_512 if int(g["H"]) >= 512 else TOL_HEAD_REL
    sub = int(g["sub"])
    for h in opt.heads:
        w = g["head_" + h]
        got = out[h].numpy()
        assert got.shape == (int(g["batch"]), opt.heads[h], int(g["H"]) // 4, int(g["W"]) // 4), h
        assert abs(float(np.abs(got).max()) - float(g["absmax_" + h])) <= rel * float(g["absmax_" + h]), h
        e = float(np.abs(got[..., ::sub, ::sub] - w).max()) / max(1e-6, float(g["absmax_" + h]))
        assert e <= rel, (h, e)
