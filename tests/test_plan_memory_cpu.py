"""Plan memory without a GPU: cp_plan_memory / cp_plan_allocations (the host-side layout of a plan, with and without
CP_PLAN_REUSE_ACTIVATIONS) and the argument checks of cp_plan_create_ex."""
import ctypes

import pytest

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200.engine import _config, plan_memory

INVALID = -1      # CP_ERR_INVALID
REUSE, MULTI_TRACK = _lib.CP_PLAN_REUSE_ACTIVATIONS, _lib.CP_PLAN_MULTI_TRACK

# (arch, tracking_task): the four network variants a plan builds
ARCHS = [("dla_34", False), ("dlav1_34", False), ("dla_34", True), ("dlav1_34", True)]


def net_config(arch, trk, B=1, H=512, W=512, prec="tf32x3"):
    opt = cpb.default_opt(arch, tracking_task=trk)
    cfg, keep = _config(arch, opt.heads, opt.head_conv, B, H, W, 0, trk, arch == "dlav1_34" and trk, prec)
    cfg._keep = keep
    return cfg


def allocations(cfg, models, flags):
    """cp_plan_allocations: list of dicts(floats, off, first, last)."""
    n = ctypes.c_int32()
    assert _lib.load().cp_plan_allocations(ctypes.byref(cfg), models, flags, None, 0, ctypes.byref(n)) == INVALID
    buf = (_lib.CpActAlloc * 1)()
    _lib.check(_lib.load().cp_plan_allocations(ctypes.byref(cfg), models, flags, buf, 0, ctypes.byref(n)),
               "cp_plan_allocations")
    buf = (_lib.CpActAlloc * n.value)()
    _lib.check(_lib.load().cp_plan_allocations(ctypes.byref(cfg), models, flags, buf, n.value, ctypes.byref(n)),
               "cp_plan_allocations")
    return [dict(floats=a.floats, off=a.off, first=a.first, last=a.last) for a in buf]


def memory(cfg, models=1, flags=0):
    m = _lib.CpMemoryInfo()
    _lib.check(_lib.load().cp_plan_memory(ctypes.byref(cfg), models, flags, ctypes.byref(m)), "cp_plan_memory")
    return m


@pytest.mark.parametrize("flags", [4, 0x80000000, REUSE | 8])
def test_unknown_flags_rejected(cplib, flags):
    cfg = net_config("dla_34", False)
    m = _lib.CpMemoryInfo()
    assert cplib.cp_plan_memory(ctypes.byref(cfg), 1, flags, ctypes.byref(m)) == INVALID
    assert b"unknown flags" in cplib.cp_last_error()
    plan = ctypes.c_void_p()
    assert cplib.cp_plan_create_ex(ctypes.byref(cfg), 1, flags, ctypes.byref(plan)) == INVALID
    assert b"cp_plan_create_ex: unknown flags" in cplib.cp_last_error()
    assert not plan.value


def test_bad_arguments_rejected(cplib):
    m = _lib.CpMemoryInfo()
    cfg = net_config("dla_34", False)
    assert cplib.cp_plan_memory(None, 1, 0, ctypes.byref(m)) == INVALID
    assert cplib.cp_plan_memory(ctypes.byref(cfg), 1, 0, None) == INVALID
    assert b"null" in cplib.cp_last_error()
    for n in (0, -1, _lib.CP_MAX_MODELS + 1):
        assert cplib.cp_plan_memory(ctypes.byref(cfg), n, REUSE, ctypes.byref(m)) == INVALID
        assert b"num_models" in cplib.cp_last_error()
    assert cplib.cp_plan_memory(ctypes.byref(cfg), 2, MULTI_TRACK, ctypes.byref(m)) == INVALID
    assert b"tracking" in cplib.cp_last_error()
    trk = net_config("dla_34", True)
    assert cplib.cp_plan_memory(ctypes.byref(trk), 2, REUSE, ctypes.byref(m)) == INVALID
    assert b"CP_PLAN_MULTI_TRACK" in cplib.cp_last_error()
    assert cplib.cp_plan_memory(ctypes.byref(trk), 2, REUSE | MULTI_TRACK, ctypes.byref(m)) == 0
    bad = net_config("dla_34", False, H=100)
    assert cplib.cp_plan_memory(ctypes.byref(bad), 1, REUSE, ctypes.byref(m)) == INVALID
    assert b"multiples of 32" in cplib.cp_last_error()
    bad = net_config("dla_34", False, prec="fp32")
    bad.precision = 9
    assert cplib.cp_plan_memory(ctypes.byref(bad), 1, 0, ctypes.byref(m)) == INVALID
    n = ctypes.c_int32()
    assert cplib.cp_plan_allocations(ctypes.byref(cfg), 1, 16, (_lib.CpActAlloc * 1)(), 1, ctypes.byref(n)) == INVALID
    plan = ctypes.c_void_p()
    assert cplib.cp_plan_create_ex(ctypes.byref(cfg), 1, 0, None) == INVALID
    assert cplib.cp_plan_create_ex(None, 1, 0, ctypes.byref(plan)) == INVALID
    assert cplib.cp_plan_create_ex(ctypes.byref(trk), 3, 0, ctypes.byref(plan)) == INVALID
    assert b"CP_PLAN_MULTI_TRACK" in cplib.cp_last_error()
    assert not plan.value


def test_existing_creators_keep_their_messages(cplib):
    plan = ctypes.c_void_p()
    assert cplib.cp_plan_create_multi(ctypes.byref(net_config("dla_34", True)), 2, ctypes.byref(plan)) == INVALID
    assert b"cp_plan_create_multi: a tracking plan made here holds one model" in cplib.cp_last_error()
    assert cplib.cp_plan_create_multi_track(ctypes.byref(net_config("dla_34", False)), 2, ctypes.byref(plan)) == INVALID
    assert b"cp_plan_create_multi_track: needs a tracking config" in cplib.cp_last_error()


# Without the flag the arena is the bump allocation plans have always made, every activation in its own region:
# (dla_34 heads, 512 x 512, batch 1) 288.4 MiB, 402.7 MiB with the tracking stems.
FULL_512_B1 = {("dla_34", False): 302415872, ("dla_34", True): 422281216}


@pytest.mark.parametrize("arch,trk", ARCHS)
@pytest.mark.parametrize("B,M", [(1, 1), (8, 1), (2, 3)])
def test_reuse_arena_is_smaller(cplib, arch, trk, B, M):
    cfg = net_config(arch, trk, B)
    mt = MULTI_TRACK if trk and M > 1 else 0
    full, reuse = memory(cfg, M, mt), memory(cfg, M, mt | REUSE)
    assert reuse.activation_bytes < full.activation_bytes / 4, (reuse.activation_bytes, full.activation_bytes)
    for f in ("weight_bytes", "tile_bytes", "workspace_bytes"):
        assert getattr(reuse, f) == getattr(full, f), f
    assert full.weight_bytes > 0 and full.tile_bytes > 0 and full.workspace_bytes > 0
    if (B, M) == (1, 1) and (arch, trk) in FULL_512_B1:
        assert full.activation_bytes == FULL_512_B1[(arch, trk)]


@pytest.mark.parametrize("arch,trk", ARCHS)
def test_full_layout_is_the_bump_allocation(cplib, arch, trk):
    """Without the flag every allocation has its own memory, in schedule order, each rounded to 64 floats."""
    cfg = net_config(arch, trk, 2, 256, 320)
    al = allocations(cfg, 1, 0)
    at = 0
    for a in al:
        assert a["off"] == at and a["floats"] % 64 == 0
        at += a["floats"]
    assert at * 4 == memory(cfg).activation_bytes


@pytest.mark.parametrize("arch,trk", ARCHS)
@pytest.mark.parametrize("prec", ["fp32", "tf32x3"])
def test_reuse_layout_is_valid(cplib, arch, trk, prec):
    """Allocations live at the same op never share memory, offsets keep the 64-float alignment, the arena is at least the
    largest live sum, the head buffers live to the end of the call, and the merged heads' hidden tile has no memory
    exactly when its 1x1s are fused (tf32x3 on dla_34)."""
    cfg = net_config(arch, trk, 1, 512, 512, prec)
    al = allocations(cfg, 1, REUSE)
    arena = memory(cfg, 1, REUSE).activation_bytes // 4
    n_ops = max(a["last"] for a in al)
    live = [0] * (n_ops + 1)
    for a in al:
        if a["off"] < 0:
            assert a["first"] < 0 and a["floats"] == 0
            continue
        assert a["off"] % 64 == 0 and a["floats"] % 64 == 0 and a["off"] + a["floats"] <= arena
        for t in range(a["first"], a["last"] + 1):
            live[t] += a["floats"]
    assert arena >= max(live)
    used = [a for a in al if a["off"] >= 0]
    for i, a in enumerate(used):
        for b in used[i + 1:]:
            if a["first"] <= b["last"] and b["first"] <= a["last"]:
                assert a["off"] + a["floats"] <= b["off"] or b["off"] + b["floats"] <= a["off"], (a, b)
    heads = len(cpb.default_opt(arch, tracking_task=trk).heads)
    assert all(a["last"] == n_ops for a in al[-heads:])
    unused = [a for a in al if a["off"] < 0]
    assert len(unused) == (1 if (arch, prec) == ("dla_34", "tf32x3") else 0)
    assert allocations(cfg, 1, REUSE) == al          # deterministic


def test_plan_memory_helper(cplib):
    opt = cpb.default_opt("dla_34")
    full = plan_memory("dla_34", opt.heads, opt.head_conv, 1, 512, 512, precision="tf32x3")
    reuse = plan_memory("dla_34", opt.heads, opt.head_conv, 1, 512, 512, precision="tf32x3", reuse_activations=True)
    assert full["activation"] == FULL_512_B1[("dla_34", False)]
    assert reuse["total"] == reuse["activation"] + reuse["weights"] + reuse["tiles"] + reuse["workspace"]
    assert reuse["total"] < full["total"]
