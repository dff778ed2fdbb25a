"""Batch-invariant plans (CP_PLAN_BATCH_INVARIANT) without a device: the fixed K segments of every launch depend on the
layer's shape only, the flag costs no memory, and the network carries it into the plans it builds."""
import ctypes

import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200 import engine as E
from centerpose_b200.engine import _config

NETS = [("dla_34", False), ("dlav1_34", False), ("res_18", False), ("dla_34", True)]
# G of every tf32x3 launch of dla_34 at 512 x 512 that has more than one segment, in schedule order
DLA34_512 = [2, 4, 4, 4, 4, 4, 4, 4, 4, 2, 4, 4, 4, 4, 8, 4, 4, 4, 4, 7, 8, 8, 8, 8, 10, 16, 32, 8, 8, 8, 16, 4, 4, 8,
             16, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 8, 16]


def _segs(arch, trk, prec, max_batch=1, models=1, invariant=True, H=512, W=512):
    opt = cpb.default_opt(arch, tracking_task=trk)
    return E.plan_ksegments(opt.arch, opt.heads, opt.head_conv, max_batch, H, W, tracking=trk,
                            tracking_task_gru=arch.startswith("dlav1") and trk, precision=prec, models=models,
                            batch_invariant=invariant)


@pytest.mark.parametrize("prec", ["tf32x3", "tf32"])
@pytest.mark.parametrize("arch,trk", NETS)
def test_segments_depend_on_the_shape_only(arch, trk, prec):
    g = _segs(arch, trk, prec)
    assert all(x >= 1 for x in g)
    # tf32 splits only the deformable convs, which the ResNets do not have
    assert any(x > 1 for x in g) == (prec == "tf32x3" or not arch.startswith("res"))
    for mb in (2, 8, 32):
        for models in (1, 3):
            assert _segs(arch, trk, prec, mb, models) == g, (mb, models)
    # no device was asked for its SM count: the rule's 132 is a constant
    assert _segs(arch, trk, prec, invariant=False) == [0] * len(g)
    if (arch, trk, prec) == ("dla_34", False, "tf32x3"):
        assert [x for x in g if x > 1] == DLA34_512


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_fp32_bf16_never_split(prec):
    assert set(_segs("dla_34", False, prec)) == {1}


@pytest.mark.parametrize("reuse", [False, True])
@pytest.mark.parametrize("arch,trk", NETS)
def test_memory_is_the_defaults(arch, trk, reuse):
    opt = cpb.default_opt(arch, tracking_task=trk)
    for models in (1, 2):
        kw = dict(tracking=trk, tracking_task_gru=False, precision="tf32x3", models=models, reuse_activations=reuse)
        a = E.plan_memory(opt.arch, opt.heads, opt.head_conv, 8, 512, 512, batch_invariant=True, **kw)
        b = E.plan_memory(opt.arch, opt.heads, opt.head_conv, 8, 512, 512, **kw)
        assert a == b


def test_flags_combine_and_unknown_bits_refused():
    L = _lib.load()
    opt = cpb.default_opt("dla_34", tracking_task=True)
    cfg, keep = _config(opt.arch, dict(opt.heads), opt.head_conv, 2, 256, 256, 0, True, False, "tf32x3")
    m = _lib.CpMemoryInfo()
    every = _lib.CP_PLAN_BATCH_INVARIANT | _lib.CP_PLAN_REUSE_ACTIVATIONS | _lib.CP_PLAN_MULTI_TRACK
    assert L.cp_plan_memory(ctypes.byref(cfg), 2, every, ctypes.byref(m)) == 0
    assert L.cp_plan_memory(ctypes.byref(cfg), 2, every | 8, ctypes.byref(m)) != 0
    assert "unknown flags" in L.cp_last_error().decode()


class _Stub(object):
    made = []

    def __init__(self, *a, **k):
        self.max_batch = a[3]
        self.weights_sig = None
        _Stub.made.append(k)

    def load_state_dict(self, sd, model=0):
        pass

    def close(self):
        pass


@pytest.mark.parametrize("flag", [False, True])
def test_network_carries_the_flag_into_its_plans(monkeypatch, flag):
    monkeypatch.setattr(E, "Engine", _Stub)
    _Stub.made = []
    opt = cpb.default_opt("dla_34", batch_invariant=flag)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    assert m.batch_invariant is flag
    m.engine(1, 512, 512, device=torch.device("cuda", 0))
    m.engine(4, 512, 512, device=torch.device("cuda", 0))        # a larger batch: a new plan, same flag
    assert [k["batch_invariant"] for k in _Stub.made] == [flag, flag]
    # the engine cache keys on the flag: switching it builds a new plan
    m.batch_invariant = not flag
    m.engine(1, 512, 512, device=torch.device("cuda", 0))
    assert _Stub.made[-1]["batch_invariant"] is (not flag)


def test_reference_namespace_without_the_field():
    class Ns(object):
        pass
    o = Ns()
    for k, v in vars(cpb.default_opt("dla_34")).items():
        if k != "batch_invariant":
            setattr(o, k, v)
    m = cpb.create_model(o.arch, o.heads, o.head_conv, o)
    assert m.batch_invariant is False


def _bare_detector_init(self, opt, model=None):
    """ObjectPoseDetector.__init__ without the device: the multi-category set-up keeps opt and drops the model."""
    opt.device = torch.device("cuda", 0)
    self.opt = opt
    self.model = model
    self.tracker = None
    self._slots = None


@pytest.fixture()
def stubbed(monkeypatch):
    """Engine replaced by the recording stub wherever the package binds it, and the detector set-up made device-free."""
    from centerpose_b200 import detector as D
    monkeypatch.setattr(E, "Engine", _Stub)
    monkeypatch.setattr(D, "Engine", _Stub)
    monkeypatch.setattr(D.ObjectPoseDetector, "__init__", _bare_detector_init)
    _Stub.made = []
    return D


def _checkpoints(tmp_path, trk, cats=("chair", "cup")):
    opt = cpb.default_opt("dla_34", tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    paths = {}
    for c in cats:
        paths[c] = str(tmp_path / ("%s_%d.pth" % (c, trk)))
        cpb.save_model(paths[c], 1, m)
    return paths


@pytest.mark.parametrize("flag", [False, True])
def test_every_engine_the_package_builds_carries_the_flag(stubbed, tmp_path, flag):
    """MultiCategoryDetector / MultiCategoryTracker (detector.py) and the graphs' plans (graph.py, both branches) build
    their Engine with the network's flag."""
    from centerpose_b200.graph import _SlotGraph
    from types import SimpleNamespace
    graph_self = SimpleNamespace(device=torch.device("cuda", 0))
    # several categories, detection and tracking: det.engine (run_batch, both MultiCategory graphs)
    for trk in (False, True):
        opt = cpb.default_opt("dla_34", tracking_task=trk, batch_invariant=flag)
        cls = cpb.MultiCategoryTracker if trk else cpb.MultiCategoryDetector
        det = cls(opt, _checkpoints(tmp_path, trk))
        assert det._plan_cfg["batch_invariant"] is flag
        det.engine(2, 512, 512)
        assert _Stub.made[-1]["batch_invariant"] is flag and _Stub.made[-1]["models"] == 2
        if trk:
            det._track_engine(3, torch.empty((3, 3, 512, 512), device="meta"))
            assert _Stub.made[-1]["batch_invariant"] is flag
        _SlotGraph._plan(graph_self, det, 3, 512, 512)
        assert _Stub.made[-1]["batch_invariant"] is flag and _Stub.made[-1]["models"] == 2
    # one category: the network's own plans (run, run_batch, the pipelines) and the graphs' copy of it
    for trk in (False, True):
        opt = cpb.default_opt("dla_34", tracking_task=trk, batch_invariant=flag)
        m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
        _SlotGraph._plan(graph_self, SimpleNamespace(model=m, opt=opt), 4, 512, 512)
        assert _Stub.made[-1]["batch_invariant"] is flag
    assert len(_Stub.made) == 7


@pytest.fixture(scope="module")
def ks_host():
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "host", "ksegments_host.cpp")
    hdr = os.path.join(root, "centerpose_b200", "csrc", "ksegments.h")
    out_dir = os.path.join(root, "tests", "host", "_build")
    so = os.path.join(out_dir, "libksegments_host.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.ks_fixed.argtypes = [ctypes.c_longlong, ctypes.c_int]
    return lib


def _rule(tiles1, slabs):
    """The issue's rule restated: the largest divisor g of slabs with tiles1 * g <= 132 (1 when none is larger)."""
    return max([g for g in range(1, slabs + 1) if slabs % g == 0 and tiles1 * g <= 132] or [1])


def test_the_header_rule(ks_host):
    assert ks_host.ks_sms() == 132
    for tiles1 in list(range(1, 140)) + [200, 1 << 20]:
        for slabs in (1, 2, 3, 4, 7, 8, 10, 16, 24, 32, 36, 64):
            assert ks_host.ks_fixed(tiles1, slabs) == _rule(tiles1, slabs), (tiles1, slabs)
    # a level-5 3x3 conv of dla_34 at 512 x 512: 3 position tiles (16 rows of 18) x 4 N tiles of 128, 16 slabs
    assert ks_host.ks_fixed(3 * 4, 16) == 8
