"""C-ABI checks that need no GPU: the library builds, loads and exports every
symbol include/centerpose_b200.h declares; argument validation returns error
codes (never throws); the Python product path fails loudly without CUDA."""
import ctypes
import os
import re

import pytest
import torch

from tests.util import ROOT


def _declared_symbols():
    txt = open(os.path.join(ROOT, "include", "centerpose_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(cp_[a-z0-9_]+)\s*\(", txt)))


def test_header_symbols_exported(cplib):
    syms = _declared_symbols()
    assert "cp_forward" in syms and "cp_decode_pnp" in syms and len(syms) >= 12
    for s in syms:
        assert hasattr(cplib, s), "libcenterpose_b200.so does not export %s" % s


def test_exports_match_python_binding(cplib):
    from centerpose_b200 import _lib
    assert sorted(_lib.EXPORTS) == _declared_symbols()


def test_version_and_error_string(cplib):
    from centerpose_b200 import _lib
    assert cplib.cp_version() == 1
    rc = cplib.cp_plan_create(None, None)
    assert rc == -1
    assert b"null" in cplib.cp_last_error()
    with pytest.raises(RuntimeError):
        _lib.check(rc, "cp_plan_create")


def test_decode_param_validation(cplib):
    from centerpose_b200 import _lib
    from centerpose_b200.engine import decode_params
    p = decode_params(None)
    p.batch, p.out_h, p.out_w = 2, 128, 128
    assert cplib.cp_decode_workspace_bytes(ctypes.byref(p)) > 2 * 100 * 128 * 4
    p.rep_mode = 2            # random GMM sampling: unsupported, reported not silently ignored
    assert cplib.cp_decode_workspace_bytes(ctypes.byref(p)) == 0
    assert b"rep_mode" in cplib.cp_last_error()
    p.rep_mode = 1
    p.K = 200
    assert cplib.cp_decode_workspace_bytes(ctypes.byref(p)) == 0
    p.K = 100
    p.num_classes = 3         # multi-class heat maps: K candidates per class
    assert cplib.cp_decode_workspace_bytes(ctypes.byref(p)) > 2 * 3 * 100 * 4
    p.num_classes = 81        # > CP_MAX_CLASSES
    assert cplib.cp_decode_workspace_bytes(ctypes.byref(p)) == 0
    p.num_classes = 1
    p.test_scale = -1.0
    assert cplib.cp_decode_workspace_bytes(ctypes.byref(p)) == 0
    assert b"test_scale" in cplib.cp_last_error()


def test_struct_sizes_match_header():
    from centerpose_b200 import _lib
    assert ctypes.sizeof(_lib.CpDecodeParams) == 18 * 4
    assert ctypes.sizeof(_lib.CpHeads) == 11 * ctypes.sizeof(ctypes.c_void_p)
    assert ctypes.sizeof(_lib.CpConfig) == 10 * 4 + 16 * ctypes.sizeof(ctypes.c_void_p) + 16 * 4


def test_no_cpu_fallback():
    import centerpose_b200 as cpb
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 64, 64))
    with pytest.raises(RuntimeError, match="CUDA"):
        cpb.decode_pnp({"hm": torch.zeros(1, 1, 32, 32)}, torch.zeros(1, 16, dtype=torch.float64), cpb.decode_params())
    with pytest.raises(RuntimeError):
        cpb.dcn_v2_forward(torch.zeros(1, 16, 4, 4), torch.zeros(8, 16, 3, 3), torch.zeros(8),
                           torch.zeros(1, 18, 4, 4), torch.zeros(1, 9, 4, 4))
    with pytest.raises(RuntimeError):
        cpb.dcn_v2_backward(torch.zeros(1, 16, 4, 4), torch.zeros(8, 16, 3, 3), torch.zeros(8),
                            torch.zeros(1, 18, 4, 4), torch.zeros(1, 9, 4, 4), torch.zeros(1, 8, 4, 4))


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "centerpose_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "import oracle" not in src and "from oracle" not in src, fn


def test_plan_stepping_argument_validation(cplib):
    """The diagnostic stepping calls reject null plans / outputs with an error code, like cp_forward."""
    from centerpose_b200 import _lib
    d = _lib.CpOpDesc()
    assert cplib.cp_plan_op_desc(None, 0, ctypes.byref(d)) == -1
    assert b"null" in cplib.cp_last_error()
    p, n = ctypes.c_void_p(), ctypes.c_int64()
    assert cplib.cp_plan_arena(None, ctypes.byref(p), ctypes.byref(n)) == -1
    assert cplib.cp_plan_run_ops(None, 1, 0, 1, None, None, None, None, None, None, None) == -1
    assert b"null" in cplib.cp_last_error()
