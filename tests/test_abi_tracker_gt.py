"""C-ABI checks of the tracker's seeding and render-mode entry points that need no GPU: declared, exported, bound, and
argument validation that returns CP_ERR_INVALID with a message before any device work."""
import ctypes

from centerpose_b200 import _lib
from tests.test_abi import _declared_symbols


def test_new_symbols_declared_exported_and_bound(cplib):
    for s in ("cp_tracker_seed", "cp_tracker_render_ex"):
        assert s in _declared_symbols() and s in _lib.EXPORTS and hasattr(cplib, s)
    assert cplib.cp_version() == 1
    names = [f[0] for f in _lib.CpTrackerConfig._fields_]
    assert names[-1] == "hungarian" and ctypes.sizeof(_lib.CpTrackerConfig) == 18 * 4


def test_seed_rejects_too_many_seeds_per_stream(cplib):
    n = (ctypes.c_int32 * 1)(1)
    rc = cplib.cp_tracker_seed(None, 1, None, ctypes.cast(n, ctypes.c_void_p), _lib.CP_MAX_K + 1, None)
    assert rc == -1 and b"S must be in 0..128" in cplib.cp_last_error()


def test_render_rejects_unknown_mode(cplib):
    modes = (ctypes.c_int32 * 2)(0, 3)
    rc = cplib.cp_tracker_render_ex(None, 2, None, None, 8, 8, modes, None, None, None)
    assert rc == -1 and b"unknown render mode 3" in cplib.cp_last_error()
