"""CPU test of centerpose_b200/csrc/arena_pack.h (the liveness packer of the plan's activation arena, compiled for the
host) on seeded random lifetime sets and on the lifetimes of the real schedules (cp_plan_allocations): allocations live
at the same op never overlap in memory, offsets keep the 64-float alignment, the arena is never smaller than the largest
live sum, and the layout is deterministic and the one the library uses."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests.test_plan_memory_cpu import ARCHS, REUSE, MULTI_TRACK, allocations, memory, net_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pack_host():
    src = os.path.join(ROOT, "tests", "host", "arena_pack_host.cpp")
    hdr = os.path.join(ROOT, "centerpose_b200", "csrc", "arena_pack.h")
    out_dir = os.path.join(ROOT, "tests", "host", "_build")
    so = os.path.join(out_dir, "libarena_pack_host.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, src])
    lib = ctypes.CDLL(so)
    lib.ap_align.restype = ctypes.c_int64
    lib.ap_pack.restype = ctypes.c_int64
    lib.ap_live_peak.restype = ctypes.c_int64
    return lib


def _arr(a, t):
    return np.ascontiguousarray(a, t)


def pack(lib, floats, first, last):
    f, a, b = _arr(floats, np.int64), _arr(first, np.int32), _arr(last, np.int32)
    off = np.zeros(len(f), np.int64)
    P = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    arena = lib.ap_pack(len(f), P(f), P(a), P(b), P(off))
    peak = lib.ap_live_peak(len(f), P(f), P(a), P(b))
    return off, arena, peak


def check_layout(floats, first, last, off, arena, peak, align):
    floats, first, last, off = map(np.asarray, (floats, first, last, off))
    used = (first >= 0) & (floats > 0)
    assert (off % align == 0).all()
    assert (off[used] + floats[used] <= arena).all()
    assert arena >= peak
    if used.any():
        assert arena == (off[used] + floats[used]).max()
    idx = np.nonzero(used)[0]
    for k, i in enumerate(idx):
        j = idx[k + 1:]
        live = (first[j] <= last[i]) & (first[i] <= last[j])
        apart = (off[i] + floats[i] <= off[j]) | (off[j] + floats[j] <= off[i])
        assert (apart | ~live).all(), (i, j[live & ~apart])


@pytest.mark.parametrize("seed", range(40))
def test_random_lifetimes(pack_host, seed):
    rng = np.random.default_rng(seed)
    align = pack_host.ap_align()
    n = int(rng.integers(1, 120))
    ops = int(rng.integers(1, 90))
    floats = rng.integers(1, 2000, n) * align
    if seed % 4 == 0:
        floats = rng.choice([align, 4 * align, 16 * align], n)       # many equal sizes: the tie-break decides
    first = rng.integers(0, ops, n)
    last = np.minimum(first + rng.geometric(0.15, n) - 1, ops)
    dead = rng.random(n) < 0.05                                     # never touched: no memory
    first[dead], last[dead] = -1, -1
    off, arena, peak = pack(pack_host, floats, first, last)
    check_layout(floats, first, last, off, arena, peak, align)
    assert (off[dead] == 0).all()
    again = pack(pack_host, floats, first, last)
    assert (again[0] == off).all() and again[1] == arena


def test_disjoint_lifetimes_share_one_region(pack_host):
    a = pack_host.ap_align()
    off, arena, peak = pack(pack_host, [4 * a, 2 * a, 3 * a], [0, 2, 4], [1, 3, 5])
    assert list(off) == [0, 0, 0] and arena == 4 * a == peak


def test_chain_of_two_live_tensors(pack_host):
    """Each op reads one tensor and writes the next: two regions alternate, the peak is two tensors."""
    a = pack_host.ap_align()
    n = 10
    off, arena, peak = pack(pack_host, [8 * a] * n, list(range(n)), [i + 1 for i in range(n)])
    assert arena == peak == 16 * a
    assert all(off[i] != off[i + 1] for i in range(n - 1))


@pytest.mark.parametrize("arch,trk", ARCHS)
@pytest.mark.parametrize("B,M,prec", [(1, 1, "tf32x3"), (8, 1, "fp32"), (2, 3, "bf16")])
def test_real_schedules(cplib, pack_host, arch, trk, B, M, prec):
    """The lifetimes of the real schedules, packed on the host, give the library's own layout."""
    cfg = net_config(arch, trk, B, 512, 512, prec)
    flags = REUSE | (MULTI_TRACK if trk and M > 1 else 0)
    al = allocations(cfg, M, flags)
    full = allocations(cfg, M, flags & ~REUSE)             # the sizes of allocations without memory
    floats = [f["floats"] for f in full]
    first = [a["first"] for a in al]
    last = [a["last"] for a in al]
    off, arena, peak = pack(pack_host, floats, first, last)
    check_layout(floats, first, last, off, arena, peak, pack_host.ap_align())
    assert arena * 4 == memory(cfg, M, flags).activation_bytes
    for a, o in zip(al, off):
        assert a["off"] == (o if a["first"] >= 0 else -1)
    print("%s%s b%d M%d %s: arena %.1f MiB, live peak %.1f MiB, full %.1f MiB" % (
        arch, "+trk" if trk else "", B, M, prec, arena * 4 / 2**20, peak * 4 / 2**20, sum(floats) * 4 / 2**20))
