"""Every pre-process entry point of two builds of the library, compared bit for bit (SHA-256 of `out`, and of `prev` /
`store` where written) and timed with CUDA events.

    python scripts/preprocess_ab.py LIB_A LIB_B OUT_DIR [--rounds N]   # digests, then timings A B A B ... (CP_LIB_PATH)
    python scripts/preprocess_ab.py --dump OUT.json                    # the digests of the library CP_LIB_PATH names
    python scripts/preprocess_ab.py --time OUT.json                    # its per-call times in microseconds

The bit cases run every entry point in every format it accepts: uniform batches of 32 1080p frames to 512 x 512 (and
481 x 640 for the formats that allow an odd height), ragged batches of mixed sizes with odd heights at unaligned byte
offsets, a rotated anisotropic trans_input, a per-frame batch of all eight formats, slot launches with mixed start
flags, and the rows form at 5 of 8 live slots over 3 steps with the store exchange.  The times are at user sizes:
cp_preprocess at 32 x 512 x 512 (bench.py's pre-process breakdown), the host-table calls at 32 x 1080p and the
graph-safe forms at 8 slots of 1280 x 720.  B is accepted when no entry point's median is slower than A's by more than
the spread of A's own rounds.
"""
import ctypes
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MEAN, STD = (0.408, 0.447, 0.470), (0.289, 0.274, 0.278)
ODD_OK = ("bgr", "rgb24", "rgba", "bgra", "yuyv422", "uyvy422")     # the formats whose frames may have an odd height
# a rotated (0.3 rad), anisotropic forward affine around a 1080p frame's centre into 512 x 512
_c, _s = np.cos(0.3), np.sin(0.3)
ROT = np.array([[0.31 * _c, -0.27 * _s, 256 - 0.31 * _c * 960 + 0.27 * _s * 540],
                [0.31 * _s, 0.27 * _c, 256 - 0.31 * _s * 960 - 0.27 * _c * 540]], np.float64)


def _env():
    import torch
    from centerpose_b200 import _lib as L
    return torch, L, L.load()


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _ptr(a, ct):
    return None if a is None else a.ctypes.data_as(ctypes.POINTER(ct))


def _nbytes(fmt, h, w):
    return h * w * {"bgr": 3, "rgb24": 3, "rgba": 4, "bgra": 4, "yuyv422": 2, "uyvy422": 2}.get(fmt, 1.5)


def _packed(torch, sizes, fmts, seed, gaps=None):
    """Random bytes holding frame b (sizes[b], fmts[b]) at offs[b], gaps[b] bytes after the previous frame."""
    offs, off = [], 0
    for b, ((h, w), f) in enumerate(zip(sizes, fmts)):
        off += gaps[b] if gaps else 0
        offs.append(off)
        off += int(_nbytes(f, h, w))
    buf = np.random.default_rng(seed).integers(0, 256, off, dtype=np.uint8)
    return torch.from_numpy(buf).cuda(), np.array(offs, np.int64), np.array(sizes, np.int32)


class Lib:
    """The entry points of one build, called as the package's wrappers do, on the current stream."""

    def __init__(self):
        self.torch, self.L, self.c = _env()
        self.m = (ctypes.c_float * 3)(*MEAN)
        self.s = (ctypes.c_float * 3)(*STD)

    def st(self):
        return ctypes.c_void_p(self.torch.cuda.current_stream().cuda_stream)

    def out(self, B, dh, dw, fill=float("nan")):
        return self.torch.full((B, 3, dh, dw), fill, dtype=self.torch.float32, device="cuda")

    def uniform(self, frames, B, sh, sw, out, trans=None):
        if trans is None:
            rc = self.c.cp_preprocess(_p(frames), _p(out), B, sh, sw, out.shape[2], out.shape[3], self.m, self.s, self.st())
        else:
            tm = (ctypes.c_double * 6)(*trans.reshape(-1))
            rc = self.c.cp_preprocess_affine(_p(frames), _p(out), B, sh, sw, out.shape[2], out.shape[3], tm, self.m,
                                             self.s, self.st())
        self.L.check(rc, "cp_preprocess")

    def ragged(self, entry, packed, offs, hw, fmts, out, trans=None):
        """cp_preprocess_ragged / _yuv420 / _formats over a host table."""
        B = len(offs)
        tr = None if trans is None else np.ascontiguousarray(trans, np.float64)
        args = [_p(packed), packed.numel(), _ptr(offs, ctypes.c_int64), _ptr(hw, ctypes.c_int32)]
        codes = np.array([self.L.PIXEL_FORMAT_CODES[f] for f in fmts], np.int32)
        if entry == "cp_preprocess_yuv420":
            args.append(int(codes[0]))
        elif entry == "cp_preprocess_formats":
            args.append(_ptr(codes, ctypes.c_int32))
        args += [_p(out), B, out.shape[2], out.shape[3], _ptr(tr, ctypes.c_double), self.m, self.s, self.st()]
        self.L.check(getattr(self.c, entry)(*args), entry)

    def table(self, packed, offs, hw, fmts, dh, dw, trans=None):
        """A device frame table of one format or of per-frame formats -> (table, launch format)."""
        B = len(offs)
        table = self.torch.zeros(int(self.c.cp_preprocess_frame_table_bytes(B)), dtype=self.torch.uint8, device="cuda")
        tr = None if trans is None else np.ascontiguousarray(trans, np.float64)
        args = (packed.numel(), _ptr(offs, ctypes.c_int64), _ptr(hw, ctypes.c_int32))
        codes = np.array([self.L.PIXEL_FORMAT_CODES[f] for f in fmts], np.int32)
        if len(set(fmts)) == 1:
            self.L.check(self.c.cp_preprocess_frame_table(*args, int(codes[0]), B, dh, dw, _ptr(tr, ctypes.c_double),
                                                          _p(table), self.st()), "cp_preprocess_frame_table")
            return table, int(codes[0])
        self.L.check(self.c.cp_preprocess_frame_table_formats(*args, _ptr(codes, ctypes.c_int32), B, dh, dw,
                                                              _ptr(tr, ctypes.c_double), _p(table), self.st()),
                     "cp_preprocess_frame_table_formats")
        return table, self.L.CP_PIX_PER_FRAME

    def slots(self, frames, fmt, B, sh, sw, out, start=None, prev=None, trans=None):
        tm = None if trans is None else (ctypes.c_double * 6)(*trans.reshape(-1))
        self.L.check(self.c.cp_preprocess_slots_dev(_p(frames), self.L.PIXEL_FORMAT_CODES[fmt], B, sh, sw, out.shape[2],
                                                    out.shape[3], tm, self.m, self.s, _p(start), _p(out), _p(prev),
                                                    self.st()), "cp_preprocess_slots_dev")

    def slots_ragged(self, packed, table, code, out, start=None, prev=None):
        self.L.check(self.c.cp_preprocess_slots_ragged_dev(_p(packed), _p(table), code, out.shape[0], out.shape[2],
                                                           out.shape[3], self.m, self.s, _p(start), _p(out), _p(prev),
                                                           self.st()), "cp_preprocess_slots_ragged_dev")

    def slots_rows(self, packed, table, code, rows, out, start=None, store=None, prev=None):
        self.L.check(self.c.cp_preprocess_slots_rows_dev(_p(packed), _p(table), code, _p(rows), out.shape[0],
                                                         out.shape[2], out.shape[3], self.m, self.s, _p(start),
                                                         _p(store), _p(out), _p(prev), self.st()),
                     "cp_preprocess_slots_rows_dev")


def _digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def dump(path):
    lib = Lib()
    torch, L = lib.torch, lib.L
    fmts_all = list(L.PIXEL_FORMATS)
    out = {}

    def put(name, **tensors):
        torch.cuda.synchronize()
        for k, t in tensors.items():
            out["%s/%s" % (name, k)] = _digest(t)

    def i32(v):
        return torch.tensor(v, dtype=torch.int32, device="cuda")

    # uniform batches: cp_preprocess(_affine) (BGR) and cp_preprocess_slots_dev (every format, with and without start
    # flags), 32 x 1080p -> 512 x 512 and 481 x 640 where an odd height is allowed
    start32 = i32([(b * 7) % 3 == 0 for b in range(32)])
    for sh, sw in ((1080, 1920), (481, 640)):
        for fmt in fmts_all:
            if sh % 2 and fmt not in ODD_OK:
                continue
            frames, _, _ = _packed(torch, [(sh, sw)] * 32, [fmt] * 32, seed=sh + len(fmt))
            for tname, trans in (("fixres", None), ("rot", ROT)):
                tag = "%dx%d %s %s" % (sh, sw, fmt, tname)
                if fmt == "bgr":
                    o = lib.out(32, 512, 512)
                    lib.uniform(frames, 32, sh, sw, o, trans)
                    put("cp_preprocess " + tag, out=o)
                o = lib.out(32, 512, 512)
                lib.slots(frames, fmt, 32, sh, sw, o, trans=trans)
                put("slots_dev " + tag, out=o)
                o, prev = lib.out(32, 512, 512), lib.out(32, 512, 512, 7.0)
                lib.slots(frames, fmt, 32, sh, sw, o, start32, prev, trans=trans)
                put("slots_dev twin " + tag, out=o, prev=prev)
                del o, prev
            # the host-table calls on the uniform batch
            offs = np.arange(32, dtype=np.int64) * int(_nbytes(fmt, sh, sw))
            hw = np.array([(sh, sw)] * 32, np.int32)
            for entry in _ragged_entries(fmt):
                o = lib.out(32, 512, 512)
                lib.ragged(entry, frames, offs, hw, [fmt] * 32, o)
                put("%s uniform %dx%d %s" % (entry, sh, sw, fmt), out=o)
            del frames

    # ragged batches: mixed sizes with odd heights (even ones for 4:2:0) at unaligned offsets, default and rotated
    # affines, through the host-table calls and device tables (slots-ragged with start flags, rows with the exchange)
    odd = [(481, 640), (1081, 1920), (37, 62), (720, 1280), (301, 200), (1080, 1920), (599, 800), (2, 2)]
    even = [(480, 640), (1080, 1920), (36, 62), (720, 1280), (300, 200), (1080, 1920), (600, 800), (2, 2)]
    gaps = [3, 1, 2, 5, 7, 1, 3, 6]
    rot8 = np.stack([ROT] * 8)
    for fmt in fmts_all + ["mixed"]:
        fmts = fmts_all if fmt == "mixed" else [fmt] * 8
        sizes = even if fmt in ("nv12", "i420", "mixed") else odd
        packed, offs, hw = _packed(torch, sizes, fmts, seed=100 + len(fmt), gaps=gaps)
        for tname, trans in (("fixres", None), ("rot", rot8)):
            tag = "%s %s" % (fmt, tname)
            for entry in _ragged_entries(fmt):
                o = lib.out(8, 512, 384)
                lib.ragged(entry, packed, offs, hw, fmts, o, trans)
                put("%s ragged %s" % (entry, tag), out=o)
            table, code = lib.table(packed, offs, hw, fmts, 512, 384, trans)
            o = lib.out(8, 512, 384)
            lib.slots_ragged(packed, table, code, o)
            put("slots_ragged_dev " + tag, out=o)
            o, prev = lib.out(8, 512, 384), lib.out(8, 512, 384, 7.0)
            lib.slots_ragged(packed, table, code, o, i32([1, 0, 1, 1, 0, 0, 1, 0]), prev)
            put("slots_ragged_dev twin " + tag, out=o, prev=prev)
            # rows: 5 of 8 live slots over 3 steps, the store carried from step to step
            store = torch.randn((8, 3, 512, 384), generator=torch.Generator(device="cuda").manual_seed(3), device="cuda")
            steps = [([7, 0, 3, 5, 2], [1, 1, 1, 1, 1, 1, 1, 1]), ([1, 3, 5, 7, 6], [0, 1, 0, 0, 0, 0, 1, 0]),
                     ([0, 2, 4, 6, 1], [0, 0, 0, 1, 1, 0, 0, 0])]
            for k, (rows, start) in enumerate(steps):
                o, prev = lib.out(5, 512, 384), lib.out(5, 512, 384)
                lib.slots_rows(packed, table, code, i32(rows), o, i32(start), store, prev)
                put("slots_rows_dev exchange %s step %d" % (tag, k), out=o, prev=prev, store=store)
            o = lib.out(5, 512, 384)
            lib.slots_rows(packed, table, code, i32(steps[0][0]), o, i32(steps[0][1]))
            put("slots_rows_dev " + tag, out=o)
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)


def _ragged_entries(fmt):
    """The host-table entry points that accept frames of fmt ("mixed": per-frame formats)."""
    return (["cp_preprocess_ragged"] if fmt == "bgr" else ["cp_preprocess_yuv420"] if fmt in ("nv12", "i420") else []) + \
        ["cp_preprocess_formats"]


def timings(path, calls=200, warmup=20):
    lib = Lib()
    torch, L = lib.torch, lib.L
    res = {}

    def time_it(name, fn):
        for _ in range(warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res[name] = e0.elapsed_time(e1) * 1e3 / calls

    frames, _, _ = _packed(torch, [(512, 512)] * 32, ["bgr"] * 32, seed=1)
    o = lib.out(32, 512, 512)
    time_it("cp_preprocess 32x512x512", lambda: lib.uniform(frames, 32, 512, 512, o))
    for fmt in list(L.PIXEL_FORMATS) + ["mixed"]:
        fmts = list(L.PIXEL_FORMATS) * 4 if fmt == "mixed" else [fmt] * 32
        packed, offs, hw = _packed(torch, [(1080, 1920)] * 32, fmts, seed=2)
        for entry in _ragged_entries(fmt):
            time_it("%s 32x1080p %s" % (entry, fmt), lambda: lib.ragged(entry, packed, offs, hw, fmts, o))
        fm8 = fmts[:8]
        packed, offs, hw = _packed(torch, [(720, 1280)] * 8, fm8, seed=3)
        o8, prev, store = lib.out(8, 512, 512), lib.out(8, 512, 512), lib.out(8, 512, 512, 0.0)
        start = torch.tensor([1, 0, 0, 1, 0, 0, 0, 0], dtype=torch.int32, device="cuda")
        rows = torch.arange(8, dtype=torch.int32, device="cuda")
        if fmt != "mixed":
            time_it("slots_dev 8x720p %s" % fmt, lambda: lib.slots(packed, fmt, 8, 720, 1280, o8, start, prev))
        table, code = lib.table(packed, offs, hw, fm8, 512, 512)
        time_it("slots_ragged_dev 8x720p %s" % fmt, lambda: lib.slots_ragged(packed, table, code, o8, start, prev))
        time_it("slots_rows_dev 8x720p %s" % fmt,
                lambda: lib.slots_rows(packed, table, code, rows, o8, start, store, prev))
        del packed
    with open(path, "w") as f:
        json.dump(res, f, indent=0, sort_keys=True)


def compare(a, b):
    A, B = json.load(open(a)), json.load(open(b))
    assert sorted(A) == sorted(B), (sorted(set(A) ^ set(B)))
    bad = [k for k in A if A[k] != B[k]]
    for k in sorted(bad):
        print("DIFFER %s" % k)
    print("%d of %d digests equal" % (len(A) - len(bad), len(A)))
    return not bad


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except OSError as e:
        return "nvidia-smi: %s" % e


if __name__ == "__main__":
    if sys.argv[1] in ("--dump", "--time"):
        (dump if sys.argv[1] == "--dump" else timings)(sys.argv[2])
        sys.exit(0)
    lib_a, lib_b, out_dir = sys.argv[1:4]
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 4
    os.makedirs(out_dir, exist_ok=True)
    libs = (("a", lib_a), ("b", lib_b))

    def run(mode, tag, lib, suffix=""):
        p = os.path.join(out_dir, "%s_%s%s.json" % (mode, tag, suffix))
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--" + mode, p],
                              env=dict(os.environ, CP_LIB_PATH=os.path.abspath(lib)))
        return json.load(open(p))

    print("card: %s" % _card(), flush=True)
    for tag, lib in libs:
        run("dump", tag, lib)
    same = compare(os.path.join(out_dir, "dump_a.json"), os.path.join(out_dir, "dump_b.json"))
    times = {"a": [], "b": []}
    for r in range(rounds):
        for tag, lib in libs:
            times[tag].append(run("time", tag, lib, "_%d" % r))
    slower = []
    print("%-44s %10s %10s %10s %8s" % ("entry point (us per call)", "median A", "median B", "A spread", "B - A"))
    for k in sorted(times["a"][0]):
        a = [t[k] for t in times["a"]]
        b = [t[k] for t in times["b"]]
        ma, mb, spread = float(np.median(a)), float(np.median(b)), max(a) - min(a)
        if mb - ma > spread:
            slower.append(k)
        print("%-44s %10.1f %10.1f %10.1f %+8.1f%s" % (k, ma, mb, spread, mb - ma, "  SLOWER" if k in slower else ""))
    print("card: %s" % _card())
    print("digests %s; %d of %d entry points slower than the A-vs-A spread"
          % ("all equal" if same else "DIFFER", len(slower), len(times["a"][0])))
    sys.exit(0 if same and not slower else 1)
