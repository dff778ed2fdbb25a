"""Build libcenterpose_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m centerpose_b200.build [--force]

The shared library lands next to this file so that it travels to the GPU box
with the repository; nothing is JIT-compiled at run time.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcenterpose_b200.so")
SOURCES = ["plan.cu", "igemm_fp32.cu", "elementwise.cu", "decode.cu", "ext_ops.cu", "conv_select.cu", "igemm_umma.cu", "stem_conv.cu", "conv_tma.cu", "dcn_tma.cu", "tracker.cu", "dcn_bwd.cu"]
def _headers():
    """Every header a .cu may include: editing shared code (umma_common.cuh, pose_core.h ...) must rebuild the objects."""
    hs = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    return hs + [os.path.join("..", "..", "include", "centerpose_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    """Compile every .cu to an object (parallelisable, incremental) and link the .so."""
    objdir = os.path.join(CSRC, "build")
    os.makedirs(objdir, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in _headers()]
    objs = []
    procs = []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [sp] + hdrs):
            cmd = [_nvcc()] + NVCC_FLAGS + ["-c", sp, "-o", obj]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    logs = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        logs.append("==== %s\n%s" % (src, out))
        if p.returncode != 0:
            failed = True
    log_path = os.path.join(objdir, "nvcc.log")
    if procs:
        with open(log_path, "w") as f:
            f.write("\n".join(logs))
    if failed:
        sys.stderr.write("\n".join(logs))
        raise RuntimeError("nvcc failed; see %s" % log_path)
    if verbose and logs:
        print("\n".join(logs))
    if force or procs or _stale(LIB, objs):
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
