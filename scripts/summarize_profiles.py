"""Turn raw profiler artefacts (ncu launch lists and reports) into small summaries under profiles/ (kept out of git).

    python scripts/summarize_profiles.py <tag>      e.g. r01_fp32

  gpurun_out/launches_<x>.csv  (ncu --metrics gpu__time_duration.sum)  -> profiles/<tag>_launches.md
  gpurun_out/<x>.ncu-rep       (ncu --set full)                        -> profiles/<tag>_<x>_ncu.md
"""
import collections
import csv
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "profiles")
GP = os.path.join(ROOT, "gpurun_out")

KEYS = [
    "Kernel Name", "Grid Size", "Block Size", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers",
    "launch__occupancy_limit_shared_mem", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
    "smsp__inst_executed.sum", "sm__cycles_elapsed.max", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "l1tex__m_xbar2l1tex_read_bytes.sum", "l1tex__m_xbar2l1tex_read_bytes.sum.per_second",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "smsp__sass_inst_executed_op_shared_ld.sum", "smsp__sass_inst_executed_op_shared_st.sum",
]


def launches(path, tag, title):
    rows = [r for r in csv.reader(open(path, errors="ignore")) if len(r) > 10]
    hdr = rows[0]
    ki, vi, gi = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Grid Size")
    agg = collections.OrderedDict()
    for r in rows[1:]:
        name = re.sub(r"\(.*", "", r[ki]).replace("void ", "").replace("unnamed>::", "")
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += float(r[vi].replace(",", ""))
    tot = sum(v[1] for v in agg.values())
    with open(os.path.join(OUT, tag + "_launches.md"), "w") as f:
        f.write("# %s\n\n`ncu --metrics gpu__time_duration.sum --clock-control none` launch list of `bench.py` "
                "(cold-cache, serialised: compare SHARES, not absolutes).  %d launches, %.2f ms total.\n\n" %
                (title, len(rows) - 1, tot / 1e6))
        f.write("| kernel | launches | total ms | share |\n|---|---:|---:|---:|\n")
        for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write("| `%s` | %d | %.3f | %.1f %% |\n" % (k, v[0], v[1] / 1e6, 100 * v[1] / tot))
    print("wrote", tag + "_launches.md")


def full(rep, tag, title, note=""):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units, vals = rows[0], rows[1], rows[2]
    d = {h: (v, u) for h, u, v in zip(hdr, units, vals)}
    name = os.path.splitext(os.path.basename(rep))[0]
    with open(os.path.join(OUT, "%s_%s_ncu.md" % (tag, name)), "w") as f:
        f.write("# %s\n\n`ncu --set full --clock-control none --import-source on` (one launch; report not committed, "
                "%d metrics).  %s\n\n| metric | value | unit |\n|---|---:|---|\n" % (title, len(hdr), note))
        for k in KEYS:
            if k in d:
                f.write("| %s | %s | %s |\n" % (k, d[k][0], d[k][1]))
        try:
            sc = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
            rd = float(d["dram__bytes_read.sum"][0].replace(",", "")) * sc[d["dram__bytes_read.sum"][1]]
            wr = float(d["dram__bytes_write.sum"][0].replace(",", "")) * sc[d["dram__bytes_write.sum"][1]]
            f.write("\nDRAM traffic (read + write) = %.4f GB per launch.\n" % ((rd + wr) / 1e9))
        except Exception:
            pass
    print("wrote", "%s_%s_ncu.md" % (tag, name))
    try:
        return d["Kernel Name"][0], rd + wr, "byte"
    except Exception:
        return None


if __name__ == "__main__":
    # usage: summarize_profiles.py <tag> [file ...]   (files relative to gpurun_out/; default: everything there)
    tag = sys.argv[1]
    os.makedirs(OUT, exist_ok=True)
    files = sys.argv[2:] or sorted(os.listdir(GP))
    traffic = {}
    for fn in files:
        if fn.startswith("launches") and fn.endswith(".csv"):
            launches(os.path.join(GP, fn), tag + "_" + fn[:-4].replace("launches_", "").replace("launches", "bench"),
                     "Launch list, " + fn)
        if fn.endswith(".ncu-rep"):
            r = full(os.path.join(GP, fn), tag, "ncu full capture: " + fn)
            if r:
                scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(r[2], 1.0)
                traffic[fn[:-8]] = {"kernel": r[0], "dram_bytes_per_launch": r[1] * scale}
    if traffic:
        import json
        json.dump(traffic, open(os.path.join(OUT, tag + "_ncu_traffic.json"), "w"), indent=1)
