"""ncu CSV (one row per launch x metric) of scripts/profile_target.py -> profiles/<tag>_perlayer_tf32x3.md (kept out of git)
   python scripts/perlayer_table.py gpurun_out/perlayer_r02.csv r02"""
import collections
import csv
import os
import re
import sys

path, tag = sys.argv[1], sys.argv[2]
rows = [r for r in csv.reader(open(path, errors="ignore")) if len(r) > 10]
hdr = rows[0]
ii, ki, gi, mi, vi, ui = (hdr.index(k) for k in ("ID", "Kernel Name", "Grid Size", "Metric Name", "Metric Value", "Metric Unit"))
L = collections.OrderedDict()
for r in rows[1:]:
    d = L.setdefault(int(r[ii]), {"k": re.sub(r"\(.*", "", r[ki]).replace("void ", "").replace("cp::", "").replace("<unnamed>::", "").replace("unnamed>::", ""),
                                  "g": r[gi]})
    v = float(r[vi].replace(",", ""))
    u = r[ui]
    scale = {"Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "byte": 1.0, "us": 1.0, "ms": 1e3, "ns": 1e-3}.get(u, 1.0)
    d[r[mi]] = v * scale
ids = sorted(L)
ids = ids[len(ids) // 2:]                      # second of two forwards
tot = sum(L[i].get("gpu__time_duration.sum", 0) for i in ids)
os.makedirs("profiles", exist_ok=True)
with open("profiles/%s_perlayer_tf32x3.md" % tag, "w") as f:
    f.write("# Per-launch metrics of one forward, tf32x3 (default) mode, batch 32 @ 512x512 (%s)\n\n" % tag)
    f.write("`ncu --metrics gpu__time_duration.sum,sm__pipe_tensor_cycles_active...,l1tex__m_xbar2l1tex_read_bytes.sum,dram__bytes_read.sum,"
            "dram__bytes_write.sum,lts__throughput...,l1tex__data_pipe_lsu_wavefronts_mem_shared... --clock-control none "
            "-k regex:conv_tma|dcn_tma|igemm_umma|conv3_c16|stem_conv|igemm_fp32|upsample|maxpool python scripts/profile_target.py` "
            "(second of two forwards; launches in schedule order; cold-cache, serialised: %.2f ms in total).\n\n" % (tot / 1e3))
    f.write("| # | kernel | grid | us | tensor pipe active % | LSU shared wavefronts % | L2->SM MB | DRAM read MB | DRAM write MB | lts % |\n|---:|---|---|---:|---:|---:|---:|---:|---:|---:|\n")
    for n, i in enumerate(ids):
        d = L[i]
        f.write("| %d | `%s` | %s | %.1f | %.1f | %.1f | %.0f | %.1f | %.1f | %.1f |\n" % (
            n, d["k"], d["g"], d.get("gpu__time_duration.sum", 0),
            d.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 0),
            d.get("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", 0),
            d.get("l1tex__m_xbar2l1tex_read_bytes.sum", 0) / 1e6, d.get("dram__bytes_read.sum", 0) / 1e6,
            d.get("dram__bytes_write.sum", 0) / 1e6, d.get("lts__throughput.avg.pct_of_peak_sustained_elapsed", 0)))
print("wrote profiles/%s_perlayer_tf32x3.md (%d launches, %.2f ms)" % (tag, len(ids), tot / 1e3))
