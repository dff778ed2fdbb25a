#!/bin/bash
# One run that produces the raw records scripts/summarize_profiles.py turns into profiles/ (kept out of git):
#   bash scripts/final_capture.sh <tag>
TAG=${1:-r02}
mkdir -p gpurun_out
python -m pytest tests -m gpu -q 2>&1 | grep -v Warning | tail -3 | tee gpurun_out/${TAG}_gputests.log
python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -1 | tee gpurun_out/${TAG}_smoke.log
python bench.py --steps 20 --warmup 3 > gpurun_out/${TAG}_bench_1gpu.json 2> gpurun_out/${TAG}_bench_1gpu.err
tail -1 gpurun_out/${TAG}_bench_1gpu.err
python bench.py --impl reference --steps 3 --warmup 1 > gpurun_out/${TAG}_bench_reference_arm.json 2> /dev/null
ncu --metrics gpu__time_duration.sum --clock-control none -c 6000 --csv --log-file gpurun_out/launches_${TAG}.csv \
    python bench.py --steps 2 --warmup 3 --no-extra-configs --no-fast-mode --no-cpu-baseline > gpurun_out/${TAG}_ncu_bench.log 2>&1
bash scripts/ncu_longest.sh tf32x3 conv_tma ${TAG}_heads_tf32x3
bash scripts/ncu_longest.sh tf32x3 dcn_tma ${TAG}_dcn_tf32x3
ls -la gpurun_out/*.ncu-rep | tail -4
python - <<PY
import json
d = json.load(open("gpurun_out/${TAG}_bench_1gpu.json"))
for k in ("value", "ms_per_step", "e2e", "gpu_launches", "config1", "config2", "config5", "fast_mode", "stage_ms",
          "decode_us_per_frame", "cpu_baseline", "clocks", "roofline"):
    print(k, d.get(k))
r = json.load(open("gpurun_out/${TAG}_bench_reference_arm.json"))
print("REF", r.get("value"), r.get("cpu_baseline"))
PY
