#!/bin/bash
# A/B a bring-up switch with alternating runs on the SAME box (box-to-box variation is +-3 %, larger than most effects).
# Usage:  bash tests/gpu_scripts/ab.sh "LSPG_NO_PDL=1" [batch] [mode] [rounds]
# Prints the ms/forward of every run and the medians.
mkdir -p gpurun_out
VAR="$1"; B=${2:-32}; MODE=${3:-parity}; N=${4:-3}
T="timeout 300 python tests/gpu_bringup.py time large A $MODE 512 $B"
: > gpurun_out/ab.log
for i in $(seq 1 $N); do
  echo "## base"    >> gpurun_out/ab.log; $T >> gpurun_out/ab.log 2>&1
  echo "## variant" >> gpurun_out/ab.log; env $VAR $T >> gpurun_out/ab.log 2>&1
done
python - <<'PY'
import re, statistics
cur, d = None, {"base": [], "variant": []}
for line in open("gpurun_out/ab.log"):
    if line.startswith("## "): cur = line[3:].strip()
    m = re.search(r"([\d.]+) ms/forward", line)
    if m and cur: d[cur].append(float(m.group(1)))
for k, v in d.items():
    print(k, v, "median", statistics.median(v) if v else None)
if d["base"] and d["variant"]:
    print("variant / base = %.4f" % (statistics.median(d["variant"]) / statistics.median(d["base"])))
PY
