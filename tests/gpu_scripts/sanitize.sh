#!/bin/bash
# compute-sanitizer over one forward per kernel family (SURVEY.md section 5: race / sync / memory checks of the hand-rolled
# mbarrier + wgmma pipelines).  `normal`, 256x256, batch 2 reaches conv_patch_kernel (head, tail, the wide layers, the
# 2-CTA multicast cluster), conv_umma_kernel + splitk_reduce_kernel and the input packer; plain stream launches
# (LSPG_NO_GRAPH) so that every launch is attributed.
# Usage: bash tests/gpu_scripts/sanitize.sh [per-tool timeout seconds] [log directory]
T=${1:-300}
OUT=${2:-$(mktemp -d)}
mkdir -p "$OUT"
CS=$(command -v compute-sanitizer || echo /usr/local/cuda/bin/compute-sanitizer)
for tool in memcheck synccheck racecheck; do
  echo "== $tool" > "$OUT/sanitize_$tool.log"
  LSPG_NO_GRAPH=1 timeout $T $CS --tool $tool --print-limit 20 --launch-timeout 120 \
      python tests/gpu_bringup.py final normal B parity 256 2 >> "$OUT/sanitize_$tool.log" 2>&1
  echo "rc=$?" >> "$OUT/sanitize_$tool.log"
  grep -E "ERROR SUMMARY|RACECHECK SUMMARY|max\|out-oracle\||rc=" "$OUT/sanitize_$tool.log" | tail -4
done
echo "logs: $OUT"
