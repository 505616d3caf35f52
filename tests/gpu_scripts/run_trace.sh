#!/bin/bash
# Steady-state clock64 timelines of selected conv layers (see tests/gpu_trace.py; slots documented in csrc/conv_wgmma.cuh).
# Usage:  bash tests/gpu_scripts/run_trace.sh "1,2,70" [first local tile] [batch]
LOG=$(mktemp)
LSPG_TRACE_SKIP=${2:-20} LSPG_TRACE_LAYERS=${1:-1,2} LSPG_TRACE_CTAS=0,1 timeout 600 python tests/gpu_trace.py large parity ${3:-16} > "$LOG" 2>&1
grep -E "^layer|GHz|^CTA 0:|   tile [0-5]:|mma:|epi:|wait_first_stage" "$LOG" | cut -c1-200
echo "full log: $LOG"
