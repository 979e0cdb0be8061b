#!/bin/bash
# Builds tools/probe/probe_sm90 (when its source is newer) and runs it on cuda:0; the table goes to
# profiles/probe_sm90.txt, headed by the card's name, power limit and clocks.
#   tools/probe/run_probe.sh [all|mma|ingest|exchange] [output file]
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(dirname "$(dirname "$HERE")")"
BIN="$HERE/probe_sm90"
OUT="${2:-$ROOT/profiles/probe_sm90.txt}"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
if [ ! -x "$BIN" ] || [ "$HERE/probe_sm90.cu" -nt "$BIN" ] || [ "$ROOT/anakin_b200/csrc/ptx.cuh" -nt "$BIN" ]; then
    "$NVCC" -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o "$BIN" "$HERE/probe_sm90.cu" -lcuda
fi
mkdir -p "$(dirname "$OUT")"
{
    nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader
    "$BIN" "${1:-all}"
} | tee "$OUT"
