#!/bin/bash
# Where do the warps of the intra-picture and inter kernels spend their cycles?  (variant build with -DE264_PHASE_TIMING)
cd "$(dirname "$0")/.."; TAG=${1:-run}; D=${D:-$PWD/edge264_b200/variants/timing}; OUT=${OUT:-${TMPDIR:-/tmp}}; mkdir -p "$OUT"
{
env LD_LIBRARY_PATH=$D E264_LIB_DIR=$D E264B_DIAG=1 S=8 STEPS=2 E264B_REPLAY_INFLIGHT=1 timeout -k 5 120 python tools/replay_ab.py 2>&1 | grep -E "kernel|total"
env LD_LIBRARY_PATH=$D E264_LIB_DIR=$D E264B_DIAG=1 S=32 STEPS=2 timeout -k 5 120 python tools/replay_ab.py 2>&1 | grep -E "kernel|total"
} 2>&1 | tee "$OUT/phase_timing_$TAG.txt"
