#!/bin/bash
# Timing ablations of the fused kernel (wrong output; development aid): bash tools/ablate.sh [records]
cd "$(dirname "$0")/.."
N=${1:-10000000}
for d in "" "RV_ABL_SEQITEMS=1" "RV_ABL_NOLOOKBACK=1" "RV_ABL_NOCOPY=1" "RV_ABL_NOWALK=1" "RV_ABL_NOWALK=1;RV_ABL_NOCOUNTWALK=1" "RV_ABL_NOWALK=1;RV_ABL_NOCOUNTWALK=1;RV_ABL_NOLOOKBACK=1" "RV_ABL_NOCOPY=1;RV_ABL_NOLOOKBACK=1"; do
  echo "== $d"; RV_JIT_DEFS="$d" timeout 120 python tools/sweep_jit.py --records $N --steps 10 2>&1 | tail -1
done
echo "== k=1"; timeout 120 python tools/sweep_jit.py --records $N --steps 10 --num-chunks 1 2>&1 | tail -1
echo "== k=64"; timeout 120 python tools/sweep_jit.py --records $N --steps 10 --num-chunks 64 2>&1 | tail -1
