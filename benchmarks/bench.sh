#!/bin/bash
# Wrapper: when $PROFILE names a directory, wrap the run in a profiler
# (reference benchmarks/bench.sh:4-13 wraps rank 0 and the last rank in `nsys profile`).
# Nsight Compute (ncu) must only wrap 1-GPU runs (a replayed kernel that waits for a peer never returns).
outdir=$1; shift
if test -d "$PROFILE" && test "${WORLD_SIZE:-1}" = 1; then
  ncu --set full --clock-control none --import-source on -k regex:"dft_gemm|head_bwd|kreduce|bypass" -c 12 \
      -o "$PROFILE/${outdir}_${RANK:-0}_${WORLD_SIZE:-1}" python3 bench.py "$@"
else
  python3 bench.py "$@"
fi
