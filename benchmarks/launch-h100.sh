#!/bin/bash
# Run the four generated weak-scaling sweeps on one 8xH100 box (counterpart of the reference's
# benchmarks/launch-summit.sh).  Environment knobs:
#   DFNO_BENCH_BACKEND=auto|fused|torch   engine selection (default auto: fused when supported)
#   DFNO_P2P_REPARTITION=0                portable backend: NCCL all_to_all instead of peer-memory push
#   DFNO_STAGED_SCATTER=0|1               fused engine: direct / staged peer layout (default: staged from 8 ranks)
#   DFNO_NVTX=1                           NVTX ranges around the engine phases (lift / block k spectral, bypass / head)
#   DFNO_SYNC_TIMERS=1                    dt_comm timers synchronise the device around collectives
#   PROFILE=<dir>                         wrap 1-GPU points in `ncu --set full` (see bench.sh)
#   NCCL_DEBUG=INFO                       shows whether NVLS is in use by the baseline
set -euo pipefail
cd "$(dirname "$0")"
ulimit -c 0
MAXW=${1:-8}
python gen_scripts.py --system h100 --max-workers "$MAXW" --clean-old
for kind in eval grad; do
  for axis in spatial temporal; do
    n=1
    while [ "$n" -le "$MAXW" ]; do
      ./${kind}_weak_scaling_${axis}_gpu.sh "$n"
      n=$((n * 2))
    done
  done
done
python - <<'PY'
import glob, json, os
rows = []
for f in sorted(glob.glob("*_weak_scaling_*_gpu/*.json")):
    r = json.load(open(f))
    rows.append((os.path.dirname(f), os.path.basename(f), r.get("dt"), r.get("dt_comm"), r.get("dt_grad")))
for r in rows:
    print(*r, sep="\t")
PY
