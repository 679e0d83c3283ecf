#!/bin/bash
# One-time setup on an H100 box (counterpart of the reference's benchmarks/install_summit.sh, which
# builds a conda env + mpi4py + cupy + a patched DistDL).  Nothing is downloaded here: the framework
# needs PyTorch (>= 2.6, CUDA 12.8+) and nvcc only; the sm_90a extension is compiled in-tree.
set -euo pipefail
cd "$(dirname "$0")/.."

python - <<'PY'
import shutil, sys, torch
print("python      ", sys.version.split()[0])
print("torch       ", torch.__version__, "cuda", torch.version.cuda)
print("nvcc        ", shutil.which("nvcc"))
print("GPUs        ", torch.cuda.device_count(), [torch.cuda.get_device_name(i) for i in range(torch.cuda.device_count())])
print("nccl / gloo ", torch.distributed.is_nccl_available(), torch.distributed.is_gloo_available())
if torch.cuda.is_available():
    cc = torch.cuda.get_device_capability(0)
    assert cc == (9, 0), f"the fused engine targets sm_90a (H100); found sm_{cc[0]}{cc[1]} -- the portable backend still works"
PY

python __graft_entry__.py                       # nvcc -gencode arch=compute_90a,code=sm_90a -> dfno_b200/_build/*.so
python -m pip install --no-deps --no-build-isolation -e . 2>/dev/null || echo "(editable install skipped: run from the repo root instead)"
python -m pytest tests -q -m "not gpu" -x
if python -c "import torch,sys; sys.exit(0 if torch.cuda.is_available() else 1)"; then
  python -m pytest tests -q -m gpu -x
fi
