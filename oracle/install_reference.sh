#!/bin/bash
# Install the UNMODIFIED reference package (slimgroup/dfno) into oracle/_ref (git-ignored), without its
# dependencies: DistDL / mpi4py resolve to the stand-in in baseline/compat.  Used by `bench.py --impl reference`
# (baseline/reference_arm.py) and by oracle/gen_reference_parity.py.
#   oracle/install_reference.sh <path of a slimgroup/dfno checkout>
set -euo pipefail
src=${1:?usage: oracle/install_reference.sh <path of a slimgroup/dfno checkout>}
cd "$(dirname "$0")"
rm -rf _ref
python -m pip install -q --no-deps --no-index --no-build-isolation --target _ref "$src"
python -c "import sys; sys.path.insert(0, '_ref'); import importlib.util as u; assert u.find_spec('dfno'), 'dfno missing'"
echo "reference package installed in $(pwd)/_ref"
