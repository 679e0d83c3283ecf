#!/bin/bash
# compute-sanitizer passes over the sm_90a kernels (run on an H100; slow -- the tests below use small shapes).
#   tools/sanitize.sh [memcheck|racecheck|synccheck|initcheck]        1 GPU: GEMM, fused pointwise, FFT, engine step
#   N=2 tools/sanitize.sh memcheck                                     + the peer-scatter / barrier path on 2 GPUs
# Logs go to sanitize_logs/sanitize_<tool>[_2gpu].log; the exit code is the sanitizer's.
tool=${1:-memcheck}
cd "$(dirname "$0")/.."
mkdir -p sanitize_logs
CS="compute-sanitizer --tool $tool --error-exitcode 1 --launch-timeout 120 --target-processes all"
rc=0
$CS python -m pytest tests/test_dft_gemm_gpu.py tests/test_fused_pointwise_gpu.py tests/test_fft_radix_gpu.py \
    tests/test_spectral_in_gpu.py -x -q -k "rowmajor or scatter or spectral_out or dpre_dw or head or forward_inverse or spectral_in" \
    > sanitize_logs/sanitize_${tool}.log 2>&1 || rc=$?
tail -n 5 sanitize_logs/sanitize_${tool}.log
# the optimizer kernels: sum of squares, both Adam paths, the replayed step
$CS python -m pytest tests/test_fused_optim_gpu.py -x -q -k "sumsq or nonfinite or (matches_torch and step) or no_host_sync" \
    > sanitize_logs/sanitize_${tool}_optim.log 2>&1 || rc=$?
tail -n 5 sanitize_logs/sanitize_${tool}_optim.log
if [ "${N:-1}" -ge 2 ]; then
  DFNO_TEST_WORLD=2 $CS python -m pytest tests/test_fused_multigpu.py tests/test_p2p_multigpu.py -x -q \
      > sanitize_logs/sanitize_${tool}_2gpu.log 2>&1 || rc=$?
  tail -n 5 sanitize_logs/sanitize_${tool}_2gpu.log
fi
exit $rc
