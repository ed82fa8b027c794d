#!/bin/bash
# Memory / race checks of our kernels on the GPU (SURVEY.md §5.2: the reference has none):
#   bash profiles/run_sanitizer.sh
# Small shapes only: compute-sanitizer slows kernels down by 10-100x.
set -x
mkdir -p profiles_out
export ODB_LOGLEVEL=WARNING
T1="python -m pytest tests/test_kernels_gpu.py -x -q -k 'embedding or rmsnorm or rope or swiglu or adamw or nesterov or cross_entropy or (tcgen05_attention and 1-128-1-1)'"
T2="python -m pytest tests/test_tc_gemm_gpu.py -x -q -k '128-256-64 or 300-520-200'"
timeout 200 compute-sanitizer --tool memcheck --error-exitcode 3 bash -c "$T1" > profiles_out/sanitizer_memcheck.log 2>&1; echo "memcheck(elementwise+attention) rc=$?"
timeout 150 compute-sanitizer --tool memcheck --error-exitcode 3 bash -c "$T2" > profiles_out/sanitizer_memcheck_gemm.log 2>&1; echo "memcheck(gemm) rc=$?"
timeout 150 compute-sanitizer --tool racecheck --error-exitcode 3 bash -c "python -m pytest tests/test_kernels_gpu.py -x -q -k 'rmsnorm or cross_entropy or adamw'" > profiles_out/sanitizer_racecheck.log 2>&1; echo "racecheck(block-reduction kernels) rc=$?"
for f in profiles_out/sanitizer_*.log; do echo "== $f"; tail -n 4 "$f"; done
