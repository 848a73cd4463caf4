#!/bin/bash
# compute-sanitizer racecheck / synccheck / memcheck over the GPU tests that
# exercise the shared-memory kernels (mbarrier rings of the TMA kernels, the
# in-place shared-memory FFT, the regrid staging, the threshold kernel's
# shared-memory accumulators and its __syncthreads under a col_w branch, the
# mbarrier rings at unusual nstage / maxslots of the region-reduction cases).  Full-size cases are
# deselected (the tools slow kernels down 10-100x).  Logs go to OUT_DIR.
#   bash benchmarks/sanitize.sh [OUT_DIR]
OUT="${1:-$(mktemp -d)}"
mkdir -p "$OUT"
SEL='not fullsize and not full_size and not headline and not 721 and not m50 and not correlated and not k1_tma_scratch and not test_realistic_family and not long_time_sum and not claimed_instance'
TESTS="tests/test_spectrum_pfa_gpu.py tests/test_spectrum_cases_gpu.py tests/test_regrid_tma_gpu.py tests/test_regrid_cases_gpu.py tests/test_det_metrics_gpu.py tests/test_host_streaming_gpu.py tests/test_ens_metrics_gpu.py tests/test_threshold_abi_gpu.py tests/test_wind_dynamics_gpu.py tests/test_region_reduce_gpu.py tests/test_precip_accumulation_gpu.py tests/test_column_integrals_gpu.py tests/test_interp_cases_gpu.py"
for tool in racecheck synccheck memcheck; do
  timeout 900 compute-sanitizer --tool $tool --print-limit 20 \
    python -m pytest $TESTS -x -q -m gpu -k "$SEL" -p no:cacheprovider \
    > "$OUT/sanitizer_$tool.txt" 2>&1
  echo "== $tool rc=$?"; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed|hazard" "$OUT/sanitizer_$tool.txt" | tail -5
done
