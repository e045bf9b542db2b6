#!/bin/bash
# compute-sanitizer passes over the CUDA kernels (run on a GPU machine: bash tools/sanitize_gpu.sh).
# memcheck: out-of-bounds / misaligned accesses; synccheck: illegal barrier / warp-sync use;
# racecheck: shared-memory hazards. The tests are the small-shape numerics tests (the sanitizers
# slow kernels down 10-100x). Output: $OUT/sanitize_*.log (default sanitize_out/)
set -u
OUT=${OUT:-sanitize_out}
mkdir -p "$OUT"
T="tests/test_gpu_sparse_engine.py::test_hot_rows_many_duplicates tests/test_gpu_sparse_engine.py::test_virtual_ranks tests/test_gpu_sparse_engine.py::test_planned_batches tests/test_gpu_sparse_engine.py::test_split_row_feature tests/test_gpu_sparse_engine.py::test_context_version_guard tests/test_gpu_sparse_exact.py::test_layouts_exact tests/test_gpu_sparse_exact.py::test_hash_shard_capacity tests/test_gpu_gemm.py::test_dw_mn_major tests/test_gpu_gemm.py::test_cin_own_kernels_match_torch tests/test_gpu_gemm.py::test_chain_matches_single_launches tests/test_gpu_gemm_epilogue_src.py tests/test_gpu_gemm_exact.py::test_dx_mask_edge_values tests/test_gpu_gemm_exact.py::test_dx_fm_d_and_fm_cols tests/test_gpu_gemm_exact.py::test_argument_errors_raise tests/test_gpu_gemm_exact.py::test_chain_forward_backward[128-exact] tests/test_gpu_gemm_exact.py::test_chain_forward_backward[300-exact] tests/test_gpu_fused.py::test_fused_step_matches_reference tests/test_gpu_host_tier.py::test_tiered_equals_untiered_bitwise"
for tool in memcheck synccheck racecheck; do
  timeout ${SAN_TIMEOUT:-900} compute-sanitizer --tool $tool --error-exitcode 99 --target-processes all \
      python -m pytest $T -x -q -k "${SAN_FILTER:-}" > "$OUT/sanitize_$tool.log" 2>&1
  echo "$tool: exit $? ; $(grep -c 'ERROR SUMMARY' "$OUT/sanitize_$tool.log") summaries; $(grep 'ERROR SUMMARY' "$OUT/sanitize_$tool.log" | tail -1)"
done
