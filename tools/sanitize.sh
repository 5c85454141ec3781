#!/bin/bash
# compute-sanitizer pass over a representative subset of the GPU tests (memcheck: out-of-bounds / misaligned accesses in
# every kernel of the library; racecheck on the shared-memory hand-offs of the search, GEMM and loss kernels).
#   bash tools/sanitize.sh [OUT_DIR]      (summaries go to OUT_DIR, default: a fresh temporary directory)
OUT=${1:-$(mktemp -d -t openmatch-sanitize.XXXXXX)}
mkdir -p "$OUT"
SEL="tests/test_search_gpu.py::test_integer_data_exact tests/test_search_gpu.py::test_small_duplicate_cluster_resolved_by_wide_level tests/test_search_gpu.py::test_near_duplicate_cluster_is_exact tests/test_search_gpu.py::test_sharded_merge_matches_unsharded tests/test_search_gpu.py::test_pair_scan_and_single_cta_scan_agree[9000-64-257-10] tests/test_scan_cluster_gpu.py::test_query_edges[200-4x2] tests/test_scan_cluster_gpu.py::test_last_cluster_tile_edges[1-4x2] tests/test_scan_cluster_gpu.py::test_massive_ties_overflow_the_stash[2x2] tests/test_search_numerics_gpu.py::test_merge_accepted[3-4096-4096] tests/test_search_numerics_gpu.py::test_small_dims[1-300] tests/test_search_numerics_gpu.py::test_small_dims[17-300] tests/test_search_numerics_gpu.py::test_largest_k[4096-30000-7] tests/test_loss_gpu.py tests/test_loss_numerics_gpu.py::test_matrix[split3_odd_d] tests/test_loss_numerics_gpu.py::test_call_sequence tests/test_encoder_gpu.py::test_bert_small_matches_reference_golden tests/test_encoder_gpu.py::test_t5_small_matches_reference_golden tests/test_encoder_numerics_gpu.py::test_non_prefix_masks[holes_17] tests/test_encoder_numerics_gpu.py::test_online_softmax_tile_maxima_bert[256-3-max_in_last_tile]"
timeout 1200 compute-sanitizer --tool memcheck --error-exitcode 3 --print-limit 20 python -m pytest $SEL -m gpu -x -q -p no:cacheprovider > "$OUT/memcheck.log" 2>&1
echo "memcheck rc=$?" >> "$OUT/memcheck.log"
tail -5 "$OUT/memcheck.log"
timeout 900 compute-sanitizer --tool racecheck --error-exitcode 3 --print-limit 20 python -m pytest "tests/test_search_gpu.py::test_integer_data_exact" "tests/test_search_gpu.py::test_massive_ties" "tests/test_search_gpu.py::test_pair_scan_and_single_cta_scan_agree[9000-64-257-10]" "tests/test_scan_cluster_gpu.py::test_last_cluster_tile_edges[1-4x2]" "tests/test_scan_cluster_gpu.py::test_massive_ties_overflow_the_stash[2x2]" "tests/test_loss_gpu.py::test_gradients_are_run_to_run_identical" -m gpu -x -q -p no:cacheprovider > "$OUT/racecheck.log" 2>&1
echo "racecheck rc=$?" >> "$OUT/racecheck.log"
tail -5 "$OUT/racecheck.log"
