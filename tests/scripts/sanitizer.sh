#!/bin/bash
# compute-sanitizer over the small-n GPU matrix (the reference wraps its tests the same way,
# tools/cuda/compute_sanitizer_wrapper.sh). Usage: tests/scripts/sanitizer.sh <log dir>
OUT=${1:?usage: sanitizer.sh <log dir>}
mkdir -p "$OUT"
SEL="test_edge_cases or test_reference_golden_commitments or test_fixed_packed_vlen_and_file_roundtrip or test_upload_pieces_weierstrass or test_get_generators_and_one_commit or test_handle_from_reference_partition_table_file"
timeout 1500 compute-sanitizer --tool memcheck --error-exitcode 9 --launch-timeout 300 python -m pytest tests/test_gpu_parity.py -m gpu -x -q -k "$SEL" > "$OUT/sanitizer_memcheck.log" 2>&1
echo "memcheck rc=$?" | tee -a "$OUT/sanitizer_memcheck.log"
timeout 1500 compute-sanitizer --tool racecheck --error-exitcode 9 --launch-timeout 300 python -m pytest tests/test_gpu_parity.py -m gpu -x -q -k "test_reference_golden_commitments or test_get_generators_and_one_commit" > "$OUT/sanitizer_racecheck.log" 2>&1
echo "racecheck rc=$?" | tee -a "$OUT/sanitizer_racecheck.log"
tail -5 "$OUT/sanitizer_memcheck.log" "$OUT/sanitizer_racecheck.log"
