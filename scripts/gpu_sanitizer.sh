#!/bin/bash
# compute-sanitizer over small parity tests: memcheck (out-of-bounds / misaligned, incl. shared memory and bulk copies),
# racecheck (shared-memory hazards), synccheck (barrier misuse).  Logs -> <dir>/sanitizer_*.log
#   scripts/gpu_sanitizer.sh [dir]   (default: a new temporary directory)
OUT="${1:-$(mktemp -d)}"
mkdir -p "$OUT"
echo "logs in $OUT"
# world batches (k_generic_jit_batch): shape parity with the oracle at one instance of the batch kernel
T="tests/test_gpu_batch_oracle.py::test_shape_parity_with_the_oracle[item128_rows2] tests/test_gpu_component_presence.py tests/test_gpu_box_game.py tests/test_gpu_engine_edges.py tests/test_gpu_desync_capture.py tests/test_gpu_checkpoint.py::test_refusals_leave_the_engine_unchanged tests/test_gpu_checkpoint.py::test_zero_rows_roundtrip"
P='tests/test_gpu_parity_particles.py -k "fused_matches_oracle and not 50000 or despawn_inside or spawn_particles_inside or odd_sizes or many_tiles or 3000-40 or 257 or 700"'
for tool in memcheck racecheck synccheck; do
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 9 --print-limit 20 python -m pytest $T -m gpu -x -q > "$OUT"/sanitizer_$tool.log 2>&1
  echo "$tool generic/stepwise rc=$?  $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|passed|failed' "$OUT"/sanitizer_$tool.log | tr '\n' ' ')"
  eval timeout 900 compute-sanitizer --tool $tool --error-exitcode 9 --print-limit 20 python -m pytest $P -m gpu -x -q > "$OUT"/sanitizer_${tool}_particles.log 2>&1
  echo "$tool particles rc=$?  $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|passed|failed' "$OUT"/sanitizer_${tool}_particles.log | tr '\n' ' ')"
done
