#!/bin/bash
# compute-sanitizer passes over a small parity workload (run under gpurun): memcheck + racecheck + synccheck.
# Logs -> gpurun_out/sanitizer_<tool>.log; the summary lines are what profiles/<round>_sanitizer.md quotes.
set -u
mkdir -p gpurun_out
SEL="window or demo_corridor_batch or generic_and_specialised or no_polytopes or exact_miqp or device_side_fill or pairs_match_oracle or early_exit or wrong_polytope_size or infeasibility_certificates or full_active_set or specialised_limit or face_cap or shared_memory_limit or generic_limit or thirty_two or stall_and_statuses or device_statuses"
for tool in memcheck racecheck synccheck; do
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 9 python -m pytest tests/test_parity_gpu.py tests/test_pair_gpu.py tests/test_certificates_gpu.py tests/test_capacity_gpu.py tests/test_pair_window_gpu.py tests/test_map_paths_gpu.py tests/test_jps_batch_gpu.py -x -q \
      -k "$SEL" > gpurun_out/sanitizer_$tool.log 2>&1
  echo "$tool rc=$?" >> gpurun_out/sanitizer_$tool.log
done
grep -h -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed|rc=" gpurun_out/sanitizer_*.log
