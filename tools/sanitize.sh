#!/bin/bash
# compute-sanitizer gate (SURVEY.md section 5: the reference has no sanitizer runs at all): memcheck over small instances of every
# kernel family through the C ABI, racecheck over the shared-memory kernels of the TSDF path.  Run under gpurun from the repo root.
# Every leg is time-bounded; results land in gpurun_out/<R>_sanitize_*.log, the last lines are the sanitizer's summary.
R=${1:-r02}
T1=${2:-420}
T2=${3:-150}
mkdir -p gpurun_out
CS="compute-sanitizer --error-exitcode 9 --print-limit 10 --launch-timeout 60"
leg() {  # name, timeout, tool, pytest selection...
  local name=$1 to=$2 tool=$3; shift 3
  timeout $to $CS --tool $tool python -m pytest "$@" -m gpu -q -x -p no:cacheprovider > gpurun_out/${R}_sanitize_${name}.log 2>&1
  echo "$name ($tool): exit $? | $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|passed|failed' gpurun_out/${R}_sanitize_${name}.log | tr '\n' ' ')"
}
leg mem $T1 memcheck tests/test_fusion_gpu.py tests/test_tracker_gpu.py tests/test_front_gpu.py tests/test_mvsnet_gpu.py \
  -k "integrate_and_render or negative_coordinates or mesh_matches_oracle_bit_exact or roundtrip or bucket_overflow or (calc_res and size0) or cutoff or (pyramid and not size0) or (dense_reference_matches and not True) or (lm_loop and size0) or (config1 and mixed16) or interleaved or pixel_partitioned or mesh_state_machine or batched_hypotheses"
leg race $T2 racecheck tests/test_fusion_gpu.py tests/test_mvsnet_gpu.py -k "mesh_call_order or negative_coordinates"
leg pyramid_mem $T1 memcheck tests/test_track_pyramid_gpu.py -k "not shim and not size1"
leg pyramid_race $T2 racecheck tests/test_track_pyramid_gpu.py -k "equals_host and size0"
leg new_coarse_mem $T1 memcheck tests/test_track_new_coarse_gpu.py -k "not shim and not size1"
leg new_coarse_race $T2 racecheck tests/test_track_new_coarse_gpu.py -k "host_loop and size0 and retrack"
leg conv_is_mem $T1 memcheck tests/test_conv_is_gpu.py -k "abl04"
leg feature_cache_mem $T1 memcheck tests/test_mvsnet_feature_cache_gpu.py -k "handoff or golden"
leg feature_cache_race $T2 racecheck tests/test_mvsnet_feature_cache_gpu.py -k "handoff"
leg trace_mem $T1 memcheck tests/test_trace_gpu.py -k "not shim and not random and not 2560"
leg activate_mem $T1 memcheck tests/test_activate_gpu.py -k "not shim and not random"
leg pixsel_mem $T1 memcheck tests/test_pixsel_gpu.py -k "not shim and not sequences"
leg undistort_mem $T1 memcheck tests/test_undistort_gpu.py -k "not shim and not tracker and not trace"
leg linearize_mem $T1 memcheck tests/test_linearize_gpu.py -k "not shim and not seeded"
leg accumulate_mem $T1 memcheck tests/test_accumulate_gpu.py -k "room or invalid or zero"
