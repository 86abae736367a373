#!/bin/bash
# compute-sanitizer over the round-2 kernels (small problems; memcheck, racecheck and synccheck on the shared-memory kernels)
OUT=gpurun_out/r02_compute_sanitizer.txt
: > $OUT
T="tests/test_gpu_assoc.py::test_window_associate_equals_single_calls tests/test_gpu_assoc.py::test_window_slide_equals_fresh_window tests/test_features.py tests/test_marginalize.py tests/test_gpu_stride8.py::test_batch_frames_stride8 tests/test_gpu_edge_cases.py"
echo "=== memcheck" >> $OUT
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest $T -x -q -m gpu 2>&1 | grep -E "ERROR SUMMARY|passed|failed|Invalid|error" | tail -6 >> $OUT
echo "=== racecheck" >> $OUT
timeout 900 compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_assoc.py::test_window_associate_equals_single_calls tests/test_features.py -x -q -m gpu 2>&1 | grep -E "RACECHECK SUMMARY|passed|failed|hazard" | tail -6 >> $OUT
echo "=== synccheck" >> $OUT
timeout 600 compute-sanitizer --tool synccheck --error-exitcode 9 python -m pytest tests/test_gpu_assoc.py::test_window_associate_equals_single_calls tests/test_features.py -x -q -m gpu 2>&1 | grep -E "ERROR SUMMARY|passed|failed" | tail -4 >> $OUT
cat $OUT
