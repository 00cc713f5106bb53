#!/bin/bash
# compute-sanitizer over the small parity tests of the new kernels, then the whole GPU suite
OUT=runs/sanitize; mkdir -p $OUT
K='corner_cases or send_list or (compact_stream_submission and 40000) or (step_begin_records and (900 or 30000)) or golden or every_ingest_path or fused_tile_step_learners'
timeout 1500 compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -m gpu -x -q -k "$K" > $OUT/memcheck.txt 2>&1; echo "memcheck rc=$?" | tee -a $OUT/memcheck.txt
grep -E "ERROR SUMMARY|passed|failed|Invalid|out of bounds" $OUT/memcheck.txt | tail -6
timeout 1500 compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -m gpu -x -q -k "corner_cases or (compact_stream_submission and 40000) or fused_tile_step_learners or (every_ingest_path and 1)" > $OUT/racecheck.txt 2>&1; echo "racecheck rc=$?" | tee -a $OUT/racecheck.txt
grep -E "RACECHECK SUMMARY|passed|failed|hazard" $OUT/racecheck.txt | tail -6
if [ -z "$1" ]; then timeout 1500 python -m pytest tests -m gpu -x -q > $OUT/pytest_gpu.txt 2>&1; tail -n 4 $OUT/pytest_gpu.txt; fi
