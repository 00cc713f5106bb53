#!/bin/bash
# Round-2 second sanitizer call (code added after the first): compute-sanitizer racecheck + memcheck on the fused kernels'
# new stage hand-over (wait_stage) at small sizes, and the host side of the wide-group / hybrid / fallback code under
# ASan + UBSan.  usage: scripts/gpu_sanitize_r2b.sh <tag>
TAG=${1:-r02s2}; OUT=runs/$TAG; mkdir -p $OUT
K="fused_compact_step_corner or fused_tile_step_learners or fused_kernels_in_their_other or golden_vectors_through_a_wide or wide_control"
timeout 400 compute-sanitizer --tool racecheck --error-exitcode 7 python -m pytest tests -m gpu -x -q -k "$K" > $OUT/racecheck.txt 2>&1; echo "racecheck rc=$?" >> $OUT/racecheck.txt
timeout 400 compute-sanitizer --tool memcheck --error-exitcode 7 python -m pytest tests -m gpu -x -q -k "$K or steps_over_mixed" > $OUT/memcheck.txt 2>&1; echo "memcheck rc=$?" >> $OUT/memcheck.txt
tail -n 3 $OUT/racecheck.txt; tail -n 3 $OUT/memcheck.txt
cp raft-rs_b200/libraftgpu.so /tmp/libraftgpu_plain.so && cp raft-rs_b200/libraftgpu_asan.so raft-rs_b200/libraftgpu.so
ASAN=$(gcc -print-file-name=libasan.so); UBSAN=$(gcc -print-file-name=libubsan.so)
LD_PRELOAD="$ASAN $UBSAN" ASAN_OPTIONS=protect_shadow_gap=0:detect_leaks=0:abort_on_error=0:halt_on_error=0 UBSAN_OPTIONS=print_stacktrace=1 \
  timeout 600 python -m pytest tests -m gpu -x -q -k "wide or hybrid or only_some_groups or inflights or every_ingest or concurrent or async_record or step_begin_records" > $OUT/asan.txt 2>&1; echo "asan rc=$?" >> $OUT/asan.txt
cp /tmp/libraftgpu_plain.so raft-rs_b200/libraftgpu.so
echo "sanitizer reports: $(grep -c 'ERROR: AddressSanitizer\|runtime error' $OUT/asan.txt)"; tail -n 3 $OUT/asan.txt
