#!/bin/bash
# Round-2 sanitizer call: compute-sanitizer (memcheck + racecheck) on the new / changed kernels, and the whole
# -m gpu suite's host side under an ASan + UBSan build of the library.  usage: scripts/gpu_sanitize_r2.sh <tag>
TAG=${1:-r02s}; OUT=runs/$TAG; mkdir -p $OUT
K="wire or heartbeat or update_state or every_ingest or raw_record or async_record"
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 7 python -m pytest tests -m gpu -x -q -k "$K" > $OUT/memcheck.txt 2>&1; echo "memcheck rc=$?" >> $OUT/memcheck.txt
timeout 900 compute-sanitizer --tool racecheck --error-exitcode 7 python -m pytest tests/test_gpu_wire.py tests/test_gpu_parity.py -m gpu -x -q -k "wire_golden or golden_messages or every_ingest or heartbeat" > $OUT/racecheck.txt 2>&1; echo "racecheck rc=$?" >> $OUT/racecheck.txt
tail -n 4 $OUT/memcheck.txt; tail -n 4 $OUT/racecheck.txt
# host side under ASan + UBSan: the library built with -fsanitize=address,undefined stands in for libraftgpu.so
if [ -f raft-rs_b200/libraftgpu_asan.so ]; then
  cp raft-rs_b200/libraftgpu.so /tmp/libraftgpu_plain.so && cp raft-rs_b200/libraftgpu_asan.so raft-rs_b200/libraftgpu.so
  ASAN=$(gcc -print-file-name=libasan.so); UBSAN=$(gcc -print-file-name=libubsan.so)
  LD_PRELOAD="$ASAN $UBSAN" ASAN_OPTIONS=protect_shadow_gap=0:detect_leaks=0:abort_on_error=0:halt_on_error=0 UBSAN_OPTIONS=print_stacktrace=1 \
    timeout 1200 python -m pytest tests -m gpu -x -q -k "every_ingest or wire or concurrent or async_record or raw_record or compact or enqueue or heartbeat or update_state or synthetic_stream_elementwise" > $OUT/asan.txt 2>&1; echo "asan rc=$?" >> $OUT/asan.txt
  cp /tmp/libraftgpu_plain.so raft-rs_b200/libraftgpu.so
  grep -c "ERROR: AddressSanitizer\|runtime error" $OUT/asan.txt; tail -n 4 $OUT/asan.txt
fi
