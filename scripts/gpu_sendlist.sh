#!/bin/bash
OUT=runs/sendlist; mkdir -p $OUT
timeout 900 python -m pytest tests/test_gpu_parity.py -m gpu -x -q -k "send_list" 2>&1 | tail -5
timeout 600 python scripts/micro_send_list.py 2>&1 | tee $OUT/micro_send_list.txt | tail -4
