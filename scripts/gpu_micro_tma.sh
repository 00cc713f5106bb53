#!/bin/bash
OUT=runs/micro_tma; mkdir -p $OUT
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/tma_chunks scripts/micro/tma_chunks.cu || exit 1
{
for cfg in "1024 25 8" "2048 25 4" "4096 25 2" "2048 12 8" "4096 12 4" "8192 6 4" "10240 5 4" "16384 3 4" "51200 1 4" "25600 1 8" "10240 5 2" "10240 5 3" "2048 25 2" "2048 25 3" "12288 4 4" "12288 4 3"; do
  timeout 60 /tmp/tma_chunks $cfg 200
done
} | tee $OUT/tma_chunks.txt
