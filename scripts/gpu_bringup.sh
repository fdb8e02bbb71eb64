#!/bin/bash
# Kernel bring-up on an H100: every probe in its own process, bounded by timeout; logs under $MIMO_OUT (default mimo_out/).
OUT=${MIMO_OUT:-mimo_out}
mkdir -p $OUT
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.draw,memory.total --format=csv > $OUT/smi.txt 2>&1
LOG=$OUT/bringup.log
: > $LOG
for t in ${@:-gemm_basic gemm_shapes gemm_persistent gemm_epilogue conv_basic conv_shapes norms temporal elementwise spatial_basic spatial_shapes perf}; do
  echo "##### $t" >> $LOG
  timeout 240 python scripts/gpu_probe.py $t >> $LOG 2>&1
  echo "exit=$?" >> $LOG
done
grep -E "^\[|^==|exit=|#####|TFLOP|GB/s" $LOG | tail -150
