#!/bin/bash
# Multi-GPU round on an N-GPU machine: the sharded == single-GPU check, then bench lines.
#   scripts/run_mgpu.sh <N> [bench steps] [extra bench configs, e.g. "4 5"]     (logs under $MIMO_OUT, default mimo_out/)
OUT=${MIMO_OUT:-mimo_out}
N=${1:-2}; STEPS=${2:-3}; EXTRA=${3:-}
mkdir -p $OUT
export NCCL_DEBUG=WARN
PORT=29711
echo "== mgpu_check N=$N"
timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $PORT \
    scripts/mgpu_check.py --out $OUT/r2_mgpu_check_n$N.json > $OUT/r2_mgpu_check_n$N.log 2>&1
echo "mgpu_check rc=$?" | tee -a $OUT/r2_mgpu_check_n$N.log
tail -12 $OUT/r2_mgpu_check_n$N.log
echo "== bench N=$N"
timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $((PORT+1)) \
    bench.py --gpus $N --steps $STEPS --warmup 3 --no-cpu-baseline > $OUT/r2_bench_n$N.json 2> $OUT/r2_bench_n$N.err
echo "bench rc=$?"; head -c 700 $OUT/r2_bench_n$N.json; echo; tail -5 $OUT/r2_bench_n$N.err
for C in $EXTRA; do
  echo "== bench N=$N config $C"
  timeout 1200 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $((PORT+1+C)) \
      bench.py --gpus $N --config $C --steps 2 --warmup 3 --no-cpu-baseline > $OUT/r2_bench_n${N}_cfg$C.json 2> $OUT/r2_bench_n${N}_cfg$C.err
  echo "bench cfg$C rc=$?"; head -c 700 $OUT/r2_bench_n${N}_cfg$C.json; echo; tail -5 $OUT/r2_bench_n${N}_cfg$C.err
done
