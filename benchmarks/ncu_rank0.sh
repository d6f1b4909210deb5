#!/bin/bash
# Profile the multi-GPU all-reduce kernel on ONE rank while the other ranks run plain.
#
#   benchmarks/ncu_rank0.sh N OUT_PREFIX [script args...]      (from the repo root, on an N-GPU box)
#
# ncu replays a kernel once per metric pass, and a kernel that waits for the other processes' flags
# cannot be replayed (the peers run it once).  So rank 0 runs under ncu with a metric list that fits ONE
# pass (no replay: --replay-mode application is not used either), ranks 1..N-1 run without a profiler, and
# the device-side flag timeout is short so that a mistake fails fast instead of hanging the box.  The
# script each rank runs is benchmarks/trace_fuse.py (a few sync_model calls on ResNet-sized gradient lists).
# Writes OUT_PREFIX.csv (ncu raw page) and OUT_PREFIX.log.
set -u
N=${1:-8}; OUT=${2:-$(mktemp -d)/ncu_rank0}; shift 2 || true
PORT=${MASTER_PORT:-29533}
METRICS="gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,launch__registers_per_thread,launch__grid_size,launch__block_size,smsp__warps_active.avg.per_cycle_active,lts__t_sectors_srcunit_tex_op_read.sum,lts__t_sectors_srcunit_tex_op_write.sum"
export MASTER_ADDR=127.0.0.1 MASTER_PORT=$PORT WORLD_SIZE=$N FLASHY_B200_DEVICE_TIMEOUT=${FLASHY_B200_DEVICE_TIMEOUT:-20}
pids=()
for r in $(seq 1 $((N-1))); do
  RANK=$r LOCAL_RANK=$r python benchmarks/trace_fuse.py "$@" > /dev/null 2>> $OUT.log &
  pids+=($!)
done
RANK=0 LOCAL_RANK=0 ncu --metrics $METRICS --clock-control none --cache-control none --replay-mode kernel \
  -k regex:k_fuse --launch-skip 4 --launch-count 3 --csv --page raw --log-file $OUT.csv \
  python benchmarks/trace_fuse.py "$@" > $OUT.rank0.out 2>> $OUT.log
rc=$?
for p in "${pids[@]}"; do wait $p; done
echo "ncu rank0 rc=$rc" >> $OUT.log
exit $rc
