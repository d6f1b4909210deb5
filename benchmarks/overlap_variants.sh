#!/bin/bash
# Step time of bench.py with / without backward overlap at 2 GPUs (one rank per GPU), on a machine with 2 GPUs:
#   OUT=<dir> bash benchmarks/overlap_variants.sh        (raw lines go to OUT, default a new temporary directory)
OUT=${OUT:-$(mktemp -d)}
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1"
run() { tag=$1; shift; env "$@" timeout 150 $TR --master-port 29510 bench.py --gpus 2 --world 2 --steps 15 --warmup 3 --no-parity $EXTRA > $OUT/ovl_$tag.json 2> $OUT/ovl_$tag.err; python - <<PY
import json
try:
    d=json.loads(open("$OUT/ovl_$tag.json").read().strip().splitlines()[-1])
    print("$tag", "ms_step", round(d["ms_per_step"],4), "single", round(d["aux"]["single_rank_no_sync_ms_per_step"],4), "exposed_us", round(1e3*d["aux"]["exposed_sync_ms"],1), "launches", d["gpu_launches"], "kernel_us", round(1e3*d["allreduce"]["kernel_ms"],1))
except Exception as e:
    print("$tag failed", e)
PY
}
EXTRA="" run noovl A=1
EXTRA="--overlap" run b32 FLASHY_B200_OVERLAP_BLOCKS=32
EXTRA="--overlap" run b132 FLASHY_B200_OVERLAP_BLOCKS=132
EXTRA="--overlap" run b16 FLASHY_B200_OVERLAP_BLOCKS=16
EXTRA="--overlap" run b32_4mb FLASHY_B200_OVERLAP_BLOCKS=32 FLASHY_B200_OVERLAP_BUCKET_MB=4
EXTRA="--overlap" run b32_nvls FLASHY_B200_OVERLAP_BLOCKS=32 FLASHY_B200_NVLS_MIN_WORLD=2
