#!/bin/bash
# Multi-GPU evidence run (one box): NCCL == single-GPU test, then bench.py at N ranks for the variants BASELINE.json names.
# usage: [OUT=dir] [TRAIN=1] tools/run_scale.sh <N> <tag> [models...]   (results go to $OUT, default scale_out/)
N=$1; TAG=$2; shift 2
MODELS=${@:-"dinounet_l dinounet_b dinounet_s"}
OUT=${OUT:-scale_out}
mkdir -p "$OUT"
if [ "$N" -ge 2 ]; then
  timeout 600 python -m pytest tests/test_gpu_multi.py -q -m gpu 2>&1 | tail -3 > $OUT/${TAG}_nccl_test.txt
  cat $OUT/${TAG}_nccl_test.txt
fi
PORT=29511
for M in $MODELS; do
  B=32; [ "$M" = "dinounet_7b" ] && B=16
  PORT=$((PORT+1))
  if [ "$N" -eq 1 ]; then
    timeout 600 python bench.py --gpus 1 --steps 10 --warmup 3 --model $M --batch $B --cpu-sample 0 --eager-steps 0 > $OUT/${TAG}_${M}_n${N}.json 2> $OUT/${TAG}_${M}_n${N}.err
  else
    timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $PORT bench.py --gpus $N --steps 10 --warmup 3 --model $M --batch $B --cpu-sample 0 --eager-steps 0 > $OUT/${TAG}_${M}_n${N}.json 2> $OUT/${TAG}_${M}_n${N}.err
  fi
  python - <<PY
import json
try:
    d=json.loads(open("$OUT/${TAG}_${M}_n${N}.json").read().strip().splitlines()[-1])
    print("${M} N=${N}:", round(d["value"],1), "patches/s", round(d["ms_per_step"],2), "ms/step  e2e", round(d["e2e"]["value"],1), d["clocks"])
except Exception as e:
    print("${M} N=${N}: FAILED", e)
PY
done
if [ -n "$TRAIN" ]; then
  PORT=$((PORT+1))
  if [ "$N" -eq 1 ]; then
    timeout 900 python bench.py --mode train --model dinounet_b --batch 32 --steps 3 --warmup 3 > $OUT/${TAG}_train_b_n${N}.json 2> $OUT/${TAG}_train_b_n${N}.err
  else
    timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $PORT bench.py --mode train --gpus $N --model dinounet_b --batch 32 --steps 3 --warmup 3 > $OUT/${TAG}_train_b_n${N}.json 2> $OUT/${TAG}_train_b_n${N}.err
  fi
  tail -c 400 $OUT/${TAG}_train_b_n${N}.json | head -c 400; echo
  python -c "
import json
d=json.loads(open('$OUT/${TAG}_train_b_n${N}.json').read().strip().splitlines()[-1]); print('train dinounet_b N=${N}:', round(d['value'],1), 'patches/s', round(d['ms_per_step'],1), 'ms/step')" || tail -3 $OUT/${TAG}_train_b_n${N}.err
fi
