#!/bin/bash
# Multi-GPU evidence run on a machine with N GPUs: bench at every G <= N given on the command line.
# usage: tools/final_multi.sh <tag> 2 4 8
tag=$1; shift
mkdir -p runs
for g in "$@"; do
  python -m torch.distributed.run --nnodes=1 --nproc-per-node $g --master-addr 127.0.0.1 --master-port $((29500 + g)) bench.py --gpus $g --steps 20 --warmup 5 > runs/${tag}_bench_g${g}.json 2> runs/${tag}_bench_g${g}.err
  echo "G=$g rc=$?"; tail -c 1800 runs/${tag}_bench_g${g}.json; echo; tail -3 runs/${tag}_bench_g${g}.err
done
