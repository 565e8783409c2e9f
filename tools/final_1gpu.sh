#!/bin/bash
# One-GPU evidence run: GPU test suite, bench line, A/B of the reach box, ncu launch list + full capture.
# usage: tools/final_1gpu.sh <tag>      -> runs/<tag>_*
tag=${1:-r02}
mkdir -p runs
python -m pytest tests -q -m gpu 2>&1 | tail -8 | tee runs/${tag}_pytest_gpu.txt
python bench.py --steps 20 --warmup 5 > runs/${tag}_bench_1gpu.json 2> runs/${tag}_bench_1gpu.err
tail -c 300 runs/${tag}_bench_1gpu.json; echo
B200MPPI_SAMPLE_BOX=off python bench.py --steps 20 --warmup 5 --no-cpu --no-numba --no-others > runs/${tag}_bench_1gpu_wholemaps.json 2>/dev/null
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -s 24 -c 24 --csv --log-file runs/${tag}_launches.csv python tools/ncu_target.py c5 8 > /dev/null 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:"rollout_win|sample_grids_v2|noise_prepare|update_partial|cvar|advance" -s 12 -c 12 -o runs/prof_${tag} -f python tools/ncu_target.py c5 4 > runs/${tag}_ncu.log 2>&1
tail -2 runs/${tag}_ncu.log
