#!/bin/bash
# A/B on one machine (the spread between machines is larger than the differences of interest): library variants built beforehand into mppi_numba_b200/ab/lib_<name>.so
# (e.g. B200MPPI_NVCC_FLAGS=-DWIN_ROUND_FP64=0 python mppi_numba_b200/build.py --force; cp mppi_numba_b200/libb200mppi.so
# mppi_numba_b200/ab/lib_intround.so), each timed twice, interleaved: bench stage times + one rank of 8 / 4 alone.
#   tools/ab_libs.sh <name> <name> ...
b() { python bench.py --steps 30 --warmup 5 --no-numba --no-others 2>/dev/null | python -c "
import json,sys
for l in sys.stdin:
    if l.startswith('{'):
        d=json.loads(l); print(d['ms_per_step'], d['roofline'].get('stage_ms'), d.get('clocks'))"; }
for L in "$@" "$@"; do
  cp mppi_numba_b200/ab/lib_$L.so mppi_numba_b200/libb200mppi.so
  echo "== $L"; b
  for u in 0 1; do echo "-- unit $u"; B200MPPI_WIN_UNIT=$u python tools/rank_stage_times.py c5 8 4 2>&1 | tail -4; done
done
