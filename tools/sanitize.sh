#!/bin/bash
# compute-sanitizer over smoke() and a stochastic-mode solve (boxed sampler, state advance, fused noise + controls, TMA
# windowed rollout, CVaR, fused update): memcheck, racecheck, synccheck.   usage: tools/sanitize.sh <tag>   -> runs/<tag>_compute_sanitizer.md
tag=${1:-r02}
mkdir -p runs
out=runs/${tag}_compute_sanitizer.md
echo "# compute-sanitizer, smoke() and two solves of bench workload c3 (N 1024, M 64, T 64, stochastic mode)" > $out
for tool in memcheck racecheck synccheck; do
  for target in "-c 'import __graft_entry__ as g; g.smoke()'" "tools/ncu_target.py c3 2"; do
    echo -e "\n## $tool: python $target\n\`\`\`" >> $out
    eval timeout 600 compute-sanitizer --tool $tool python $target 2>&1 | grep -v "^MPPI planner\|^TDM has" | tail -6 >> $out
    echo '```' >> $out
  done
done
cat $out
