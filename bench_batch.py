#!/usr/bin/env python
"""bench_batch.py -- K one-map planners: K sequential solve() calls against one batched MPPI_Batch.solve().

    python bench_batch.py --workload c2|c4 --batch K [--steps S] [--warmup W]

K planners of the workload (bench.py's WORKLOADS, seeds 1..K: different maps, start poses and goals; num_opt = 1).
First one MPPI_Batch.solve() is checked against K solve() calls on identical twins, bit for bit (u, u_prev, costs,
weights, noise, the planners' and the TDMs' RNG states, the sampled maps); a mismatch exits non-zero.  Then a round of K
sequential solve() calls and one batch solve are timed, alternating (sequential, batched, sequential, batched): CUDA
events on the one stream all planners and the batch use, and the wall clock (each round ends in a host
synchronisation); solves/s, state-steps/s and kernel launches per round.  Prints one JSON line; writes nothing to the
tree (the library is built by build() beforehand).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import WORKLOADS, make_planner, workload_name_of   # noqa: E402


def run(args, emit):
    import ctypes as C
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from mppi_numba_b200._lib import lib, check
    from tests.scenarios import make_scenario
    K = args.batch
    mode, N, M, T, H, res, B, da = WORKLOADS[args.workload]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scs = [make_scenario(mode, N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=k + 1, det_alpha=da) for k in range(K)]
    A, S = [[make_planner(E, sc, 0)[3] for sc in scs] for _ in range(2)]     # A: batched, S: one solve() at a time
    stream = torch.cuda.Stream(device=dev)
    for p in A + S:
        check(lib.b200mppi_planner_set_stream(p._handle, C.c_void_p(stream.cuda_stream)))
    batch = E.MPPI_Batch(A)
    batch.set_stream(stream.cuda_stream)

    def state(p):
        d = [p.u_cur_d, p.u_prev_d, p.costs_d, p.weights_d, p.noise_samples_d, p.rng_states_d, p.lin_tdm.rng_states_d,
             p.ang_tdm.rng_states_d, p.lin_tdm.sample_grid_batch_d, p.ang_tdm.sample_grid_batch_d]
        return [a.copy_to_host() for a in d]

    # ---- parity: one batch solve == K sequential solves, bit for bit
    ub = batch.solve()
    us = np.stack([p.solve() for p in S])
    same_u = bool(np.array_equal(ub, us))
    same_state = all(all(np.array_equal(x, y) for x, y in zip(state(a), state(s))) for a, s in zip(A, S))
    parity = {"passed": same_u and same_state, "u_bitwise": same_u, "state_bitwise": same_state, "planners": K,
              "against": "K solve() calls on identical twins (u, u_prev, costs, weights, noise, RNG states, sampled maps)"}
    if not parity["passed"]:
        sys.stderr.write("bench_batch.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        emit(json.dumps({"metric": "batched one-map solves", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    def seq_round():
        for p in S:
            p.solve()

    def batch_round():
        batch.solve()

    for _ in range(max(args.warmup, 3)):                  # warm up both paths, then keep the GPU busy ~0.3 s
        seq_round()
        batch_round()
    t_w = time.perf_counter()
    while time.perf_counter() - t_w < 0.3:
        batch_round()
    res = {"sequential": [], "batched": []}
    launches = {}

    def count(name):
        return sum(p.launch_count() for p in S) if name == "sequential" else batch.launch_count()
    for _ in range(2):                                    # alternate: sequential, batched, sequential, batched
        for name, fn in (("sequential", seq_round), ("batched", batch_round)):
            l0 = count(name)
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            t0 = time.perf_counter()
            for _ in range(args.steps):
                fn()
            wall = (time.perf_counter() - t0) / args.steps
            e1.record(stream)
            torch.cuda.synchronize(dev)
            launches[name] = (count(name) - l0) / args.steps
            res[name].append((e0.elapsed_time(e1) / args.steps, wall * 1e3))

    def summary(name):
        ev = float(np.median([r[0] for r in res[name]]))
        wall = float(np.median([r[1] for r in res[name]]))
        return {"ms_per_round_events": ev, "ms_per_round_wall": wall,
                "ms_per_round_events_runs": [r[0] for r in res[name]], "ms_per_round_wall_runs": [r[1] for r in res[name]],
                "solves_per_s": K / (wall * 1e-3), "state_steps_per_s": K * N * T / (wall * 1e-3),
                "kernel_launches_per_round": launches[name]}
    seq, bat = summary("sequential"), summary("batched")
    gpu = {"name": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        gpu["power_limit_and_max_sm_clock"] = q
    except Exception as e:                               # noqa: BLE001
        gpu["power_limit_and_max_sm_clock"] = "unavailable (%r)" % e
    emit(json.dumps({"metric": "batched one-map solves: K sequential solve() calls vs one MPPI_Batch.solve()",
                     "unit": "solves/s", "value": bat["solves_per_s"], "higher_is_better": True,
                     "config": {"workload": workload_name_of(args.workload), "batch": K,
                                "planners": "seeds 1..K (different maps, start poses and goals), num_opt=1"},
                     "steps": args.steps, "warmup": args.warmup, "gpu": gpu, "parity_check": parity,
                     "sequential": seq, "batched": bat,
                     "speedup_wall": seq["ms_per_round_wall"] / bat["ms_per_round_wall"],
                     "speedup_events": seq["ms_per_round_events"] / bat["ms_per_round_events"]}))


def main():
    # one JSON line on stdout: everything else (the engine's allocation notices, ...) goes to stderr
    real_stdout = os.dup(1)
    os.dup2(2, 1)
    sys.stdout = os.fdopen(os.dup(2), "w", buffering=1)

    def emit(line):
        os.write(real_stdout, (line + "\n").encode())
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[1])
    ap.add_argument("--workload", default="c2", choices=["c2", "c4"])
    ap.add_argument("--batch", type=int, default=64, metavar="K", help="planners in the batch")
    ap.add_argument("--steps", type=int, default=20, help="timed rounds per measurement")
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.batch < 1 or args.steps < 1:
        ap.error("--batch and --steps must be at least 1")
    run(args, emit)


if __name__ == "__main__":
    main()
