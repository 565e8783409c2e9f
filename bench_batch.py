#!/usr/bin/env python
"""bench_batch.py -- K planners: K sequential solve() calls against one batched MPPI_Batch / MPPI_StochasticBatch solve().

    python bench_batch.py --workload c2|c3|c4|c3m --batch K [--steps S] [--warmup W] [--profile] [--share-tdms]

K planners of the workload (bench.py's WORKLOADS, seeds 1..K: different maps, start poses and goals; num_opt = 1).
First one MPPI_Batch.solve() is checked against K solve() calls on identical twins, bit for bit (u, u_prev, costs,
weights, noise, the planners' and the TDMs' RNG states, the sampled maps); a mismatch exits non-zero.  Then a round of K
sequential solve() calls and one batch solve are timed, alternating (sequential, batched, sequential, batched): CUDA
events on the one stream all planners and the batch use, and the wall clock (each round ends in a host
synchronisation); solves/s, state-steps/s and kernel launches per round.  Prints one JSON line; writes nothing to the
tree (the library is built by build() beforehand).
c3 (stochastic, use_tdm) runs MPPI_StochasticBatch; its parity check also compares the per-(m, n) costs and the reach
box of every planner.  c3m is c3 with 2048 sampled maps (defined here): its CVaR runs the CTA kernel, one CTA per
control sequence, instead of the warp kernel.  --profile adds a torch.profiler split of one batched round's kernel time
into map sampler, rollout and the rest (a separate run after the timings).
--share-tdms: many planners on one terrain belief (multi-robot planning on one map).  The workload becomes seed 1's
map with K planners whose start poses, warm starts and goals come from seeds 1..K, and two legs on the same inputs: K
private TDM pairs of that map (the batch as without the option) and ONE pair shared by all K (share_tdms=True, sampled
once per solve).  The parity check holds every planner's state (and the TDMs' states and completed maps) byte for byte
between the legs; then rounds of the two legs alternate.  The JSON line adds the device bytes of each leg's TDM
allocations, computed from the shapes.
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

# config 3 with M 2048: above the warp CVaR kernel's 1024 maps
LOCAL_WORKLOADS = {"c3m": WORKLOADS["c3"][:2] + (2048,) + WORKLOADS["c3"][3:]}


def local_name_of(name):
    mode, N, M, T, H, res, B, da = LOCAL_WORKLOADS[name]
    return "%s: CVaR-cost MPPI N=%d M=%d T=%d, %dx%d PMF grid (%d bins, res %.1f m), num_opt=1 (config 3 with M %d)" % (
        name, N, M, T, H, H, B, res, M)


def shared_map_planners(E, scs, shared, cvar_alphas=None, device=0):
    """K planners on the map of scs[0] (its PMFs, masks and Config), planner k with the start pose, goal and warm start
    (sc["u0"], when the scenario has one) of scs[k] and, with cvar_alphas, cvar_alpha cvar_alphas[k % len]: on ONE TDM
    pair (shared) or each on a private pair of that map (the same PMF and seed, so the same generator states).  Also used
    by bench_trials.py --share-tdms."""
    sc0 = scs[0]
    cfg = E.Config(**sc0["cfg"])

    def pair():
        lin, ang = E.TDM_Numba(cfg, device=device), E.TDM_Numba(cfg, device=device)
        lin.set_TDM_from_PMF_grid(sc0["pmf_lin"], sc0["tdm_dict"], sc0["obstacle"], sc0["unknown"])
        ang.set_TDM_from_PMF_grid(sc0["pmf_ang"], sc0["tdm_dict"], sc0["obstacle"], sc0["unknown"])
        return lin, ang
    common = pair() if shared else None
    out = []
    for k, sc in enumerate(scs):
        lin, ang = common or pair()
        params = dict(sc0["params"], x0=sc["params"]["x0"].copy(), xgoal=np.array(sc["params"]["xgoal"], dtype=np.float64))
        if cvar_alphas:
            params["cvar_alpha"] = cvar_alphas[k % len(cvar_alphas)]
        pl = E.MPPI_Numba(cfg, device=device)
        pl.setup(params, lin, ang)
        if "u0" in sc:
            pl.u_cur_d.copy_to_device(sc["u0"])
        out.append(pl)
    return out


def tdm_bytes(planners):
    """Device bytes of the distinct TDMs of `planners`, from their shapes: the sampled maps (M, max rows, pitch), the two
    generator-state buffers, the PMF, its cumulative table and the obstacle / unknown masks."""
    seen, total = set(), 0
    for p in planners:
        for t in (p.lin_tdm, p.ang_tdm):
            if id(t) in seen:
                continue
            seen.add(id(t))
            Bn, rows, cols = (int(v) for v in t.pmf_grid_d.shape)
            M = int(t.sample_grid_batch_d.shape[0])
            rmax, cmax = (int(v) for v in t.cfg.max_map_dim)
            tx, ty = (int(v) for v in t.cfg.tdm_sample_thread_dim)
            total += (M * rmax * ((cmax + 15) // 16 * 16) + 2 * tx * ty * M * 16 + Bn * rows * cols
                      + rows * cols * ((Bn + 3) // 4 * 4) + 2 * rows * cols)
    return total


def gpu_info(dev):
    import torch
    gpu = {"name": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        gpu["power_limit_and_max_sm_clock"] = q
    except Exception as e:                               # noqa: BLE001
        gpu["power_limit_and_max_sm_clock"] = "unavailable (%r)" % e
    return gpu


def planner_state(p, stochastic):
    """Everything a solve writes into planner p (without the reach box, which a shared pair reports for its group)."""
    d = [p.u_cur_d, p.u_prev_d, p.costs_d, p.weights_d, p.noise_samples_d, p.rng_states_d]
    if stochastic:
        d.append(p.costs_nm_d)
    return [a.copy_to_host() for a in d]


def pair_state(p):
    return [a.copy_to_host() for a in (p.lin_tdm.rng_states_d, p.ang_tdm.rng_states_d, p.lin_tdm.sample_grid_batch_d,
                                       p.ang_tdm.sample_grid_batch_d)]


def same(xs, ys):
    return all(x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes() for x, y in zip(xs, ys))


def run_shared(args, emit):
    """--share-tdms: K planners on one map, K private TDM pairs against one shared pair."""
    import ctypes as C
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from mppi_numba_b200._lib import lib, check
    from tests.scenarios import make_scenario
    K = args.batch
    mode, N, M, T, H, res, B, da = LOCAL_WORKLOADS.get(args.workload) or WORKLOADS[args.workload]
    stochastic = mode == "tdm"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scs = [make_scenario(mode, N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=k + 1, det_alpha=da, warm_start=True)
           for k in range(K)]
    P = shared_map_planners(E, scs, False)                # private pairs
    Q = shared_map_planners(E, scs, True)                 # one shared pair
    stream = torch.cuda.Stream(device=dev)
    for p in P + Q:
        check(lib.b200mppi_planner_set_stream(p._handle, C.c_void_p(stream.cuda_stream)))
    Batch = E.MPPI_StochasticBatch if stochastic else E.MPPI_Batch
    bp, bq = Batch(P), Batch(Q, share_tdms=True)
    bp.set_stream(stream.cuda_stream)
    bq.set_stream(stream.cuda_stream)
    start = [same(pair_state(p), pair_state(q)) for p, q in zip(P, Q)]

    # ---- parity: one solve of each leg, every planner byte for byte, the shared pair as every private one
    up, uq = bp.solve(), bq.solve()
    same_u = bool(np.array_equal(up, uq))
    same_state = all(same(planner_state(p, stochastic), planner_state(q, stochastic)) for p, q in zip(P, Q))
    same_pairs = all(same(pair_state(p), pair_state(q)) for p, q in zip(P, Q))
    parity = {"passed": bool(all(start) and same_u and same_state and same_pairs), "same_start": bool(all(start)),
              "u_bitwise": same_u, "state_bitwise": same_state, "tdm_states_and_maps_bitwise": same_pairs,
              "planners": K, "against": "the same planners on K private TDM pairs of the map (u, u_prev, costs, "
                                        "weights, noise, RNG states; the TDMs' RNG states and completed maps)"}
    if not parity["passed"]:
        sys.stderr.write("bench_batch.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        emit(json.dumps({"metric": "batched solves on one map", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    legs = (("private", bp), ("shared", bq))
    for _ in range(max(args.warmup, 3)):
        for _, b in legs:
            b.solve()
    res = {name: [] for name, _ in legs}
    launches = {}
    for _ in range(2):                                    # alternate: private, shared, private, shared
        for name, b in legs:
            l0 = b.launch_count()
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            t0 = time.perf_counter()
            for _ in range(args.steps):
                b.solve()
            wall = (time.perf_counter() - t0) / args.steps
            e1.record(stream)
            torch.cuda.synchronize(dev)
            launches[name] = (b.launch_count() - l0) / args.steps
            res[name].append((e0.elapsed_time(e1) / args.steps, wall * 1e3))

    def summary(name, planners):
        ev = float(np.median([r[0] for r in res[name]]))
        wall = float(np.median([r[1] for r in res[name]]))
        return {"ms_per_round_events": ev, "ms_per_round_wall": wall,
                "ms_per_round_events_runs": [r[0] for r in res[name]], "ms_per_round_wall_runs": [r[1] for r in res[name]],
                "solves_per_s": K / (wall * 1e-3), "kernel_launches_per_round": launches[name],
                "tdm_device_bytes": tdm_bytes(planners)}
    pri, sha = summary("private", P), summary("shared", Q)
    name = local_name_of(args.workload) if args.workload in LOCAL_WORKLOADS else workload_name_of(args.workload)
    out = {"metric": "batched solves of K planners on one map: K private TDM pairs vs one shared pair",
           "unit": "solves/s", "value": sha["solves_per_s"], "higher_is_better": True,
           "config": {"workload": name, "batch": K,
                      "planners": "seed 1's map; start poses, goals and warm starts of seeds 1..K; num_opt=1"},
           "steps": args.steps, "warmup": args.warmup, "gpu": gpu_info(dev), "parity_check": parity,
           "private": pri, "shared": sha,
           "speedup_wall": pri["ms_per_round_wall"] / sha["ms_per_round_wall"],
           "speedup_events": pri["ms_per_round_events"] / sha["ms_per_round_events"]}
    if args.profile:
        out["profile_private_round"] = profile_round(bp.solve, dev, stream)
        out["profile_shared_round"] = profile_round(bq.solve, dev, stream)
    emit(json.dumps(out))


def run(args, emit):
    import ctypes as C
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from mppi_numba_b200._lib import lib, check
    from tests.scenarios import make_scenario
    K = args.batch
    mode, N, M, T, H, res, B, da = LOCAL_WORKLOADS.get(args.workload) or WORKLOADS[args.workload]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scs = [make_scenario(mode, N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=k + 1, det_alpha=da) for k in range(K)]
    A, S = [[make_planner(E, sc, 0)[3] for sc in scs] for _ in range(2)]     # A: batched, S: one solve() at a time
    stream = torch.cuda.Stream(device=dev)
    for p in A + S:
        check(lib.b200mppi_planner_set_stream(p._handle, C.c_void_p(stream.cuda_stream)))
    stochastic = mode == "tdm"
    batch = E.MPPI_StochasticBatch(A) if stochastic else E.MPPI_Batch(A)
    batch.set_stream(stream.cuda_stream)

    def state(p):
        d = [p.u_cur_d, p.u_prev_d, p.costs_d, p.weights_d, p.noise_samples_d, p.rng_states_d, p.lin_tdm.rng_states_d,
             p.ang_tdm.rng_states_d, p.lin_tdm.sample_grid_batch_d, p.ang_tdm.sample_grid_batch_d]
        if stochastic:
            d.append(p.costs_nm_d)
            return [np.asarray(p.sample_box())] + [a.copy_to_host() for a in d]
        return [a.copy_to_host() for a in d]

    # ---- parity: one batch solve == K sequential solves, bit for bit
    ub = batch.solve()
    us = np.stack([p.solve() for p in S])
    same_u = bool(np.array_equal(ub, us))
    same_state = all(all(np.array_equal(x, y) for x, y in zip(state(a), state(s))) for a, s in zip(A, S))
    parity = {"passed": same_u and same_state, "u_bitwise": same_u, "state_bitwise": same_state, "planners": K,
              "against": "K solve() calls on identical twins (u, u_prev, costs, weights, noise, RNG states, sampled maps)"}
    if stochastic:
        parity["against"] = ("K solve() calls on identical twins (u, u_prev, costs, per-(m, n) costs, weights, noise, RNG "
                             "states, sampled maps, reach box)")
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
    out = {"metric": "batched one-map solves: K sequential solve() calls vs one MPPI_Batch.solve()",
                     "unit": "solves/s", "value": bat["solves_per_s"], "higher_is_better": True,
                     "config": {"workload": (local_name_of(args.workload) if args.workload in LOCAL_WORKLOADS else
                                             workload_name_of(args.workload)), "batch": K,
                                "planners": "seeds 1..K (different maps, start poses and goals), num_opt=1"},
                     "steps": args.steps, "warmup": args.warmup, "gpu": gpu, "parity_check": parity,
                     "sequential": seq, "batched": bat,
                     "speedup_wall": seq["ms_per_round_wall"] / bat["ms_per_round_wall"],
                     "speedup_events": seq["ms_per_round_events"] / bat["ms_per_round_events"]}
    if stochastic:
        out["metric"] = "batched stochastic solves: K sequential solve() calls vs one MPPI_StochasticBatch.solve()"
        out["config"]["planners"] = "seeds 1..K (different maps, start poses and goals), use_tdm, num_opt=1"
    if args.profile:
        out["profile_batched_round"] = profile_round(batch_round, dev, stream)
    emit(json.dumps(out))


def profile_round(fn, dev, stream, rounds=5):
    """Kernel time per batched round by group (torch.profiler, CUDA activities), over `rounds` rounds."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize(dev)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            fn()
        torch.cuda.synchronize(dev)
    groups = {"sampler": 0.0, "rollout": 0.0, "rest": 0.0}
    kernels = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or "memcpy" in ev.name.lower() or "memset" in ev.name.lower():
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        name = ev.name
        g = "sampler" if ("sample_grids" in name or "advance_states" in name) else (
            "rollout" if "rollout_win" in name else "rest")
        groups[g] += us
        short = name.split("(")[0][-60:]
        kernels[short] = kernels.get(short, 0.0) + us
    return {"kernel_ms_per_round": {k: v / rounds / 1e3 for k, v in groups.items()},
            "kernel_ms_per_round_by_kernel": {k: v / rounds / 1e3 for k, v in sorted(kernels.items())},
            "rounds": rounds}


def main():
    # one JSON line on stdout: everything else (the engine's allocation notices, ...) goes to stderr
    real_stdout = os.dup(1)
    os.dup2(2, 1)
    sys.stdout = os.fdopen(os.dup(2), "w", buffering=1)

    def emit(line):
        os.write(real_stdout, (line + "\n").encode())
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[1])
    ap.add_argument("--workload", default="c2", choices=["c2", "c3", "c4", "c3m"])
    ap.add_argument("--batch", type=int, default=64, metavar="K", help="planners in the batch")
    ap.add_argument("--steps", type=int, default=20, help="timed rounds per measurement")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="add a torch.profiler kernel-time split of a batched round")
    ap.add_argument("--share-tdms", action="store_true",
                    help="K planners on one map: K private TDM pairs against one pair shared by all (share_tdms=True)")
    args = ap.parse_args()
    if args.batch < 1 or args.steps < 1:
        ap.error("--batch and --steps must be at least 1")
    (run_shared if args.share_tdms else run)(args, emit)


if __name__ == "__main__":
    main()
