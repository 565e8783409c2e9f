"""The reference benchmark's method comparison in one call: MPPI_MixedBatch.run_trial_sequences against the three
per-kind calls it replaces.

The reference benchmark (benchmark.ipynb) runs, per environment, its methods noisy_dyn (use_tdm, CVaR cost),
risk_dyn (use_det_dynamics) and nom_dyn_risk_cost (use_nom_dynamics_with_speed_map) at five alphas each, over the same
ground-truth realisations.  This script builds that sweep at the reference's shape (bench_trials.py's ``ref``: N 1024,
M 1024, T 100, 9 x 9-cell maps at 1 m): per environment, for each alpha of BENCH_ALPHAS,
  noisy_dyn at cvar_alpha alpha on the environment's one shared TDM pair,
  risk_dyn at alpha_dyn alpha and nom_dyn_risk_cost at alpha_dyn alpha, each on its own collapsed pair,
and runs every planner through the same R realisations back to back (reset_x0=False, the benchmark's loop, max_steps
150).

1. Parity: the mixed call on one set of planners against the three per-kind calls (MPPI_Batch of the risk_dyn planners,
   MPPI_Batch of the nom_dyn_risk_cost planners, MPPI_StochasticBatch of the noisy_dyn planners, share_tdms on) on
   identical twins: every output, every planner's buffers and every TDM pair, bit for bit.  A failure exits 3.
2. Rounds alternate one mixed call with the three per-kind calls in sequence, each from the same start (x0 and warm
   start reset; the RNG streams run on).
Prints one JSON line: seconds per round of each leg (min, median, max), launches per round, and the GPU's name, power
limit and maximum SM clock, read in the same run.  Writes nothing to the tree.

    python bench_methods.py [--envs 8] [--realisations 3] [--rounds 5]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import make_planner                       # noqa: E402
from bench_trials import BENCH_ALPHAS, LOCAL_WORKLOADS, _quiet   # noqa: E402

MAX_STEPS = 150
METHODS = ("noisy_dyn", "risk_dyn", "nom_dyn_risk_cost")
MODES = {"noisy_dyn": "tdm", "risk_dyn": "det", "nom_dyn_risk_cost": "spd"}


def build(E, n_env):
    """(planners, method of each, environment of each, starting (x0, u0) of each): per environment the noisy_dyn sweep
    on one shared pair, then the risk_dyn and nom_dyn_risk_cost sweeps on private collapsed pairs."""
    from bench_batch import shared_map_planners
    from tests.scenarios import make_scenario
    _, N, M, T, H, res, B, _ = LOCAL_WORKLOADS["ref"]
    pls, methods, envs, starts = [], [], [], []
    for e in range(n_env):
        base = make_scenario("tdm", N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=e + 1, warm_start=True)
        base["params"]["xgoal"] = base["params"]["x0"][:2] + np.array([3.0, 2.5])
        noisy = shared_map_planners(E, [base] * len(BENCH_ALPHAS), True, BENCH_ALPHAS)
        pls += noisy
        methods += ["noisy_dyn"] * len(noisy)
        for method in ("risk_dyn", "nom_dyn_risk_cost"):
            for a in BENCH_ALPHAS:
                sc = make_scenario(MODES[method], N=N, M=1, T=T, H=H, W=H, res=res, B=B, seed=e + 1, det_alpha=a,
                                   warm_start=True)
                sc["params"]["x0"], sc["params"]["xgoal"] = base["params"]["x0"].copy(), base["params"]["xgoal"].copy()
                pls.append(make_planner(E, sc, 0)[3])
                methods.append(method)
        envs += [e] * (len(pls) - len(envs))
    for p in pls:
        starts.append((np.array(p.params["x0"], dtype=np.float64), p.u_cur_d.copy_to_host()))
    return pls, methods, envs, starts


def reset(pls, starts):
    for p, (x0, u0) in zip(pls, starts):
        p.params["x0"] = x0.copy()
        p.u_cur_d.copy_to_device(u0)


def per_kind_batches(E, pls, methods):
    """[(indices, batch)] of the three per-kind calls."""
    out = []
    for m in METHODS:
        idx = [i for i, x in enumerate(methods) if x == m]
        cls = E.MPPI_StochasticBatch if MODES[m] == "tdm" else E.MPPI_Batch
        out.append((idx, cls([pls[i] for i in idx], share_tdms=True)))
    return out


def stats(xs):
    return {"min": float(np.min(xs)), "median": float(np.median(xs)), "max": float(np.max(xs))}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--envs", type=int, default=8)
    ap.add_argument("--realisations", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from bench_batch import gpu_info, pair_state, planner_state, same
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _, _, _, _, H, res, _, _ = LOCAL_WORKLOADS["ref"]
    with _quiet():
        A, methods, envs, starts = build(E, args.envs)
        B, _, _, _ = build(E, args.envs)
    rng = np.random.default_rng(11)
    real = [[E.TractionGrid(rng.uniform(0.3, 1.0, (H, H)), rng.uniform(0.3, 1.0, (H, H)), res=res)
             for _ in range(args.realisations)] for _ in range(args.envs)]
    seqs = [real[e] for e in envs]                    # every planner of an environment on its realisations
    mixed = E.MPPI_MixedBatch(A, share_tdms=True)
    kinds = per_kind_batches(E, B, methods)

    def mixed_round():
        reset(A, starts)
        n0 = mixed.launch_count()
        t0 = time.perf_counter()
        out = mixed.run_trial_sequences(seqs, MAX_STEPS)
        torch.cuda.synchronize(dev)
        return time.perf_counter() - t0, mixed.launch_count() - n0, out

    def kinds_round():
        reset(B, starts)
        n0 = sum(b.launch_count() for _, b in kinds)
        t0 = time.perf_counter()
        outs = [(idx, b.run_trial_sequences([seqs[i] for i in idx], MAX_STEPS)) for idx, b in kinds]
        torch.cuda.synchronize(dev)
        return time.perf_counter() - t0, sum(b.launch_count() for _, b in kinds) - n0, outs

    # ---- parity: one round of each on the twins, from the same start
    with _quiet():
        _, _, om = mixed_round()
        _, _, ok = kinds_round()
    ok_out = True
    for idx, o in ok:
        for j, i in enumerate(idx):
            for key in ("xhist", "uhist", "steps", "episodes_run"):
                ok_out &= bool(np.asarray(om[key][i]).tobytes() == np.asarray(o[key][j]).tobytes())
            ok_out &= om["status"][i] == o["status"][j]
    ok_state = all(same(planner_state(a, m == "noisy_dyn") + [a.params["x0"]],
                        planner_state(b, m == "noisy_dyn") + [b.params["x0"]]) for a, b, m in zip(A, B, methods))
    ok_pair = all(same(pair_state(a), pair_state(b)) for a, b in zip(A, B))
    parity = {"passed": bool(ok_out and ok_state and ok_pair), "outputs_bitwise": ok_out, "state_bitwise": ok_state,
              "tdm_pairs_bitwise": ok_pair, "planners": len(A), "steps_per_method": {
                  m: int(sum(om["steps"][i].sum() for i in range(len(A)) if methods[i] == m)) for m in METHODS},
              "against": "MPPI_Batch (risk_dyn), MPPI_Batch (nom_dyn_risk_cost) and MPPI_StochasticBatch (noisy_dyn) "
                         "run_trial_sequences on identical twins"}
    if not parity["passed"]:
        sys.stderr.write("bench_methods.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        print(json.dumps({"metric": "method comparison", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    # ---- timed rounds, alternating
    tm, tk, lm, lk = [], [], [], []
    with _quiet():
        for _ in range(args.rounds):
            t, n, _ = mixed_round()
            tm.append(t)
            lm.append(n)
            t, n, _ = kinds_round()
            tk.append(t)
            lk.append(n)
    print(json.dumps({
        "metric": "method comparison: run_trial_sequences of noisy_dyn, risk_dyn and nom_dyn_risk_cost",
        "workload": {"envs": args.envs, "alphas": BENCH_ALPHAS, "planners": len(A), "realisations": args.realisations,
                     "max_steps": MAX_STEPS, "N": LOCAL_WORKLOADS["ref"][1], "M": LOCAL_WORKLOADS["ref"][2],
                     "T": LOCAL_WORKLOADS["ref"][3], "map_cells": H},
        "seconds_per_round": {"mixed": stats(tm), "per_kind": stats(tk)},
        "speedup_median": float(np.median(tk) / np.median(tm)),
        "launches_per_round": {"mixed": int(np.median(lm)), "per_kind": int(np.median(lk))},
        "rounds": args.rounds, "gpu": gpu_info(dev), "parity_check": parity}))


if __name__ == "__main__":
    main()
