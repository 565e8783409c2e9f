#!/usr/bin/env python
"""bench_trials.py -- closed-loop episodes of K planners: the host-driven loop against the batch's device episodes.

    python bench_trials.py --workload c2|c4|c3|ref|refm|gif|mix|bb --batch K --closed-loop S [--rounds R] [--profile]
                           [--record-every n] [--share-tdms] [--episodes E [--device-grids]]

c2 and c4 are one-map workloads (MPPI_Batch.run_trials); c3 and ref are stochastic (use_tdm, CVaR cost:
MPPI_StochasticBatch.run_stochastic_trials).  ref is the reference benchmark's noisy_dyn trial shape (N 1024, M 1024,
T 100, a 9 x 9-cell map at 1 m), defined here: every reach box leaves that map, so every step samples whole maps.
refm is ref with 2048 sampled maps: a less noisy tail estimate, whose CVaR runs the CTA kernel.  bb is the barebone
notebook's map-free loop (MPPI_Batch.run_barebone_trials, run_bb below), whose parity check also holds the obstacle
contact counts against numpy's rule on the device's trajectory.  gif is the shape of the reference's GIF notebook
(use_tdm, N 1024, M 1024, T 100, 100 visualisation rollouts, a 12 x 6-cell map at 1 m), whose loop draws every step.
mix is c3's N, M and T with planner k on a map of MIX_SIZES[k % 3] cells a side at c3's resolution and MIX_BINS[k % 2]
bins: six map geometries in two launch classes (the bins pad to 12 and 8), one run_stochastic_trials call for all.  Its
rounds add a third leg, "device_per_geometry": one run_stochastic_trials call per map geometry, one after the other,
the only way to run such planners before trials took several launch classes.

K planners of the workload (bench.py's WORKLOADS, seeds 1..K: different maps, start poses and warm starts), each with
a seeded ground-truth TractionGrid over its map; every other planner has its goal 1.5 m away (reached within S steps),
the others the workload's distant goal (they run all S steps).  First the parity check: run_trials on one set of
planners, and on identical twins the host loop replayed with the device's trajectory -- u[0] of every solve and the
final planner state (u, u_prev, noise, costs, weights, RNG states, sampled maps, params['x0']) bit for bit; a mismatch
exits non-zero.  Then R rounds of each, alternating, every round from the same start (params, warm start):
  host: the best host loop available -- the batch's solve() of all K, then per running planner a numpy plant step and
        shift_and_update, until every planner has stopped;
  device: one run_trials(grids, S) (run_stochastic_trials for c3, ref and refm).
Wall clock per round (each ends in a host synchronisation); control steps/s (planner-steps run), episodes/s, kernel
launches per round.  Prints one JSON line with the card's name and power limit; writes nothing to the tree.
--record-every n (not bb): the notebooks' drawing loop, get_state_rollout() at every n-th step after solve() and before
shift_and_update.  The parity check also holds the device's records (run_trials(..., record_every=n)) against the
replayed host loop's get_state_rollout(), bit for bit; the host rounds call it; and device rounds with recording are
timed alternately with those without.  --profile then profiles a recording round and reports the share of the
visualisation and map-completion kernels.
--share-tdms (not bb): many planners on one terrain belief.  The workload becomes seed 1's map with K planners whose
start poses, warm starts and goals come from seeds 1..K (for ref and refm the planners also cycle cvar_alpha through the
reference benchmark's [1.0, 0.8, 0.6, 0.4, 0.2]: its noisy_dyn sweep on one environment), and two legs of device
episodes on the same inputs: K private TDM pairs of that map and ONE pair shared by all K (share_tdms=True: sampled once
per step while any planner runs).  The parity check holds the histories, steps, statuses (and records), every
planner's state and the shared pair against the longest-running planner's private pair, byte for byte; then rounds of
the two legs alternate.  The JSON line adds the device bytes of each leg's TDM allocations, computed from the shapes.
--episodes E (c2, c3, ref; with or without --share-tdms): the reference benchmark's loop over trials_per_env = E
ground-truth realisations on the same planners (run_episodes below).  Each planner gets E seeded grids.  The parity check
runs run_trial_sequences (no reset: the benchmark's loop) and replays the host sequence loop with the device's trajectory
on twins, each on a private TDM pair: u[0] of every solve and every planner's final state bit for bit (with
--share-tdms, the shared pair against the private pair of the planner that ran the most steps).  Then rounds of three
legs, all with params['x0'] set back to the start before each episode: "sequence", one run_trial_sequences(...,
reset_x0=True) call; "calls", E run_trials calls, each running until its slowest planner stops (without --share-tdms
its histories must equal the sequence's, bit for bit, or the run fails); "host", the host loop over the E episodes.
--device-grids (with --episodes E; c4, ref): the E realisations every planner runs are drawn from a ground-truth use_tdm
pair of the workload's map geometry and M (run_device_grids below), as the reference's real-world evaluation does.  The
parity check holds draw_traction_grids against the notebook's sample_traction_grid on a twin pair (every plane bit for
bit), then one run_trial_sequences(..., reset_x0=True) on the device set against the same call with the helper's host
grids on twin planners (histories, steps, statuses and every planner's state bit for bit).  Then rounds of two legs,
alternating: "host_grids" (the helper's grids, uploaded by each call) and "device_grids" (one shared set, read in
place); then the draw itself against the helper's sample, copy and convert.  The JSON line adds the grid bytes each call
uploads, computed from the shapes.
--episodes E --record-every n (c3, ref, gif) and --workload bb --episodes E [--record-every n]: recorded and barebone
trial sequences (run_recorded_episodes below).  The parity check runs the benchmark's loop (no reset) with recording
and replays the host sequence loop on twins with the device's trajectory, calling get_state_rollout() at each episode's
steps t % n == 0: u[0], every record (NaN where nothing was recorded), bb's contact counts per episode and every
planner's final state (state_rollout_batch_d included), bit for bit.  Then rounds of the legs, alternating, all with
reset_x0: "recorded" (one recorded sequence call), "unrecorded" (the same call without recording, on twins; with
--record-every) and "host" (the drawing host loop: the batch's solve() and, at recorded steps, get_state_rollout()).
"""
import argparse
import functools
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

# the reference benchmark's noisy_dyn trial: N 1024, M 1024, T 100 on a 9 x 9-cell map at 1 m (c3's bins)
LOCAL_WORKLOADS = {"ref": ("tdm", 1024, 1024, 100, 9, 1.0) + tuple(WORKLOADS["c3"][6:]),
                   "refm": ("tdm", 1024, 2048, 100, 9, 1.0) + tuple(WORKLOADS["c3"][6:]),
                   "gif": ("tdm", 1024, 1024, 100, 6, 1.0) + tuple(WORKLOADS["c3"][6:]),
                   "mix": WORKLOADS["c3"]}
# mix: planner k's map size (cells a side) and bin count
MIX_SIZES = [512, 384, 256]
MIX_BINS = [12, 8]
# the GIF notebook's map is 12 cells wide and 6 high, and it draws 100 rollouts; elsewhere square maps, the scenario's V
MAP_WIDTH = {"gif": 12}
VIS_ROLLOUTS = {"gif": 100}


def run(args, emit):
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from tests.scenarios import make_scenario
    from tests.trial_loop import plant_step, within
    K, S = args.batch, args.closed_loop
    mode, N, M, T, H, res, B, da = LOCAL_WORKLOADS.get(args.workload) or WORKLOADS[args.workload]
    stochastic = mode == "tdm"
    Batch = E.MPPI_StochasticBatch if stochastic else E.MPPI_Batch
    trials = ((lambda b, g, s, **kw: b.run_stochastic_trials(g, s, **kw)) if stochastic else
              (lambda b, g, s, **kw: b.run_trials(g, s, **kw)))
    W, every = MAP_WIDTH.get(args.workload, H), args.record_every
    mix = args.workload == "mix"
    shape = [(MIX_SIZES[k % 3], MIX_SIZES[k % 3], MIX_BINS[k % 2]) if mix else (H, W, B) for k in range(K)]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scs = []
    for k in range(K):
        Hk, Wk, Bk = shape[k]
        sc = make_scenario(mode, N=N, M=M, T=T, H=Hk, W=Wk, res=res, B=Bk, seed=k + 1, det_alpha=da, warm_start=True)
        if args.workload in VIS_ROLLOUTS:
            sc["cfg"]["num_vis_state_rollouts"] = VIS_ROLLOUTS[args.workload]
        if k % 2 == 0:
            sc["params"]["xgoal"] = sc["params"]["x0"][:2] + np.array([1.2, -0.9])
        scs.append(sc)
    rng = np.random.default_rng(7)
    grids = [E.TractionGrid(rng.uniform(0.3, 1.0, shape[k][:2]), rng.uniform(0.3, 1.0, shape[k][:2]), res=res)
             for k in range(K)]
    A, Bs = [[make_planner(E, sc, 0)[3] for sc in scs] for _ in range(2)]

    def reset(pls):
        for p, sc in zip(pls, scs):
            p.params["x0"] = sc["params"]["x0"].copy()
            p.u_cur_d.copy_to_device(sc["u0"])

    reset(A), reset(Bs)
    ba, bb = Batch(A), Batch(Bs)

    # ---- parity: the device episodes == the host loop replayed with the device's trajectory
    out = trials(ba, grids, S, **({} if every is None else dict(record_every=every)))
    ok_u = ok_rec = True
    for k, p in enumerate(Bs):
        one = Batch([p])
        n = int(out["steps"][k])
        for t in range(n):
            useq = one.solve()[0]
            ok_u &= bool(np.array_equal(useq[0], out["uhist"][k, t]))
            if every is not None and t % every == 0:
                ok_rec &= p.get_state_rollout().tobytes() == out["state_rollouts"][k, t // every].tobytes()
            p.shift_and_update(out["xhist"][k, t + 1], useq, 1)
        if every is not None:
            ok_rec &= bool(np.isnan(out["state_rollouts"][k, -(-n // every):]).all())

    def state(p):
        d = [p.u_cur_d, p.u_prev_d, p.costs_d, p.weights_d, p.noise_samples_d, p.rng_states_d, p.lin_tdm.rng_states_d,
             p.ang_tdm.rng_states_d, p.lin_tdm.sample_grid_batch_d, p.ang_tdm.sample_grid_batch_d]
        if stochastic:
            d.append(p.costs_nm_d)
        return [a.copy_to_host() for a in d] + [p.params["x0"], np.asarray(p.sample_box())]
    ok_state = all(all(np.array_equal(x, y) for x, y in zip(state(a), state(b))) for a, b in zip(A, Bs))
    parity = {"passed": bool(ok_u and ok_state and ok_rec), "u_bitwise": ok_u, "state_bitwise": ok_state, "planners": K,
              "steps": out["steps"].tolist(), "status": out["status"],
              "against": "the host loop replayed with the device's trajectory on identical twins"}
    if every is not None:
        parity["records_bitwise"] = bool(ok_rec)
    if not parity["passed"]:
        sys.stderr.write("bench_trials.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        emit(json.dumps({"metric": "closed-loop trials", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    def host_round():
        reset(Bs)
        x = [np.asarray(p.params["x0"], dtype=np.float64) for p in Bs]
        running, steps = list(range(K)), 0
        for t in range(S):
            u = bb.solve()
            still = []
            for k in running:
                p = Bs[k]
                xn = plant_step(grids[k], x[k], u[k, 0], float(p.params["dt"]))
                if every is not None and t % every == 0:
                    p.get_state_rollout()
                p.shift_and_update(xn, u[k], 1)
                x[k] = xn
                steps += 1
                d = np.linalg.norm(xn[:2] - p.params["xgoal"]) - p.params["goal_tolerance"]
                if d > 0 and within(p, xn):
                    still.append(k)
            running = still
            if not running:
                break
        torch.cuda.synchronize(dev)
        return steps

    def device_round(**kw):
        reset(A)
        o = trials(ba, grids, S, **kw)
        torch.cuda.synchronize(dev)
        return int(o["steps"].sum())

    config = {"workload": (args.workload if args.workload in LOCAL_WORKLOADS else workload_name_of(args.workload)),
              "batch": K, "max_steps": S, "vis_rollouts": A[0].num_vis_state_rollouts,
              "planners": "seeds 1..K, warm started; even k: goal 1.5 m away, odd k: distant goal"}
    if every is not None:
        config["record_every"] = every
        config["host"] = "the host loop calls get_state_rollout() at every recorded step of every running planner"
    extra = []
    if mix:
        geos = sorted(set(shape), reverse=True)
        parts = [[k for k in range(K) if shape[k] == g] for g in geos]
        split = [(Batch([A[k] for k in ks]), [grids[k] for k in ks]) for ks in parts]

        def per_geometry_round():
            reset(A)
            steps = sum(int(trials(b, g, S)["steps"].sum()) for b, g in split)
            torch.cuda.synchronize(dev)
            return steps

        class Launches:                                  # the launches of every per-geometry batch
            def launch_count(self):
                return sum(b.launch_count() for b, _ in split)
        extra.append(("device_per_geometry", per_geometry_round, Launches()))
        config.update(workload="mix: c3's N, M, T on maps of %s cells a side (res %.1f m), %s bins; planner k: size k %% 3, "
                               "bins k %% 2" % (MIX_SIZES, res, MIX_BINS),
                      geometries=[{"cells": g[0], "bins": g[2], "planners": len(ks)} for g, ks in zip(geos, parts)])
    measure(args, emit, host_round, device_round, ba, bb, parity, dev,
            "closed-loop trials: host-driven loop vs " +
            ("MPPI_StochasticBatch.run_stochastic_trials" if stochastic else "MPPI_Batch.run_trials"), config,
            None if every is None else functools.partial(device_round, record_every=every), extra)


BENCH_ALPHAS = [1.0, 0.8, 0.6, 0.4, 0.2]               # the reference benchmark's cvar_alpha sweep


def run_shared(args, emit):
    """--share-tdms: device episodes of K planners on one map, K private TDM pairs against one shared pair."""
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from bench_batch import gpu_info, pair_state, planner_state, same, shared_map_planners, tdm_bytes
    from tests.scenarios import make_scenario
    K, S, every = args.batch, args.closed_loop, args.record_every
    mode, N, M, T, H, res, B, da = LOCAL_WORKLOADS.get(args.workload) or WORKLOADS[args.workload]
    stochastic = mode == "tdm"
    Batch = E.MPPI_StochasticBatch if stochastic else E.MPPI_Batch
    trials = ((lambda b, g, s, **kw: b.run_stochastic_trials(g, s, **kw)) if stochastic else
              (lambda b, g, s, **kw: b.run_trials(g, s, **kw)))
    W = MAP_WIDTH.get(args.workload, H)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scs = []
    for k in range(K):
        sc = make_scenario(mode, N=N, M=M, T=T, H=H, W=W, res=res, B=B, seed=k + 1, det_alpha=da, warm_start=True)
        if args.workload in VIS_ROLLOUTS:
            sc["cfg"]["num_vis_state_rollouts"] = VIS_ROLLOUTS[args.workload]
        if k % 2 == 0:
            sc["params"]["xgoal"] = sc["params"]["x0"][:2] + np.array([1.2, -0.9])
        scs.append(sc)
    alphas = BENCH_ALPHAS if args.workload in ("ref", "refm") else None
    grid = E.TractionGrid(*np.random.default_rng(7).uniform(0.3, 1.0, (2, H, W)), res=res)   # one ground truth
    grids = [grid] * K
    with _quiet():
        P = shared_map_planners(E, scs, False, alphas)    # private pairs
        Q = shared_map_planners(E, scs, True, alphas)     # one shared pair
    bp, bq = Batch(P), Batch(Q, share_tdms=True)

    def reset(pls):
        for p, sc in zip(pls, scs):
            p.params["x0"] = sc["params"]["x0"].copy()
            p.u_cur_d.copy_to_device(sc["u0"])

    def leg(b, pls, **kw):
        reset(pls)
        o = trials(b, grids, S, **kw)
        torch.cuda.synchronize(dev)
        return o

    start = all(same(pair_state(p), pair_state(q)) for p, q in zip(P, Q))
    kw = {} if every is None else dict(record_every=every)
    with _quiet():
        op, oq = leg(bp, P, **kw), leg(bq, Q, **kw)
    keys = ["xhist", "uhist", "steps"] + ([] if every is None else ["state_rollouts"])
    ok_hist = all(op[k].tobytes() == oq[k].tobytes() for k in keys) and op["status"] == oq["status"]
    ok_state = all(same(planner_state(p, stochastic) + [p.params["x0"]], planner_state(q, stochastic) + [q.params["x0"]])
                   for p, q in zip(P, Q))
    longest = int(np.argmax(op["steps"]))
    ok_pair = same(pair_state(Q[0]), pair_state(P[longest]))
    parity = {"passed": bool(start and ok_hist and ok_state and ok_pair), "same_start": bool(start),
              "histories_bitwise": bool(ok_hist), "state_bitwise": bool(ok_state),
              "shared_pair_equals_longest_private": bool(ok_pair), "planners": K, "steps": op["steps"].tolist(),
              "against": "the same planners' device episodes on K private TDM pairs of the map"}
    if not parity["passed"]:
        sys.stderr.write("bench_trials.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        emit(json.dumps({"metric": "closed-loop trials on one map", "error": "parity_check failed",
                         "parity_check": parity}))
        raise SystemExit(3)

    legs = (("private", bp, P), ("shared", bq, Q))
    res_ = {name: [] for name, _, _ in legs}
    launches = {}
    for _ in range(args.rounds):                         # alternate: private, shared, ...
        for name, b, pls in legs:
            l0 = b.launch_count()
            t0 = time.perf_counter()
            with _quiet():
                o = leg(b, pls, **kw)
            res_[name].append((time.perf_counter() - t0, int(o["steps"].sum())))
            launches[name] = b.launch_count() - l0

    def summary(name, pls):
        wall = [r[0] for r in res_[name]]
        med = float(np.median(wall))
        return {"s_per_round_wall": med, "s_per_round_wall_runs": wall, "control_steps_per_round": res_[name][0][1],
                "episodes_per_s": K / med, "kernel_launches_per_round": launches[name], "tdm_device_bytes": tdm_bytes(pls)}
    pri, sha = summary("private", P), summary("shared", Q)
    config = {"workload": (args.workload if args.workload in LOCAL_WORKLOADS else workload_name_of(args.workload)),
              "batch": K, "max_steps": S,
              "planners": "seed 1's map and ground truth; start poses, warm starts of seeds 1..K; even k: goal 1.5 m "
                          "away, odd k: distant goal" + ("; cvar_alpha cycling %s" % alphas if alphas else "")}
    if every is not None:
        config["record_every"] = every
    emit(json.dumps({"metric": "closed-loop trials of K planners on one map: K private TDM pairs vs one shared pair",
                     "unit": "episodes/s", "value": sha["episodes_per_s"], "higher_is_better": True, "config": config,
                     "rounds": args.rounds, "gpu": gpu_info(dev), "parity_check": parity, "private": pri,
                     "shared": sha, "speedup_wall": pri["s_per_round_wall"] / sha["s_per_round_wall"]}))


def run_episodes(args, emit):
    """--episodes E: E episodes per planner back to back, as the reference benchmark's run_trials loops over its
    ground-truth realisations."""
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from bench_batch import gpu_info, pair_state, planner_state, same, shared_map_planners
    from tests.scenarios import make_scenario
    from tests.trial_loop import plant_step, within
    K, S, n_ep = args.batch, args.closed_loop, args.episodes
    mode, N, M, T, H, res, B, da = LOCAL_WORKLOADS.get(args.workload) or WORKLOADS[args.workload]
    stochastic = mode == "tdm"
    Batch = E.MPPI_StochasticBatch if stochastic else E.MPPI_Batch
    trials = ((lambda b, g, s: b.run_stochastic_trials(g, s)) if stochastic else (lambda b, g, s: b.run_trials(g, s)))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scs = []
    for k in range(K):
        sc = make_scenario(mode, N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=k + 1, det_alpha=da, warm_start=True)
        if k % 2 == 0:
            sc["params"]["xgoal"] = sc["params"]["x0"][:2] + np.array([1.2, -0.9])
        scs.append(sc)
    rng = np.random.default_rng(7)
    seqs = [[E.TractionGrid(rng.uniform(0.3, 1.0, (H, H)), rng.uniform(0.3, 1.0, (H, H)), res=res) for _ in range(n_ep)]
            for _ in range(K)]
    alphas = BENCH_ALPHAS if args.share_tdms and args.workload == "ref" else None
    with _quiet():
        if args.share_tdms:                              # device and host legs on one shared pair, twins on private pairs
            A, Hs, Cs = (shared_map_planners(E, scs, True, alphas) for _ in range(3))
            Bs = shared_map_planners(E, scs, False, alphas)
        else:
            A, Hs, Bs, Cs = ([make_planner(E, sc, 0)[3] for sc in scs] for _ in range(4))

    def reset(pls):
        for p, sc in zip(pls, scs):
            p.params["x0"] = sc["params"]["x0"].copy()
            p.u_cur_d.copy_to_device(sc["u0"])

    for pls in (A, Hs, Bs, Cs):
        reset(pls)
    ba, bh, bc = (Batch(pls, share_tdms=args.share_tdms) for pls in (A, Hs, Cs))

    # ---- parity: the benchmark's loop on the device == the host sequence loop replayed with its trajectory
    with _quiet():
        out = ba.run_trial_sequences(seqs, S)
        ok_u = True
        for k, p in enumerate(Bs):
            one = Batch([p])
            for e in range(int(out["episodes_run"][k])):
                for t in range(int(out["steps"][k, e])):
                    useq = one.solve()[0]
                    ok_u &= bool(np.array_equal(useq[0], out["uhist"][k, e, t]))
                    p.shift_and_update(out["xhist"][k, e, t + 1], useq, 1)
    ok_state = all(same(planner_state(a, stochastic) + [a.params["x0"]], planner_state(b, stochastic) + [b.params["x0"]])
                   for a, b in zip(A, Bs))
    longest = int(np.argmax(out["steps"].sum(axis=1)))
    ok_pair = all(same(pair_state(a), pair_state(Bs[longest] if args.share_tdms else b)) for a, b in zip(A, Bs))
    parity = {"passed": bool(ok_u and ok_state and ok_pair), "u_bitwise": ok_u, "state_bitwise": ok_state,
              "tdm_pairs_bitwise": ok_pair, "planners": K, "episodes_run": out["episodes_run"].tolist(),
              "steps": out["steps"].tolist(),
              "against": "the host sequence loop replayed with the device's trajectory on identical twins (private "
                         "TDM pairs)"}
    if not parity["passed"]:
        sys.stderr.write("bench_trials.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        emit(json.dumps({"metric": "trial sequences", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    keys = ("xhist", "uhist", "steps")
    last = {}

    def sequence_round(b=ba, pls=A):
        reset(pls)
        o = b.run_trial_sequences(seqs, S, reset_x0=True)
        torch.cuda.synchronize(dev)
        last["sequence"] = o
        return int(o["steps"].sum()), b.steps_issued

    def calls_round(b=ba, pls=A):
        reset(pls)
        outs, issued = [], 0
        starts = [sc["params"]["x0"] for sc in scs]
        for e in range(n_ep):
            for p, x in zip(pls, starts):
                p.params["x0"] = x.copy()
            outs.append(trials(b, [seqs[k][e] for k in range(K)], S))
            issued += b.steps_issued
        torch.cuda.synchronize(dev)
        last["calls"] = {key: np.stack([o[key] for o in outs], axis=1) for key in keys}
        return int(sum(o["steps"].sum() for o in outs)), issued

    # the reset_x0 sequence against the consecutive calls, from the same planner state (the rounds below do not restore
    # RNG streams): a shared pair is sampled at every step any member runs, so the calls (each until its slowest member
    # stops) sample it more often than the sequence, and only private pairs give the calls' histories
    with _quiet():
        sequence_round(bh, Hs)
        calls_round(bc, Cs)
    same_hist = all(last["sequence"][key].tobytes() == last["calls"][key].tobytes() for key in keys)
    if not same_hist and not args.share_tdms:
        sys.stderr.write("bench_trials.py: the reset_x0 sequence differs from consecutive run_trials calls\n")
        emit(json.dumps({"metric": "trial sequences", "error": "sequence != consecutive run_trials calls"}))
        raise SystemExit(3)

    def host_round():
        reset(Hs)
        steps = issued = 0
        starts = [np.asarray(sc["params"]["x0"], dtype=np.float64) for sc in scs]
        for e in range(n_ep):
            x = [s.copy() for s in starts]
            for p, s in zip(Hs, starts):
                p.params["x0"] = s.copy()
            running = list(range(K))
            for t in range(S):
                u = bh.solve()
                issued += 1
                still = []
                for k in running:
                    p = Hs[k]
                    xn = plant_step(seqs[k][e], x[k], u[k, 0], float(p.params["dt"]))
                    p.shift_and_update(xn, u[k], 1)
                    x[k] = xn
                    steps += 1
                    d = np.linalg.norm(xn[:2] - p.params["xgoal"]) - p.params["goal_tolerance"]
                    if d > 0 and within(p, xn):
                        still.append(k)
                running = still
                if not running:
                    break
        torch.cuda.synchronize(dev)
        return steps, issued

    legs = [("sequence", sequence_round, ba), ("calls", calls_round, ba), ("host", host_round, bh)]
    with _quiet():
        for _, fn, _ in legs:                            # warm-up of every path
            fn()
    res_ = {name: [] for name, _, _ in legs}
    launches = {}
    for _ in range(args.rounds):                         # alternate: sequence, calls, host, ...
        for name, fn, b in legs:
            l0 = b.launch_count()
            t0 = time.perf_counter()
            with _quiet():
                steps, issued = fn()
            res_[name].append((time.perf_counter() - t0, steps, issued))
            launches[name] = b.launch_count() - l0

    def summary(name):
        wall = [r[0] for r in res_[name]]
        med = float(np.median(wall))
        return {"s_per_round_wall": med, "s_per_round_wall_runs": wall, "control_steps_per_round": res_[name][0][1],
                "steps_issued_per_round": res_[name][0][2], "episodes_per_s": K * n_ep / med,
                "kernel_launches_per_round": launches[name]}
    seq, calls, host = summary("sequence"), summary("calls"), summary("host")
    config = {"workload": (args.workload if args.workload in LOCAL_WORKLOADS else workload_name_of(args.workload)),
              "batch": K, "max_steps": S, "episodes": n_ep, "share_tdms": bool(args.share_tdms),
              "planners": "seeds 1..K, warm started; even k: goal 1.5 m away, odd k: distant goal; E seeded grids each"
                          + ("; one shared TDM pair, cvar_alpha cycling %s" % alphas if args.share_tdms and alphas
                             else "; one shared TDM pair" if args.share_tdms else "")}
    emit(json.dumps({"metric": "trial sequences: one run_trial_sequences call vs E run_trials calls vs the host loop",
                     "unit": "episodes/s", "value": seq["episodes_per_s"], "higher_is_better": True, "config": config,
                     "rounds": args.rounds, "gpu": gpu_info(dev), "parity_check": parity,
                     "sequence_equals_calls_bitwise": bool(same_hist), "sequence": seq, "calls": calls, "host": host,
                     "speedup_wall_vs_calls": calls["s_per_round_wall"] / seq["s_per_round_wall"],
                     "speedup_wall_vs_host": host["s_per_round_wall"] / seq["s_per_round_wall"]}))


def run_device_grids(args, emit):
    """--device-grids: the benchmark's E realisations per planner, drawn on the GPU from a ground-truth TDM pair and read
    in place, against the same realisations drawn by the reference notebook's helper and passed as host grids."""
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from bench_batch import gpu_info, planner_state, same
    from tests.scenarios import make_scenario
    K, S, n_ep = args.batch, args.closed_loop, args.episodes
    mode, N, M, T, H, res, B, da = LOCAL_WORKLOADS.get(args.workload) or WORKLOADS[args.workload]
    stochastic = mode == "tdm"
    Batch = E.MPPI_StochasticBatch if stochastic else E.MPPI_Batch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scs = []
    for k in range(K):
        sc = make_scenario(mode, N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=k + 1, det_alpha=da, warm_start=True)
        if k % 2 == 0:
            sc["params"]["xgoal"] = sc["params"]["x0"][:2] + np.array([1.2, -0.9])
        scs.append(sc)
    # the ground truth: a use_tdm pair of the workload's map geometry and M, as the notebook builds it next to the planner
    gsc = make_scenario("tdm", N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=1000)

    def gt_pair():
        with _quiet():
            cfg = E.Config(**gsc["cfg"])
            lin, ang = E.TDM_Numba(cfg), E.TDM_Numba(cfg)
            lin.set_TDM_from_PMF_grid(gsc["pmf_lin"], gsc["tdm_dict"])
            ang.set_TDM_from_PMF_grid(gsc["pmf_ang"], gsc["tdm_dict"])
        return lin, ang

    def helper(lin, ang):                                # the notebook's sample_traction_grid, widened to float64
        lq = lin.sample_grids().copy_to_host()[0]
        lg = lq * (lin.bin_values_bounds[1] - lin.bin_values_bounds[0]) / 100.0 + lin.bin_values_bounds[0]
        aq = ang.sample_grids().copy_to_host()[0]
        ag = aq * (ang.bin_values_bounds[1] - ang.bin_values_bounds[0]) / 100.0 + ang.bin_values_bounds[0]
        return E.TractionGrid(lg.astype(np.float64), ag.astype(np.float64), lin.res, xlimits=lin.padded_xlimits,
                              ylimits=lin.padded_ylimits)

    ga, gb = gt_pair(), gt_pair()
    with _quiet():
        A, Bs = ([make_planner(E, sc, 0)[3] for sc in scs] for _ in range(2))

    def reset(pls):
        for p, sc in zip(pls, scs):
            p.params["x0"] = sc["params"]["x0"].copy()
            p.u_cur_d.copy_to_device(sc["u0"])

    for pls in (A, Bs):
        reset(pls)
    ba, bb = Batch(A), Batch(Bs)
    dgrids = E.draw_traction_grids(ga[0], ga[1], n_ep)
    hgrids = [helper(*gb) for _ in range(n_ep)]
    dseqs, hseqs = [list(dgrids)] * K, [hgrids] * K

    # ---- parity: the realisations, then one sequence call on device realisations == the twins' call on host grids
    ok_planes = all(same(list(d.get_grids()), [h.lin_traction, h.ang_traction]) for d, h in zip(dgrids, hgrids))
    with _quiet():
        oa = ba.run_trial_sequences(dseqs, S, reset_x0=True)
        ob = bb.run_trial_sequences(hseqs, S, reset_x0=True)
    ok_out = all(oa[key].tobytes() == ob[key].tobytes() for key in ("xhist", "uhist", "steps")) and \
        oa["status"] == ob["status"]
    ok_state = all(same(planner_state(a, stochastic) + [a.params["x0"]], planner_state(b, stochastic) + [b.params["x0"]])
                   for a, b in zip(A, Bs))
    parity = {"passed": bool(ok_planes and ok_out and ok_state), "planes_bitwise": ok_planes,
              "histories_bitwise": ok_out, "state_bitwise": ok_state, "steps": oa["steps"].tolist(),
              "against": "the notebook's sample_traction_grid on a twin ground-truth pair, as host grids, on identical "
                         "twin planners"}
    if not parity["passed"]:
        sys.stderr.write("bench_trials.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        emit(json.dumps({"metric": "device realisations", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    def round_(b, pls, seqs):
        reset(pls)
        o = b.run_trial_sequences(seqs, S, reset_x0=True)
        torch.cuda.synchronize(dev)
        return int(o["steps"].sum())

    legs = [("host_grids", functools.partial(round_, bb, Bs, hseqs), bb),
            ("device_grids", functools.partial(round_, ba, A, dseqs), ba)]
    with _quiet():
        for _, fn, _ in legs:                            # warm-up of both paths
            fn()
    res_ = {name: [] for name, _, _ in legs}
    for _ in range(args.rounds):                         # alternate: host grids, device grids, ...
        for name, fn, _ in legs:
            t0 = time.perf_counter()
            with _quiet():
                steps = fn()
            res_[name].append((time.perf_counter() - t0, steps))
    # the draw itself against the helper's path, alternating (each call ends in a synchronisation)
    draw, help_ = [], []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        E.draw_traction_grids(ga[0], ga[1], n_ep)
        draw.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        with _quiet():
            [helper(*gb) for _ in range(n_ep)]
        help_.append(time.perf_counter() - t0)
    plane = dgrids.height * dgrids.width * 8

    def summary(name):
        wall = [r[0] for r in res_[name]]
        return {"s_per_round_wall": float(np.median(wall)), "s_per_round_wall_runs": wall,
                "control_steps_per_round": res_[name][0][1],
                "grid_bytes_uploaded_per_call": (2 * plane * K * n_ep if name == "host_grids" else 0)}
    host, devr = summary("host_grids"), summary("device_grids")
    config = {"workload": (args.workload if args.workload in LOCAL_WORKLOADS else workload_name_of(args.workload)),
              "batch": K, "max_steps": S, "episodes": n_ep, "reset_x0": True,
              "ground_truth": "use_tdm pair of the workload's map geometry and M %d (seed 1000); one set of E "
                              "realisations shared by every planner" % M,
              "plane_cells": [dgrids.height, dgrids.width]}
    emit(json.dumps({"metric": "trial sequences: host ground-truth grids vs device realisations read in place",
                     "unit": "s/round", "value": devr["s_per_round_wall"], "higher_is_better": False, "config": config,
                     "rounds": args.rounds, "gpu": gpu_info(dev), "parity_check": parity, "host_grids": host,
                     "device_grids": devr, "speedup_wall": host["s_per_round_wall"] / devr["s_per_round_wall"],
                     "draw_s": float(np.median(draw)), "draw_s_runs": draw, "helper_s": float(np.median(help_)),
                     "helper_s_runs": help_}))


def _quiet():
    import contextlib
    import io
    return contextlib.redirect_stdout(io.StringIO())


def measure(args, emit, host_round, device_round, ba, bb, parity, dev, metric, config, recorded_round=None, extra=()):
    """R alternating timed rounds of the host loop (on batch bb), the device episodes (on batch ba), when given the
    device episodes with recording, and the `extra` legs (name, round, object whose launch_count() counts its launches),
    then the JSON line."""
    import torch
    K = len(ba)
    legs = [("host", host_round, bb), ("device", device_round, ba)]
    if recorded_round is not None:
        legs.append(("device_recorded", recorded_round, ba))
    legs += list(extra)
    for _, fn, _ in legs:                                 # warm-up of every path
        fn()
    res = {name: [] for name, _, _ in legs}
    launches = {}
    for _ in range(args.rounds):
        for name, fn, b in legs:
            l0 = b.launch_count()
            t0 = time.perf_counter()
            steps = fn()
            res[name].append((time.perf_counter() - t0, steps))
            launches[name] = b.launch_count() - l0

    def summary(name):
        wall = [r[0] for r in res[name]]
        med = float(np.median(wall))
        return {"s_per_round_wall": med, "s_per_round_wall_runs": wall, "control_steps_per_round": res[name][0][1],
                "control_steps_per_s": res[name][0][1] / med, "episodes_per_s": K / med,
                "kernel_launches_per_round": launches[name]}
    host, devr = summary("host"), summary("device")
    split = record_share = None
    if args.profile:                                     # a separate run: tracing slows the host
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            (recorded_round or device_round)()
        split = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and ev.count:
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                split[ev.key] = {"ms": t / 1e3, "launches": ev.count}
        split = dict(sorted(split.items(), key=lambda kv: -kv[1]["ms"]))
        if recorded_round is not None:                   # the recording's own kernels in the profiled recording round
            total = sum(v["ms"] for v in split.values())
            record_share = {name: sum(v["ms"] for key, v in split.items() if name in key) / total
                            for name in ("state_rollout_batch_kernel", "sample_grids_v2_complete_batch_kernel")}
    gpu = {"name": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        gpu["power_limit_and_max_sm_clock"] = q
    except Exception as e:                               # noqa: BLE001
        gpu["power_limit_and_max_sm_clock"] = "unavailable (%r)" % e
    line = {"metric": metric, "unit": "episodes/s", "value": devr["episodes_per_s"], "higher_is_better": True,
            "config": config, "rounds": args.rounds, "gpu": gpu, "parity_check": parity, "host": host, "device": devr,
            "speedup_wall": host["s_per_round_wall"] / devr["s_per_round_wall"], "device_kernel_split_one_round": split}
    if recorded_round is not None:
        rec = summary("device_recorded")
        line.update(device_recorded=rec, speedup_wall_recorded=host["s_per_round_wall"] / rec["s_per_round_wall"],
                    recording_cost_wall=rec["s_per_round_wall"] / devr["s_per_round_wall"] - 1.0,
                    record_kernels_share_of_device_time=record_share)
    for name, _, _ in extra:
        ex = summary(name)
        line[name] = ex
        line["speedup_wall_over_" + name] = ex["s_per_round_wall"] / devr["s_per_round_wall"]
    emit(json.dumps(line))


def _bb_params(K):
    """The bb workload's planner params (run_bb)."""
    params = []
    for k in range(K):
        rng = np.random.default_rng(1000 + k)
        x0 = np.array([0.0, 0.0, np.pi / 4]) + rng.uniform(-0.3, 0.3, 3)
        xgoal = x0[:2] + np.array([0.3, 1.2]) if k % 2 == 0 else np.array([7.0, 5.0]) + rng.uniform(-0.3, 0.3, 2)
        params.append(dict(dt=0.1, x0=x0, xgoal=xgoal, goal_tolerance=0.5, dist_weight=10, lambda_weight=1.0, num_opt=1,
                           u_std=np.array([1.0, 1.0]), vrange=np.array([0.0, 2.0]), wrange=np.array([-np.pi, np.pi]),
                           obstacle_positions=np.array([[5.0, 4.5], [2.0, 1.0]]) + rng.uniform(-0.2, 0.2, (2, 2)),
                           obstacle_radius=np.array([1.5, 1.0]), obs_penalty=1e6))
    return params


def _bb_planners(params):
    from mppi_numba_b200 import barebone as BB
    pls = []
    for k, q in enumerate(params):
        p = BB.MPPI_Numba(BB.Config(T=5.0, dt=0.1, num_control_rollouts=1000, seed=k + 1))
        p.setup(q)
        pls.append(p)
    return pls


def run_bb(args, emit):
    """The bb workload: barebone planners of the notebook's shape (N 1000, T 50, dt 0.1, its two obstacles, vrange
    [0, 2], u_std [1, 1], dist_weight 10, obs_penalty 1e6, goal_tolerance 0.5), planner k with its own seed and seeded
    perturbations of the start, the goal and the obstacles; even k: a goal about 1.2 m away, odd k: the notebook's
    goal, 8.6 m away.  Host loop: the batch's solve() of all K, then per running planner the numpy plant step and
    shift_and_update; device: one run_barebone_trials(S)."""
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from mppi_numba_b200 import barebone as BB
    from tests.barebone_trial_loop import goal_distance, in_contact, obstacles, plant_step
    K, S = args.batch, args.closed_loop
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    params = _bb_params(K)
    A, Bs = _bb_planners(params), _bb_planners(params)
    T = A[0].num_steps

    def reset(pls):
        for p, q in zip(pls, params):
            p.params["x0"] = q["x0"].copy()
            p.u_cur_d.copy_to_device(np.zeros((T, 2), np.float32))

    reset(A), reset(Bs)
    ba, bb = E.MPPI_Batch(A), E.MPPI_Batch(Bs)

    # ---- parity: the device episodes == the host loop replayed with the device's trajectory; the contact counts ==
    # numpy's rule on the device's trajectory
    out = ba.run_barebone_trials(S)
    ok_u = ok_contacts = True
    for k, p in enumerate(Bs):
        one = E.MPPI_Batch([p])
        n = int(out["steps"][k])
        for t in range(n):
            useq = one.solve()[0]
            ok_u &= useq[0].tobytes() == out["uhist"][k, t].tobytes()
            p.shift_and_update(out["xhist"][k, t + 1], useq, 1)
        obs = obstacles(p)
        ok_contacts &= int(out["contact_steps"][k]) == sum(in_contact(out["xhist"][k, t], obs) for t in range(1, n + 1))

    def state(p):
        d = [p.u_cur_d, p.u_prev_d, p.costs_d, p.weights_d, p.noise_samples_d, p.rng_states_d]
        return [a.copy_to_host() for a in d] + [np.asarray(p.params["x0"])]
    ok_state = all(all(x.dtype == y.dtype and x.tobytes() == y.tobytes() for x, y in zip(state(a), state(b)))
                   for a, b in zip(A, Bs))
    parity = {"passed": bool(ok_u and ok_state and ok_contacts), "u_bitwise": bool(ok_u),
              "state_bitwise": bool(ok_state), "contacts_exact": bool(ok_contacts), "planners": K,
              "steps": out["steps"].tolist(), "status": out["status"], "contact_steps": out["contact_steps"].tolist(),
              "against": "the host loop replayed with the device's trajectory on identical twins"}
    if not parity["passed"]:
        sys.stderr.write("bench_trials.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        emit(json.dumps({"metric": "closed-loop trials", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    def host_round():
        reset(Bs)
        x = [np.asarray(p.params["x0"], dtype=np.float64) for p in Bs]
        running, steps = list(range(K)), 0
        for t in range(S):
            u = bb.solve()
            still = []
            for k in running:
                p = Bs[k]
                xn = plant_step(x[k], u[k, 0], float(p.params["dt"]))
                p.shift_and_update(xn, u[k], 1)
                x[k] = xn
                steps += 1
                if goal_distance(p, xn) > 0:
                    still.append(k)
            running = still
            if not running:
                break
        torch.cuda.synchronize(dev)
        return steps

    def device_round():
        reset(A)
        o = ba.run_barebone_trials(S)
        torch.cuda.synchronize(dev)
        return int(o["steps"].sum())

    measure(args, emit, host_round, device_round, ba, bb, parity, dev,
            "closed-loop trials: host-driven loop vs MPPI_Batch.run_barebone_trials",
            {"workload": "bb: barebone notebook (N 1000, T 50, dt 0.1, two obstacles)", "batch": K, "max_steps": S,
             "planners": "seeds 1..K, seeded start / goal / obstacle perturbations; even k: goal 1.2 m away, odd k: "
                         "the notebook's goal"})


def run_recorded_episodes(args, emit):
    """--episodes E with --record-every n (c3, ref, gif), or --workload bb --episodes E [--record-every n]: E episodes
    per planner back to back, recording each episode's steps t with t % n == 0 (bb: counting contacts per episode)."""
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from bench_batch import gpu_info
    K, S, n_ep, every = args.batch, args.closed_loop, args.episodes, args.record_every
    bb = args.workload == "bb"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    if bb:
        from tests.barebone_trial_loop import goal_distance, in_contact, obstacles
        from tests.barebone_trial_loop import plant_step as bb_step
        params = _bb_params(K)
        A, Bs, Hs, Cs = (_bb_planners(params) for _ in range(4))
        Batch, seqs = E.MPPI_Batch, None

        def reset(pls):
            for p, q in zip(pls, params):
                p.params["x0"] = q["x0"].copy()
                p.u_cur_d.copy_to_device(np.zeros((p.num_steps, 2), np.float32))

        def sequences(b, **kw):
            return b.run_barebone_trial_sequences(n_ep, S, **kw)

        def plant(k, e, x, u, p):
            return bb_step(x, u, float(p.params["dt"]))

        def stops(p, xn):
            return goal_distance(p, xn) <= 0
    else:
        from tests.scenarios import make_scenario
        from tests.trial_loop import plant_step, within
        mode, N, M, T, H, res, B, da = LOCAL_WORKLOADS.get(args.workload) or WORKLOADS[args.workload]
        W = MAP_WIDTH.get(args.workload, H)
        scs = []
        for k in range(K):
            sc = make_scenario(mode, N=N, M=M, T=T, H=H, W=W, res=res, B=B, seed=k + 1, det_alpha=da, warm_start=True)
            if args.workload in VIS_ROLLOUTS:
                sc["cfg"]["num_vis_state_rollouts"] = VIS_ROLLOUTS[args.workload]
            if k % 2 == 0:
                sc["params"]["xgoal"] = sc["params"]["x0"][:2] + np.array([1.2, -0.9])
            scs.append(sc)
        rng = np.random.default_rng(7)
        seqs = [[E.TractionGrid(rng.uniform(0.3, 1.0, (H, W)), rng.uniform(0.3, 1.0, (H, W)), res=res)
                 for _ in range(n_ep)] for _ in range(K)]
        with _quiet():
            A, Bs, Hs, Cs = ([make_planner(E, sc, 0)[3] for sc in scs] for _ in range(4))
        Batch = E.MPPI_StochasticBatch if mode == "tdm" else E.MPPI_Batch

        def reset(pls):
            for p, sc in zip(pls, scs):
                p.params["x0"] = sc["params"]["x0"].copy()
                p.u_cur_d.copy_to_device(sc["u0"])

        def sequences(b, **kw):
            return b.run_trial_sequences(seqs, S, **kw)

        def plant(k, e, x, u, p):
            return plant_step(seqs[k][e], x, u, float(p.params["dt"]))

        def stops(p, xn):
            return np.linalg.norm(xn[:2] - p.params["xgoal"]) - p.params["goal_tolerance"] <= 0 or not within(p, xn)
    for pls in (A, Bs, Hs, Cs):
        reset(pls)
    ba, bh, bc = Batch(A), Batch(Hs), Batch(Cs)
    rec_kw = {} if every is None else dict(record_every=every)

    # ---- parity: the benchmark's loop (no reset) on the device == the host sequence loop replayed on twins with the
    # device's trajectory, get_state_rollout() at each episode's recorded steps
    with _quiet():
        out = sequences(ba, **rec_kw)
        ok_u = ok_rec = ok_con = True
        for k, p in enumerate(Bs):
            one = Batch([p])
            for e in range(int(out["episodes_run"][k])):
                n = int(out["steps"][k, e])
                for t in range(n):
                    useq = one.solve()[0]
                    ok_u &= useq[0].tobytes() == out["uhist"][k, e, t].tobytes()
                    if every is not None and t % every == 0:
                        ok_rec &= p.get_state_rollout().tobytes() == out["state_rollouts"][k, e, t // every].tobytes()
                    p.shift_and_update(out["xhist"][k, e, t + 1], useq, 1)
                if every is not None:
                    ok_rec &= bool(np.isnan(out["state_rollouts"][k, e, -(-n // every):]).all())
                if bb:
                    ok_con &= int(out["contact_steps"][k, e]) == sum(
                        in_contact(out["xhist"][k, e, t], obstacles(p)) for t in range(1, n + 1))
            if every is not None:
                ok_rec &= bool(np.isnan(out["state_rollouts"][k, int(out["episodes_run"][k]):]).all())

    def state(p):
        d = [p.u_cur_d, p.u_prev_d, p.costs_d, p.weights_d, p.noise_samples_d, p.rng_states_d]
        if not bb:
            d += [p.lin_tdm.rng_states_d, p.ang_tdm.rng_states_d, p.lin_tdm.sample_grid_batch_d,
                  p.ang_tdm.sample_grid_batch_d]
        if every is not None:
            d.append(p.state_rollout_batch_d)
        return [a.copy_to_host().tobytes() for a in d] + [np.asarray(p.params["x0"]).tobytes()]
    ok_state = all(state(a) == state(b) for a, b in zip(A, Bs))
    parity = {"passed": bool(ok_u and ok_state and ok_rec and ok_con), "u_bitwise": bool(ok_u),
              "state_bitwise": bool(ok_state), "planners": K, "episodes_run": out["episodes_run"].tolist(),
              "steps": out["steps"].tolist(),
              "against": "the host sequence loop replayed with the device's trajectory on identical twins"}
    if every is not None:
        parity["records_bitwise"] = bool(ok_rec)
    if bb:
        parity["contacts_exact"] = bool(ok_con)
    if not parity["passed"]:
        sys.stderr.write("bench_trials.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        emit(json.dumps({"metric": "trial sequences", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    def device_round(b, pls, **kw):
        reset(pls)
        o = sequences(b, reset_x0=True, **kw)
        torch.cuda.synchronize(dev)
        return int(o["steps"].sum()), b.steps_issued

    def host_round():                                    # the drawing loop: the batch's solve and get_state_rollout
        reset(Hs)
        steps = issued = 0
        starts = [np.asarray(p.params["x0"], dtype=np.float64).copy() for p in Hs]
        for e in range(n_ep):
            x = [s.copy() for s in starts]
            for p, s in zip(Hs, starts):
                p.params["x0"] = s.copy()
            running = list(range(K))
            for t in range(S):
                u = bh.solve()
                issued += 1
                if every is not None and t % every == 0:
                    bh.get_state_rollout()
                still = []
                for k in running:
                    p = Hs[k]
                    xn = plant(k, e, x[k], u[k, 0], p)
                    p.shift_and_update(xn, u[k], 1)
                    x[k] = xn
                    steps += 1
                    if not stops(p, xn):
                        still.append(k)
                running = still
                if not running:
                    break
        torch.cuda.synchronize(dev)
        return steps, issued

    legs = [("recorded" if every is not None else "sequence", functools.partial(device_round, ba, A, **rec_kw), ba),
            ("host", host_round, bh)]
    if every is not None:
        legs.insert(1, ("unrecorded", functools.partial(device_round, bc, Cs), bc))
    with _quiet():
        for _, fn, _ in legs:                            # warm-up of every path
            fn()
    res_ = {name: [] for name, _, _ in legs}
    launches = {}
    for _ in range(args.rounds):                         # alternate the legs
        for name, fn, b in legs:
            l0 = b.launch_count()
            t0 = time.perf_counter()
            with _quiet():
                steps, issued = fn()
            res_[name].append((time.perf_counter() - t0, steps, issued))
            launches[name] = b.launch_count() - l0

    def summary(name):
        wall = [r[0] for r in res_[name]]
        med = float(np.median(wall))
        return {"s_per_round_wall": med, "s_per_round_wall_runs": wall, "control_steps_per_round": res_[name][0][1],
                "steps_issued_per_round": res_[name][0][2], "episodes_per_s": K * n_ep / med,
                "kernel_launches_per_round": launches[name]}
    sums = {name: summary(name) for name, _, _ in legs}
    lead = legs[0][0]
    config = {"workload": ("bb" if bb else args.workload if args.workload in LOCAL_WORKLOADS
                           else workload_name_of(args.workload)),
              "batch": K, "max_steps": S, "episodes": n_ep, "record_every": every,
              "legs": "reset_x0=True sequences on the device; host: the batch's solve()%s and a numpy plant step per "
                      "running planner" % (" and get_state_rollout() at recorded steps" if every is not None else "")}
    line = {"metric": "trial sequences%s: one device call vs the host loop" % (" with records" if every else ""),
            "unit": "episodes/s", "value": sums[lead]["episodes_per_s"], "higher_is_better": True, "config": config,
            "rounds": args.rounds, "gpu": gpu_info(dev), "parity_check": parity,
            "speedup_wall_vs_host": sums["host"]["s_per_round_wall"] / sums[lead]["s_per_round_wall"]}
    line.update(sums)
    if every is not None:
        line["recording_cost_wall"] = sums["recorded"]["s_per_round_wall"] / sums["unrecorded"]["s_per_round_wall"]
    emit(json.dumps(line))


def main():
    # one JSON line on stdout: everything else (the engine's allocation notices, ...) goes to stderr
    real_stdout = os.dup(1)
    os.dup2(2, 1)
    sys.stdout = os.fdopen(os.dup(2), "w", buffering=1)

    def emit(line):
        os.write(real_stdout, (line + "\n").encode())
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[1])
    ap.add_argument("--workload", default="c2", choices=["c2", "c4", "c3", "ref", "refm", "gif", "mix", "bb"])
    ap.add_argument("--batch", type=int, default=64, metavar="K", help="planners in the batch")
    ap.add_argument("--closed-loop", type=int, default=150, metavar="S", help="max control steps per episode")
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds of each loop")
    ap.add_argument("--profile", action="store_true", help="then one device round under torch.profiler: kernel split")
    ap.add_argument("--record-every", type=int, default=None, metavar="n",
                    help="record the visualisation rollouts of every n-th step (not bb)")
    ap.add_argument("--share-tdms", action="store_true",
                    help="K planners on one map: K private TDM pairs against one pair shared by all (not bb)")
    ap.add_argument("--episodes", type=int, default=None, metavar="E",
                    help="E ground-truth realisations per planner back to back (c2, c3, ref; with --record-every: "
                         "c3, ref, gif; bb: E barebone episodes)")
    ap.add_argument("--device-grids", action="store_true",
                    help="with --episodes: the realisations drawn and read on the GPU against host grids (c4, ref)")
    args = ap.parse_args()
    if args.batch < 1 or args.closed_loop < 1 or args.rounds < 1:
        ap.error("--batch, --closed-loop and --rounds must be at least 1")
    if args.record_every is not None and args.record_every < 1:
        ap.error("--record-every must be at least 1")
    if args.workload == "bb" and args.record_every is not None and args.episodes is None:
        ap.error("the bb workload takes --record-every only with --episodes")
    if args.share_tdms and args.workload in ("bb", "mix"):
        ap.error("--share-tdms: barebone planners have no TDMs, and mix planners no common map")
    if args.device_grids:
        if args.episodes is None or args.episodes < 1 or args.workload not in ("c4", "ref") or args.share_tdms or \
                args.record_every is not None:
            ap.error("--device-grids needs --episodes E >= 1 and workload c4 or ref, without --share-tdms and "
                     "--record-every")
        run_device_grids(args, emit)
        return
    if args.episodes is not None:
        if args.episodes < 1:
            ap.error("--episodes must be at least 1")
        if args.workload == "bb" or args.record_every is not None:
            if args.share_tdms or (args.workload != "bb" and args.workload not in ("c3", "ref", "gif")):
                ap.error("--episodes with --record-every takes workload c3, ref or gif (or bb), without --share-tdms")
            run_recorded_episodes(args, emit)
            return
        if args.workload not in ("c2", "c3", "ref"):
            ap.error("--episodes takes workload c2, c3 or ref (with --record-every: c3, ref, gif; or bb)")
        run_episodes(args, emit)
        return
    (run_bb if args.workload == "bb" else run_shared if args.share_tdms else run)(args, emit)


if __name__ == "__main__":
    main()
