#!/usr/bin/env python
"""bench_loop.py -- the receding-horizon loop with the caller's plant: the device loop against the host loop.

    python bench_loop.py --workload c2|c3|bb|ref --batch K --closed-loop S [--rounds R] [--graph-steps G]

A user whose plant is not the built-in one (a simulator, a learned model, a state estimate in GPU memory) drives the
planners with batch.device_loop(): solve() and shift_and_update(x) on the batch's stream, poses and controls in GPU
memory.  Here the plant is the benchmark's unicycle on a ground-truth traction grid (bb: the barebone notebook's
nominal unicycle), written in torch on the device.  c2 is one-map (MPPI_Batch), c3 and ref are stochastic
(MPPI_StochasticBatch; ref is bench_trials.py's reference shape), bb is barebone (bench_trials.py's bb planners).

First the parity check, for the device loop and for the graph-replayed loop: the loop with the torch plant on one set
of planners; on identical twins the host loop replayed with the loop's poses (u = MPPI_*Batch([p]).solve()[0],
p.shift_and_update(x[k], u, 1)): u of every solve and every planner's final state bit for bit; a mismatch exits
non-zero.  Then R rounds of four legs, alternating, every round from the same start (params, warm start), S steps each:
  device_loop: S x (loop.solve(), the torch plant, loop.stop(at goal), loop.shift_and_update(x)); no host wait inside;
  graph:       the device_loop step on a side stream: one eager step, then G steps of it captured into one CUDA graph
               (torch.cuda.CUDAGraph) and replayed ceil((S - 1) / G) times; the loop's open, capture and close included
               (each timed round's capture, instantiation included, is also reported on its own);
  host:        S x (batch.solve(), per running planner the numpy plant step and shift_and_update) until all stopped;
  run_trials:  one run_trials(grids, S) (run_stochastic_trials, run_barebone_trials), the built-in plant: the floor.
Planners stop at the goal on the device, so steps after that do nothing in every leg but the host's, which stops
issuing.  Wall clock per round (each ends in a host synchronisation) and kernel launches per round (issued from the
host: a replay adds none).  Prints one JSON line with the card's name, power limit and maximum SM clock; writes
nothing to the tree."""
import argparse
import contextlib
import io
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import WORKLOADS, make_planner   # noqa: E402
from bench_trials import LOCAL_WORKLOADS, _bb_params, _bb_planners   # noqa: E402


def torch_plant(torch, x, u0, dt, grids, xlo, ylo, res, goal, tol):
    """One plant step of every planner in float64 on the device: traction from its grid (TractionGrid.get: the cell
    floor((x - lo) / res), traction 0 outside; grids None: 1, the nominal unicycle), then x += dt lt cos(th) v, ...
    Returns (x_next, at_goal)."""
    v = torch.nan_to_num(u0[:, 0].double())
    w = torch.nan_to_num(u0[:, 1].double())
    if grids is None:
        lt = at = torch.ones_like(v)
    else:
        lin, ang = grids
        Hh, Ww = lin.shape[1], lin.shape[2]
        fx = torch.div(x[:, 0] - xlo, res, rounding_mode="floor")
        fy = torch.div(x[:, 1] - ylo, res, rounding_mode="floor")
        inside = (fx >= 0) & (fx < Ww) & (fy >= 0) & (fy < Hh)
        ix = torch.where(inside, fx, torch.zeros_like(fx)).long()
        iy = torch.where(inside, fy, torch.zeros_like(fy)).long()
        k = torch.arange(x.shape[0], device=x.device)
        lt = torch.where(inside, lin[k, iy, ix], torch.zeros_like(v))
        at = torch.where(inside, ang[k, iy, ix], torch.zeros_like(v))
    th = x[:, 2]
    xn = torch.stack([x[:, 0] + dt * lt * torch.cos(th) * v, x[:, 1] + dt * lt * torch.sin(th) * v,
                      th + dt * at * w], dim=1)
    return xn, torch.linalg.norm(xn[:, :2] - goal, dim=1) <= tol


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2", choices=["c2", "c3", "bb", "ref"])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--closed-loop", type=int, default=40)
    ap.add_argument("--parity-steps", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--graph-steps", type=int, default=1)
    args = ap.parse_args()
    if args.graph_steps < 1:
        ap.error("--graph-steps must be >= 1")
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from bench_batch import gpu_info
    from tests.scenarios import make_scenario
    from tests.trial_loop import plant_step, within
    K, S = args.batch, args.closed_loop
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bb = args.workload == "bb"
    stochastic = False
    if bb:
        params = _bb_params(K)
        with contextlib.redirect_stdout(io.StringIO()):
            A, Bs = _bb_planners(params), _bb_planners(params)
        starts = [(q["x0"].copy(), None) for q in params]
        grids = None
        Batch = E.MPPI_Batch
    else:
        mode, N, M, T, H, res, B, da = LOCAL_WORKLOADS.get(args.workload) or WORKLOADS[args.workload]
        stochastic = mode == "tdm"
        Batch = E.MPPI_StochasticBatch if stochastic else E.MPPI_Batch
        scs = []
        for k in range(K):
            sc = make_scenario(mode, N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=k + 1, det_alpha=da, warm_start=True)
            if k % 2 == 0:
                sc["params"]["xgoal"] = sc["params"]["x0"][:2] + np.array([1.2, -0.9])
            scs.append(sc)
        rng = np.random.default_rng(7)
        grids = [E.TractionGrid(rng.uniform(0.3, 1.0, (H, H)), rng.uniform(0.3, 1.0, (H, H)), res=res) for _ in range(K)]
        with contextlib.redirect_stdout(io.StringIO()):
            A, Bs = [[make_planner(E, sc, 0)[3] for sc in scs] for _ in range(2)]
        starts = [(sc["params"]["x0"].copy(), sc["u0"]) for sc in scs]

    def reset(pls):
        for p, (x0, u0) in zip(pls, starts):
            p.params["x0"] = x0.copy()
            if u0 is not None:
                p.u_cur_d.copy_to_device(u0)

    def trials(b):
        if bb:
            return b.run_barebone_trials(S)
        return b.run_stochastic_trials(grids, S) if stochastic else b.run_trials(grids, S)

    f64 = dict(dtype=torch.float64, device=dev)
    dt = torch.tensor([float(p.params["dt"]) for p in A], **f64)
    goal = torch.tensor(np.stack([np.asarray(p.params["xgoal"], np.float64)[:2] for p in A]), **f64)
    tol = torch.tensor([float(p.params["goal_tolerance"]) for p in A], **f64)
    if grids is None:
        tg, xlo, ylo, gres = None, 0.0, 0.0, 1.0
    else:
        tg = (torch.tensor(np.stack([g.lin_traction for g in grids]), **f64),
              torch.tensor(np.stack([g.ang_traction for g in grids]), **f64))
        xlo, ylo, gres = float(grids[0].xlimits[0]), float(grids[0].ylimits[0]), float(grids[0].res)

    def loop_round(steps, record=None):
        reset(A)
        x = torch.tensor(np.stack([np.asarray(p.params["x0"], np.float64)[:3] for p in A]), **f64)
        with ba.device_loop() as loop:
            for _ in range(steps):
                u = torch.as_tensor(loop.solve(), device=dev)
                if record is not None:
                    record.append(("solve", u.cpu().numpy().copy()))
                x, done = torch_plant(torch, x, u[:, 0], dt, tg, xlo, ylo, gres, goal, tol)
                loop.stop(done)
                loop.shift_and_update(x)
                if record is not None:
                    record.append(("stop", done.cpu().numpy()))
                    record.append(("shift", x.cpu().numpy()))
        torch.cuda.synchronize(dev)
        return loop

    G = args.graph_steps
    main_stream, side = torch.cuda.current_stream(dev), torch.cuda.Stream(dev)   # a capture needs a stream of its own
    U = [torch.empty((K, A[0].num_steps, 2), dtype=torch.float32, device=dev) for _ in range(G)]
    xs = torch.empty((K, 3), **f64)
    done = [torch.empty(K, dtype=torch.bool, device=dev) for _ in range(G)]
    xrec = [torch.empty((K, 3), **f64) for _ in range(G)]
    capture_seconds = []                                   # host time of each capture, instantiation included

    def graph_round(steps, record=None):
        """The device_loop leg's step with static tensors: one eager step, then G of them captured and replayed."""
        reset(A)
        ba.set_stream(side.cuda_stream)
        with torch.cuda.stream(side):
            xs.copy_(torch.tensor(np.stack([np.asarray(p.params["x0"], np.float64)[:3] for p in A]), **f64))

            def step(loop, j):
                loop.solve(out=U[j])
                xn, d = torch_plant(torch, xs, U[j][:, 0], dt, tg, xlo, ylo, gres, goal, tol)
                xs.copy_(xn)
                done[j].copy_(d)
                loop.stop(done[j])
                loop.shift_and_update(xs)
                if record is not None:
                    xrec[j].copy_(xs)

            def keep(n):
                for j in range(n):
                    record.append(("solve", U[j].cpu().numpy().copy()))
                    record.append(("stop", done[j].cpu().numpy()))
                    record.append(("shift", xrec[j].cpu().numpy()))

            with ba.device_loop() as loop:
                step(loop, 0)
                if record is not None:
                    keep(1)
                g = torch.cuda.CUDAGraph()
                t0 = time.perf_counter()
                g.capture_begin()
                for j in range(G):
                    step(loop, j)
                g.capture_end()
                capture_seconds.append(time.perf_counter() - t0)
                for _ in range(-(-(steps - 1) // G)):
                    g.replay()
                    if record is not None:
                        keep(G)
        torch.cuda.synchronize(dev)
        ba.set_stream(main_stream.cuda_stream)
        return loop

    ba, bh = Batch(A), Batch(Bs)
    for b in (ba, bh):                                     # the torch plant, the loop and torch's reads on one stream
        b.set_stream(main_stream.cuda_stream)

    # ---- parity: the device loop (then the graph-replayed loop) == the host loop replayed with the loop's poses on
    # identical twins
    def replayed_on_twins(calls):
        reset(Bs)
        ok_u = True
        for k, p in enumerate(Bs):
            one, running = Batch([p]), True
            for what, v in calls:
                if what == "solve":
                    if running:
                        u = one.solve()[0]
                        ok_u &= u.tobytes() == v[k].tobytes()
                    else:
                        ok_u &= bool(np.isnan(v[k]).all())
                elif what == "stop" and running and v[k]:
                    running = False
                elif what == "shift" and running:
                    p.shift_and_update(v[k].copy(), p.u_cur_d.copy_to_host(), 1)
                    running = bb or within(p, v[k])
        return ok_u

    def state(p):
        d = [p.u_cur_d, p.u_prev_d, p.costs_d, p.weights_d, p.noise_samples_d, p.rng_states_d]
        if not bb:
            d += [p.lin_tdm.rng_states_d, p.ang_tdm.rng_states_d, p.lin_tdm.sample_grid_batch_d,
                  p.ang_tdm.sample_grid_batch_d]
        if stochastic:
            d.append(p.costs_nm_d)
        return [a.copy_to_host() for a in d] + [np.asarray(p.params["x0"], np.float64)]

    parity = {"planners": K, "steps": args.parity_steps,
              "against": "the host loop replayed with the loop's poses on identical twins"}
    for name, fn in (("device_loop", loop_round), ("graph", graph_round)):
        calls = []
        with contextlib.redirect_stdout(io.StringIO()):
            loop = fn(args.parity_steps, calls)
            ok_u = replayed_on_twins(calls)
        ok_state = all(all(np.array_equal(x, y) for x, y in zip(state(a), state(b))) for a, b in zip(A, Bs))
        parity[name] = {"passed": bool(ok_u and ok_state), "u_bitwise": bool(ok_u), "state_bitwise": bool(ok_state),
                        "solves": loop.solves.tolist(), "status": loop.status}
    parity["passed"] = parity["device_loop"]["passed"] and parity["graph"]["passed"]
    if not parity["passed"]:
        sys.stderr.write("bench_loop.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        print(json.dumps({"metric": "device loop", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    def host_round():
        reset(Bs)
        x = [np.asarray(p.params["x0"], dtype=np.float64) for p in Bs]
        running = list(range(K))
        for _ in range(S):
            u = bh.solve()
            still = []
            for k in running:
                p = Bs[k]
                if bb:
                    th, dtk = x[k][2], float(p.params["dt"])
                    xn = np.array([x[k][0] + dtk * np.cos(th) * float(u[k, 0, 0]),
                                   x[k][1] + dtk * np.sin(th) * float(u[k, 0, 0]), th + dtk * float(u[k, 0, 1])])
                else:
                    xn = plant_step(grids[k], x[k], u[k, 0], float(p.params["dt"]))
                p.shift_and_update(xn, u[k], 1)
                x[k] = xn
                d = np.linalg.norm(xn[:2] - p.params["xgoal"]) - p.params["goal_tolerance"]
                if d > 0 and (bb or within(p, xn)):
                    still.append(k)
            running = still
            if not running:
                break
        torch.cuda.synchronize(dev)

    def trials_round():
        reset(A)
        trials(ba)
        torch.cuda.synchronize(dev)

    legs = [("device_loop", lambda: loop_round(S), ba), ("graph", lambda: graph_round(S), ba), ("host", host_round, bh),
            ("run_trials", trials_round, ba)]
    times = {name: [] for name, _, _ in legs}
    launches = {}
    with contextlib.redirect_stdout(io.StringIO()):
        for _, fn, _ in legs:                              # warm-up
            fn()
        del capture_seconds[:]
        for _ in range(args.rounds):
            for name, fn, b in legs:
                n0 = b.launch_count()
                t0 = time.perf_counter()
                fn()
                times[name].append(time.perf_counter() - t0)
                launches[name] = b.launch_count() - n0
    med = {name: float(np.median(v)) for name, v in times.items()}
    out = {"metric": "device loop: caller's torch plant vs host loop vs run_trials",
           "config": {"workload": args.workload, "batch": K, "steps": S, "rounds": args.rounds,
                      "plant": "unicycle on a float64 traction grid in torch" if not bb else "nominal unicycle in torch",
                      "device_loop": "S solves, plant, stop at goal, shift: no host poll, all S steps issued",
                      "graph_steps": G,
                      "graph": "one eager step, G steps captured, ceil((S - 1) / G) replays; open, capture, close "
                               "included"},
           "gpu": gpu_info(dev), "parity_check": parity,
           "round_seconds": {name: [round(t, 4) for t in v] for name, v in times.items()},
           "median_seconds": {name: round(t, 4) for name, t in med.items()},
           "host_over_device_loop": round(med["host"] / med["device_loop"], 3),
           "device_loop_over_run_trials": round(med["device_loop"] / med["run_trials"], 3),
           "device_loop_over_graph": round(med["device_loop"] / med["graph"], 3),
           "graph_capture_seconds": [round(t, 4) for t in capture_seconds],
           "launches_per_round": launches}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
