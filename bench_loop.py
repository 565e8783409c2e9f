#!/usr/bin/env python
"""bench_loop.py -- the receding-horizon loop with the caller's plant: the device loop against the host loop.

    python bench_loop.py --workload c2|c3|bb|ref --batch K --closed-loop S [--rounds R] [--graph-steps G]
    python bench_loop.py --workload swarm --batch K --closed-loop S [--rounds R] [--graph-steps G] [--profile]

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
nothing to the tree.

swarm: K barebone robots of the notebook's shape (N 1000, T 50, dt 0.1, its two obstacles) in one arena, started on a
circle around it and each cycling through its own waypoints across the arena, so their paths cross.  Every step, each
robot's obstacles are the two static ones plus the other K - 1 robots' current positions (radius 0.3), and a robot
within 0.5 of its goal moves on to its next waypoint: the task changes at every step, from GPU memory
(loop.set_goals, loop.set_obstacles).  The parity check is as above, with the goal and obstacle calls replayed through
params['xgoal'], params['obstacle_positions'] and params['obstacle_radius'].  Legs: device_loop, graph (the goals and
obstacles computed and set inside the graph) and host (batch.solve(), then per robot the numpy plant step,
shift_and_update and the new params); no run_trials leg, as the built-in plant has no moving obstacles.  --profile
instead runs the device loop under torch.profiler (a run of its own) and reports each kernel's GPU time per step, with
the robots as obstacles and with the two static obstacles only: whether the barebone rollout's per-step obstacle loop
bounds the step."""
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
    ap.add_argument("--workload", default="c2", choices=["c2", "c3", "bb", "ref", "swarm"])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--closed-loop", type=int, default=40)
    ap.add_argument("--parity-steps", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--graph-steps", type=int, default=1)
    ap.add_argument("--profile", action="store_true", help="swarm: kernel times per step under torch.profiler")
    args = ap.parse_args()
    if args.graph_steps < 1:
        ap.error("--graph-steps must be >= 1")
    if args.workload == "swarm":
        return run_swarm(args)
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


SWARM_STATIC = [[5.0, 4.5, 1.5], [2.0, 1.0, 1.0]]     # the notebook's two obstacles
SWARM_R, SWARM_CENTRE, SWARM_RADIUS, SWARM_WAYPOINTS = 0.3, (3.5, 2.75), 6.0, 3


def swarm_params(K):
    """Robot k starts on a circle of radius 6 around the arena's centre, heading in, and its waypoints are the points of
    the circle 90, 180 and 270 degrees on; the notebook's planner otherwise (the bb workload's params)."""
    cx, cy = SWARM_CENTRE
    params, ways = [], []
    for k in range(K):
        a = 2 * np.pi * k / K
        x0 = np.array([cx + SWARM_RADIUS * np.cos(a), cy + SWARM_RADIUS * np.sin(a), a + np.pi])
        w = [[cx + SWARM_RADIUS * np.cos(a + np.pi * (j + 1) / 2), cy + SWARM_RADIUS * np.sin(a + np.pi * (j + 1) / 2)]
             for j in range(SWARM_WAYPOINTS)]
        ways.append(w)
        params.append(dict(dt=0.1, x0=x0, xgoal=np.array(w[0]), goal_tolerance=0.5, dist_weight=10, lambda_weight=1.0,
                           num_opt=1, u_std=np.array([1.0, 1.0]), vrange=np.array([0.0, 2.0]),
                           wrange=np.array([-np.pi, np.pi]), obstacle_positions=np.array(SWARM_STATIC)[:, :2],
                           obstacle_radius=np.array(SWARM_STATIC)[:, 2], obs_penalty=1e6))
    return params, np.array(ways)


def run_swarm(args):
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from bench_batch import gpu_info
    K, S, G = args.batch, args.closed_loop, args.graph_steps
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    params, ways = swarm_params(K)
    with contextlib.redirect_stdout(io.StringIO()):
        A, Bs = _bb_planners(params), _bb_planners(params)
    Op = 2 + K - 1
    f64 = dict(dtype=torch.float64, device=dev)
    dt = torch.full((K,), 0.1, **f64)
    W = torch.tensor(ways, **f64)                          # (K, P, 2)
    rows = torch.arange(K, device=dev)
    others = torch.tensor([[j for j in range(K) if j != k] for k in range(K)], device=dev)
    static = torch.tensor(SWARM_STATIC, **f64).expand(K, 2, 3)
    radius = torch.full((K, K - 1, 1), SWARM_R, **f64)
    main_stream, side = torch.cuda.current_stream(dev), torch.cuda.Stream(dev)

    def reset(pls):
        for p, q in zip(pls, params):
            p.params["x0"] = q["x0"].copy()
            p.params["xgoal"] = q["xgoal"].copy()
            p.params["obstacle_positions"] = q["obstacle_positions"].copy()
            p.params["obstacle_radius"] = q["obstacle_radius"].copy()
            p.u_cur_d.copy_to_device(np.zeros((p.num_steps, 2), np.float32))

    class State(object):
        """The device-side step: plant, waypoint switch, obstacles from the robots' positions (static tensors)."""

        def __init__(self, static_only=False):
            self.x = torch.tensor(np.stack([q["x0"] for q in params]), **f64)
            self.widx = torch.zeros(K, dtype=torch.int64, device=dev)
            self.g = W[rows, self.widx].clone()
            self.obs = torch.zeros((K, Op, 3), **f64)
            self.counts = torch.full((K,), 2 if static_only else Op, dtype=torch.int32, device=dev)

        def step(self, loop, u, record=None):
            v, w = torch.nan_to_num(u[:, 0, 0].double()), torch.nan_to_num(u[:, 0, 1].double())
            th = self.x[:, 2]
            self.x.copy_(torch.stack([self.x[:, 0] + dt * torch.cos(th) * v, self.x[:, 1] + dt * torch.sin(th) * v,
                                      th + dt * w], dim=1))
            loop.shift_and_update(self.x)
            near = torch.linalg.norm(self.x[:, :2] - self.g, dim=1) <= 0.5
            self.widx.copy_((self.widx + near.long()) % SWARM_WAYPOINTS)
            self.g.copy_(W[rows, self.widx])
            loop.set_goals(self.g)
            self.obs.copy_(torch.cat([static, torch.cat([self.x[others, :2], radius], dim=2)], dim=1))
            loop.set_obstacles(self.obs, self.counts)
            if record is not None:
                record.append(("shift", self.x.cpu().numpy()))
                record.append(("goals", self.g.cpu().numpy()))
                record.append(("obstacles", self.obs.cpu().numpy(), self.counts.cpu().numpy()))

    ba, bh = E.MPPI_Batch(A), E.MPPI_Batch(Bs)
    for b in (ba, bh):
        b.set_stream(main_stream.cuda_stream)

    def loop_round(steps, record=None, static_only=False):
        reset(A)
        st = State(static_only)
        with ba.device_loop(max_obstacles=Op) as loop:
            for _ in range(steps):
                u = torch.as_tensor(loop.solve(), device=dev)
                if record is not None:
                    record.append(("solve", u.cpu().numpy().copy()))
                st.step(loop, u, record)
        torch.cuda.synchronize(dev)
        return loop

    U = [torch.empty((K, A[0].num_steps, 2), dtype=torch.float32, device=dev) for _ in range(G)]
    capture_seconds = []

    def graph_round(steps, record=None):
        reset(A)
        ba.set_stream(side.cuda_stream)
        with torch.cuda.stream(side):
            st = State()

            def step(loop, j):
                loop.solve(out=U[j])
                st.step(loop, U[j])

            def keep(j):
                record.append(("solve", U[j].cpu().numpy().copy()))
                record.append(("shift", st.x.cpu().numpy()))
                record.append(("goals", st.g.cpu().numpy()))
                record.append(("obstacles", st.obs.cpu().numpy(), st.counts.cpu().numpy()))

            with ba.device_loop(max_obstacles=Op) as loop:
                step(loop, 0)
                if record is not None:
                    keep(0)
                g = torch.cuda.CUDAGraph()
                t0 = time.perf_counter()
                g.capture_begin()
                for j in range(G):
                    step(loop, j)
                g.capture_end()
                capture_seconds.append(time.perf_counter() - t0)
                for _ in range(-(-(steps - 1) // G)):
                    g.replay()
                    if record is not None:                 # G 1 in the parity check: the step's own state
                        keep(0)
        torch.cuda.synchronize(dev)
        ba.set_stream(main_stream.cuda_stream)
        return loop

    def replayed_on_twins(calls):
        reset(Bs)
        ok = True
        for k, p in enumerate(Bs):
            one = E.MPPI_Batch([p])
            for c in calls:
                if c[0] == "solve":
                    ok &= one.solve()[0].tobytes() == c[1][k].tobytes()
                elif c[0] == "shift":
                    p.shift_and_update(c[1][k].copy(), p.u_cur_d.copy_to_host(), 1)
                elif c[0] == "goals":
                    p.params["xgoal"] = c[1][k].copy()
                else:
                    n = int(c[2][k])
                    p.params["obstacle_positions"] = c[1][k, :n, :2].copy()
                    p.params["obstacle_radius"] = c[1][k, :n, 2].copy()
        return ok

    def state(p):
        return [a.copy_to_host() for a in (p.u_cur_d, p.u_prev_d, p.costs_d, p.weights_d, p.noise_samples_d,
                                           p.rng_states_d)] + [np.asarray(p.params[q], np.float64) for q in
                                                               ("x0", "xgoal", "obstacle_positions", "obstacle_radius")]

    if args.profile:
        return swarm_profile(torch, dev, K, S, loop_round, gpu_info)

    parity = {"planners": K, "steps": args.parity_steps,
              "against": "the host loop replayed with the loop's poses, goals and obstacles on identical twins"}
    for name, fn in (("device_loop", loop_round), ("graph", graph_round)):
        if name == "graph" and G != 1:
            continue                                       # the parity record keeps one step's state per replay
        calls = []
        with contextlib.redirect_stdout(io.StringIO()):
            fn(args.parity_steps, calls)
            ok_u = replayed_on_twins(calls)
        ok_state = all(all(np.array_equal(x, y) for x, y in zip(state(a), state(b))) for a, b in zip(A, Bs))
        parity[name] = {"passed": bool(ok_u and ok_state), "u_bitwise": bool(ok_u), "state_bitwise": bool(ok_state)}
    parity["passed"] = all(v["passed"] for k, v in parity.items() if isinstance(v, dict))
    if not parity["passed"]:
        sys.stderr.write("bench_loop.py: PARITY CHECK FAILED: %s\n" % json.dumps(parity))
        print(json.dumps({"metric": "device loop swarm", "error": "parity_check failed", "parity_check": parity}))
        raise SystemExit(3)

    def host_round():
        reset(Bs)
        x = [q["x0"].copy() for q in params]
        widx = [0] * K
        for _ in range(S):
            u = bh.solve()
            for k, p in enumerate(Bs):
                th = x[k][2]
                x[k] = np.array([x[k][0] + 0.1 * np.cos(th) * float(u[k, 0, 0]),
                                 x[k][1] + 0.1 * np.sin(th) * float(u[k, 0, 0]), th + 0.1 * float(u[k, 0, 1])])
                p.shift_and_update(x[k], u[k], 1)
            for k, p in enumerate(Bs):
                if np.linalg.norm(x[k][:2] - ways[k][widx[k]]) <= 0.5:
                    widx[k] = (widx[k] + 1) % SWARM_WAYPOINTS
                p.params["xgoal"] = ways[k][widx[k]].copy()
                pos = np.array([x[j][:2] for j in range(K) if j != k]).reshape(-1, 2)
                p.params["obstacle_positions"] = np.concatenate([np.array(SWARM_STATIC)[:, :2], pos])
                p.params["obstacle_radius"] = np.concatenate([np.array(SWARM_STATIC)[:, 2], np.full(K - 1, SWARM_R)])
        torch.cuda.synchronize(dev)

    legs = [("device_loop", lambda: loop_round(S), ba), ("graph", lambda: graph_round(S), ba), ("host", host_round, bh)]
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
    print(json.dumps({
        "metric": "device loop swarm: goals and obstacles from GPU memory every step vs the host loop",
        "config": {"workload": "swarm", "batch": K, "steps": S, "rounds": args.rounds, "obstacles_per_robot": Op,
                   "N": A[0].num_control_rollouts, "T": A[0].num_steps, "graph_steps": G,
                   "device_loop": "S x (solve, torch plant, shift, waypoint switch, set_goals, set_obstacles)",
                   "graph": "one eager step, G steps captured, ceil((S - 1) / G) replays; open, capture, close included",
                   "host": "S x (batch.solve(), numpy plant, shift_and_update, params xgoal and obstacles)"},
        "gpu": gpu_info(dev), "parity_check": parity,
        "round_seconds": {name: [round(t, 4) for t in v] for name, v in times.items()},
        "median_seconds": {name: round(t, 4) for name, t in med.items()},
        "host_over_device_loop": round(med["host"] / med["device_loop"], 3),
        "device_loop_over_graph": round(med["device_loop"] / med["graph"], 3),
        "graph_capture_seconds": [round(t, 4) for t in capture_seconds],
        "launches_per_round": launches}))


def swarm_profile(torch, dev, K, S, loop_round, gpu_info):
    """Each kernel's GPU time per step of the swarm's device loop under torch.profiler, with the K + 1 obstacles and
    with the two static ones only (counts 2), and the step's wall time without the profiler."""
    from torch.profiler import ProfilerActivity, profile
    out = {"metric": "device loop swarm: kernel time per step (torch.profiler)", "gpu": gpu_info(dev),
           "config": {"batch": K, "steps": S, "obstacles_per_robot": {"robots": K + 1, "static_only": 2}}}
    with contextlib.redirect_stdout(io.StringIO()):
        for static_only in (False, True):
            loop_round(S, static_only=static_only)        # warm-up
            t0 = time.perf_counter()
            loop_round(S, static_only=static_only)
            wall = (time.perf_counter() - t0) / S
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                loop_round(S, static_only=static_only)
            kern = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                if t > 0:
                    kern[e.key] = round(t / S, 2)         # microseconds per step
            total = sum(v for k, v in kern.items() if "Memcpy" not in k and "Memset" not in k)
            top = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:8])
            out["static_only" if static_only else "robots"] = {
                "step_wall_us": round(wall * 1e6, 1), "kernel_us_per_step": round(total, 1), "top_kernels_us": top}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
