"""Closed-loop trials of batches whose planners' maps differ in size, resolution and bin count, on the GPU (run with
``-m gpu``).  The planners fall into launch classes (the same padded bins, thread tile and number of maps): a step
issues one sampler launch per class (stochastic: and one state advance; recorded: one completion).  Every case holds
the device trials against the host loop on identical twins, replayed from the device's trajectory (controls, every
planner buffer, RNG streams, sampled maps, sample_box() and the next solve bit for bit), with a map smaller than the
rollout window, a robot that leaves its map and a start whose box leaves the map; with shared and private pairs mixed
the twins run the shared batch's own solve() each step.  Launch counts follow 3 num_opt + 1 + C (one-map) and
4 num_opt + 1 + 2 C (stochastic) per step for C classes, the completion counted C times.  An unfused pair is still
refused with nothing issued."""
import numpy as np
import pytest

from tests.gpu_harness import (assert_same, eng, planner_launches, quiet, replay, snapshot,  # noqa: F401
                               solve_in_batch_of_one, tdm_pair, vary)
from tests.scenarios import make_scenario

pytestmark = pytest.mark.gpu

MAX_STEPS = 12
# (kind, H, res, bins) per planner.  kind: 0 goal within a step, 1 a nearby goal, 2 goal out of reach, 3 start near the
# map's corner (the box leaves the map), 4 an int8 ground-truth grid that throws the robot off its map.  5 bins pad to
# 8, 9 bins to 12: two launch classes.  The 12-cell map at 0.5 m is smaller than the rollout window.
SPECS = [(0, 64, 0.2, 5), (1, 48, 0.25, 9), (2, 12, 0.5, 9), (4, 40, 0.2, 5), (3, 56, 0.2, 9), (2, 72, 0.1, 5)]
ONE_CLASS = [(kind, H, res, 5) for kind, H, res, _ in SPECS]
GOALS = {0: (0.3, 0.3), 1: (0.9, -0.4), 2: (50.0, 50.0), 3: (1.5, 1.0), 4: (-1.5, 1.2)}


def scenario(mode, k, spec, num_opt=1):
    kind, H, res, B = spec
    sc = make_scenario(mode, N=200, M=24 if mode == "tdm" else 1, T=20, H=H, W=H, res=res, B=B, seed=23 + 5 * k,
                       warm_start=(k % 2 == 1), cvar_alpha=[0.5, 0.25, 1.0, 0.1][k % 4])
    sc = vary(sc, k)
    p = sc["params"]
    p["num_opt"] = num_opt
    p["dt"] = [0.1, 0.08, 0.12][k % 3]
    if kind == 3:
        p["x0"] = np.array([0.15, 0.3, 0.4])
    p["xgoal"] = np.asarray(p["x0"], dtype=np.float64)[:2] + np.asarray(GOALS[kind])
    return sc


def grid_of(E, k, spec):
    kind, H, res, _ = spec
    rng = np.random.default_rng(300 + k)
    return E.TractionGrid(rng.uniform(0.2, 1.0, (H, H)), rng.uniform(0.2, 1.0, (H, H)), res=res, use_int8=(kind == 4))


def build(E, mode, specs, num_opt=1, share=()):
    """The planners of `specs` (planner k on scenario(mode, k, specs[k])).  share: groups of planner indices on one TDM
    pair (the first member's map and PMF; each member keeps its own start, goal, lambda, u_std and dt)."""
    out = []
    pairs = {}
    with quiet():
        for k, spec in enumerate(specs):
            sc = scenario(mode, k, spec, num_opt)
            lead = next((g[0] for g in share if k in g), k)
            if lead not in pairs:
                cfg = E.Config(**sc["cfg"])
                pairs[lead] = (cfg,) + tdm_pair(E, cfg, sc["pmf_lin"], sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"],
                                                sc["unknown"])
            cfg, lin, ang = pairs[lead]
            pl = E.MPPI_Numba(cfg)
            params = sc["params"]
            if lead != k:                                     # a start and goal inside the shared pair's map
                lsc = scenario(mode, lead, specs[lead], num_opt)
                params = dict(params, x0=np.asarray(lsc["params"]["x0"], dtype=np.float64) + np.array([0.4, -0.3, 0.2]))
                params["xgoal"] = params["x0"][:2] + np.asarray(GOALS[specs[k][0]])
            pl.setup(params, lin, ang)
            if "u0" in sc:
                pl.u_cur_d.copy_to_device(sc["u0"])
            out.append(pl)
    return out


def classes(specs):
    return len({(B + 3) // 4 for _, _, _, B in specs})


def per_step(stochastic, num_opt, C):
    return 4 * num_opt + 1 + 2 * C if stochastic else 3 * num_opt + 1 + C


@pytest.mark.parametrize("case", ["two_classes", "one_class", "num_opt2", "record1", "record3"])
def test_stochastic_trials_replay(eng, case):
    E = eng
    specs = ONE_CLASS if case == "one_class" else SPECS
    num_opt = 2 if case == "num_opt2" else 1
    record_every = {"record1": 1, "record3": 3}.get(case)
    A, B = build(E, "tdm", specs, num_opt), build(E, "tdm", specs, num_opt)
    grids = [grid_of(E, k, s) for k, s in enumerate(specs)]
    batch = E.MPPI_StochasticBatch(A)
    with quiet():
        out = batch.run_stochastic_trials(grids, MAX_STEPS, record_every=record_every)
    steps, status = out["steps"], out["status"]
    print(case, "steps", steps.tolist(), "status", status, "boxes", [list(p.sample_box()) for p in A])
    C, n = classes(specs), batch.steps_issued
    rec = -(-n // record_every) * (1 + C) if record_every else 0
    assert batch.launch_count() == per_step(True, num_opt, C) * n + rec
    if record_every:                                                   # the records of a call without recording
        A2 = build(E, "tdm", specs, num_opt)
        with quiet():
            plain = E.MPPI_StochasticBatch(A2).run_stochastic_trials(grids, MAX_STEPS)
        assert_same({k: out[k] for k in ("xhist", "uhist", "steps")}, {k: plain[k] for k in ("xhist", "uhist", "steps")},
                    "histories with and without recording")
    replay(A, B, out, solve_in_batch_of_one)


@pytest.mark.parametrize("mode,record_every", [("det", None), ("spd", None), ("det", 3)])
def test_onemap_trials_replay(eng, mode, record_every):
    E = eng
    A, B = build(E, mode, SPECS), build(E, mode, SPECS)
    grids = [grid_of(E, k, s) for k, s in enumerate(SPECS)]
    batch = E.MPPI_Batch(A)
    with quiet():
        out = batch.run_trials(grids, MAX_STEPS, record_every=record_every)
    print(mode, "steps", out["steps"].tolist(), "status", out["status"])
    n = batch.steps_issued
    assert batch.launch_count() == per_step(False, 1, 2) * n + (-(-n // record_every) if record_every else 0)
    replay(A, B, out, lambda p: p.solve())


@pytest.mark.parametrize("mode", ["tdm", "det"])
def test_shared_and_private_pairs_in_two_classes(eng, mode):
    """share_tdms with planners 0 and 3 on one pair (5 bins), 1 and 4 on another (9 bins), the others private, every goal
    out of reach: the device trials against the shared batch's own solve() on twins, step by step."""
    E = eng
    specs = [(2, max(H, 24), res, B) for _, H, res, B in SPECS]
    share = [(0, 3), (1, 4)]
    A, Cs = build(E, mode, specs, share=share), build(E, mode, specs, share=share)
    grids = [grid_of(E, k, s) for k, s in enumerate(specs)]
    stochastic = mode == "tdm"
    cls = E.MPPI_StochasticBatch if stochastic else E.MPPI_Batch
    batch = cls(A, share_tdms=True)
    with quiet():
        out = (batch.run_stochastic_trials if stochastic else batch.run_trials)(grids, 6)
        assert all(s == "max_steps" for s in out["status"]), out["status"]
        host = cls(Cs, share_tdms=True)
        for t in range(6):
            u = host.solve()
            for k in range(len(Cs)):
                assert_same({"u[0]": u[k][0]}, {"u[0]": out["uhist"][k, t]}, "planner %d step %d" % (k, t))
                Cs[k].shift_and_update(out["xhist"][k, t + 1], u[k], 1)
    assert batch.launch_count() == per_step(stochastic, 1, 2) * 6
    for k in range(len(A)):
        assert_same(snapshot(A[k]), snapshot(Cs[k]), "planner %d" % k)
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=Cs[k].params["x0"]), "planner %d" % k)


@pytest.mark.parametrize("mode", ["tdm", "det"])
def test_unfused_pair_still_refused(eng, mode):
    E = eng
    A = build(E, mode, SPECS)
    grids = [grid_of(E, k, s) for k, s in enumerate(SPECS)]
    with quiet():
        A[4].lin_tdm.sample_grids()                                   # diverged lin / ang streams
    before = [snapshot(p) for p in A]
    batch = (E.MPPI_StochasticBatch if mode == "tdm" else E.MPPI_Batch)(A)
    with pytest.raises(E.B200MPPIError, match="planner 4: its TDM pair cannot join"):
        (batch.run_stochastic_trials if mode == "tdm" else batch.run_trials)(grids, 5)
    assert batch.launch_count() == 0
    for k, p in enumerate(A):
        assert_same(snapshot(p), before[k], "refused planner %d" % k)
    assert all(planner_launches(p) == 0 for p in A)
