"""Trial sequences on the GPU (run with ``-m gpu``): MPPI_Batch / MPPI_StochasticBatch.run_trial_sequences against the
same loops on identical twins -- one-episode sequences against run_trials, reset_x0 sequences against consecutive
run_trials calls with params['x0'] reset in between, the benchmark's loop (no reset) replayed from the device's
trajectory and driven fully from the host -- plus launch accounting."""
import functools

import numpy as np
import pytest

from tests import test_gpu_mixed_geometry_trials as MG
from tests import test_gpu_shared_tdm as SH
from tests.gpu_harness import (assert_same, eng, quiet, snapshot, solve_in_batch_of_one, tdm_scenario,  # noqa: F401
                               tdm_trial_setup, twins)
from tests.test_gpu_trials import trial_setup
from tests.trial_sequence_loop import host_sequence

pytestmark = pytest.mark.gpu

MAX_STEPS = 20


def episode_grids(E, grid, k, n):
    """n ground-truth grids of planner k: its own, then n - 1 more of the same geometry and kind."""
    rng = np.random.default_rng(700 + k)
    shape, int8 = grid.lin_traction.shape, grid.lin_traction.dtype == np.int8
    return [grid] + [E.TractionGrid(rng.uniform(0.2, 1.0, shape), rng.uniform(0.2, 1.0, shape), res=grid.res,
                                    use_int8=int8, xlimits=grid.xlimits, ylimits=grid.ylimits) for _ in range(n - 1)]


def setup(E, mode, num_opt=1):
    """(A, B, grids, batch class, solve of one planner) for a kind: det / spd (tests/test_gpu_trials.py) or stochastic
    (tdm_trial_setup) planners 0..4: goal within a step, a nearby goal, out of reach, (det) far goal / (tdm) the map's
    corner, and an int8 grid that throws the robot off the map."""
    if mode == "tdm":
        A, B, grids = twins(functools.partial(tdm_trial_setup, E, num_opt=num_opt), 5)
        return A, B, grids, E.MPPI_StochasticBatch, solve_in_batch_of_one
    A, B, grids = twins(functools.partial(trial_setup, E, mode), 5)
    return A, B, grids, E.MPPI_Batch, lambda p: p.solve()


def run_trials(batch, grids, S):
    f = batch.run_stochastic_trials if batch.kind == "tdm" else batch.run_trials
    return f(grids, S)


def replay_sequences(A, B, out, solve_one, reset_x0):
    """The host sequence loop fed with the device's trajectory on the twins B: u[0] of every solve bit for bit, NaN
    exactly where nothing ran, then every buffer, params['x0'] and one more solve()."""
    for k, p in enumerate(B):
        x_start = np.array(p.params["x0"], dtype=np.float64)
        run = int(out["episodes_run"][k])
        assert out["status"][k][run:] == ["not_run"] * (len(out["status"][k]) - run)
        assert all(log is None for log in out["logs"][k][run:]) and (out["steps"][k, run:] == 0).all()
        assert np.isnan(out["xhist"][k, run:]).all() and np.isnan(out["uhist"][k, run:]).all()
        with quiet():
            for e in range(run):
                n = int(out["steps"][k, e])
                assert np.array_equal(out["xhist"][k, e, 0], x_start)
                assert not np.isnan(out["xhist"][k, e, :n + 1]).any() and np.isnan(out["xhist"][k, e, n + 1:]).all()
                assert np.isnan(out["uhist"][k, e, n:]).all()
                if reset_x0:
                    p.params["x0"] = x_start.copy()
                for t in range(n):
                    useq = solve_one(p)
                    assert_same({"u[0]": useq[0]}, {"u[0]": out["uhist"][k, e, t]},
                                "planner %d episode %d step %d" % (k, e, t))
                    p.shift_and_update(out["xhist"][k, e, t + 1], useq, 1)
        assert_same(snapshot(A[k]), snapshot(p), "planner %d" % k)
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=p.params["x0"]), "planner %d" % k)
    with quiet():
        for k in range(len(A)):
            ua, ub = A[k].solve(), B[k].solve()
            if out["status"][k][int(out["episodes_run"][k]) - 1] == "left_map":
                assert ua is None and ub is None
            else:
                assert_same(dict(u=ua), dict(u=ub), "planner %d: the next solve" % k)
                assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d after one more solve" % k)


@pytest.mark.parametrize("mode", ["det", "spd", "tdm"])
def test_one_episode_equals_run_trials(eng, mode):
    E = eng
    A, B, grids, cls, _ = setup(E, mode)
    ba, bb = cls(A), cls(B)
    with quiet():
        out = ba.run_trial_sequences([[g] for g in grids], MAX_STEPS)
        want = run_trials(bb, grids, MAX_STEPS)
    assert_same(dict(xhist=out["xhist"][:, 0], uhist=out["uhist"][:, 0], steps=out["steps"][:, 0]),
                {k: want[k] for k in ("xhist", "uhist", "steps")}, "histories")
    assert [s[0] for s in out["status"]] == want["status"] and out["episodes_run"].tolist() == [1] * 5
    for k in range(5):
        assert_same({n: np.asarray(v) for n, v in out["logs"][k][0].items()},
                    {n: np.asarray(v) for n, v in want["logs"][k].items()}, "planner %d: log" % k)
        assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d" % k)
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=B[k].params["x0"]), "planner %d" % k)
    assert ba.steps_issued == bb.steps_issued and ba.launch_count() == bb.launch_count()


def reset_cases(E, case):
    if case == "shared":
        # every goal out of reach: each member runs every episode to max_steps, so the shared pair is sampled as often in
        # the sequence as in the consecutive calls (in general a shared pair follows its members' total steps)
        sc = tdm_scenario(1, H=128)
        goals = [(50.0, 50.0)] * 4
        A = SH.build(E, sc, 4, shared=True, goals=goals)
        B = SH.build(E, sc, 4, shared=True, goals=goals)
        grids = SH._grids(E, 4, 128, 0.2)
        return A, B, grids, functools.partial(E.MPPI_StochasticBatch, share_tdms=True)
    A, B, grids, cls, _ = setup(E, case)
    return A, B, grids, cls


@pytest.mark.parametrize("case", ["det", "tdm", "shared"])
def test_reset_equals_consecutive_run_trials(eng, case):
    """reset_x0=True == E run_trials calls on the twins with params['x0'] set back to the start before each: histories,
    logs, every buffer, RNG stream, sampled map, sample_box() and params['x0'], bit for bit."""
    E = eng
    A, B, grids, cls = reset_cases(E, case)
    K, n_ep, S = len(A), 3, 12
    seqs = [episode_grids(E, g, k, n_ep) for k, g in enumerate(grids)]
    starts = [np.array(p.params["x0"], dtype=np.float64) for p in B]
    with quiet():
        out = cls(A).run_trial_sequences(seqs, S, reset_x0=True)
        bb = cls(B)
        for e in range(n_ep):
            for k, p in enumerate(B):
                p.params["x0"] = starts[k].copy()
            want = run_trials(bb, [seqs[k][e] for k in range(K)], S)
            assert_same(dict(xhist=out["xhist"][:, e], uhist=out["uhist"][:, e], steps=out["steps"][:, e]),
                        {k: want[k] for k in ("xhist", "uhist", "steps")}, "episode %d" % e)
            assert [s[e] for s in out["status"]] == want["status"]
            for k in range(K):
                assert_same({n: np.asarray(v) for n, v in out["logs"][k][e].items()},
                            {n: np.asarray(v) for n, v in want["logs"][k].items()}, "planner %d episode %d" % (k, e))
    print(case, "status", out["status"])
    assert (out["episodes_run"] == n_ep).all()
    for k in range(K):
        assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d" % k)
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=B[k].params["x0"]), "planner %d" % k)
        if case != "det":
            assert list(A[k].sample_box()) == list(B[k].sample_box())


# ragged episode counts; planner 4's int8 grids throw it off the map (its sequence ends there, the rest not_run)
EPISODES = [2, 5, 1, 2, 3]


@pytest.mark.parametrize("case", ["det", "spd", "tdm", "tdm_num_opt2", "tdm_mixed"])
def test_benchmark_loop_replay(eng, case):
    E = eng
    if case == "tdm_mixed":
        specs = MG.SPECS[:5]
        A, B = MG.build(E, "tdm", specs), MG.build(E, "tdm", specs)
        grids = [MG.grid_of(E, k, s) for k, s in enumerate(specs)]
        cls, solve_one = E.MPPI_StochasticBatch, solve_in_batch_of_one
        episodes = [2, 5, 1, 3, 2]                   # planner 3 (kind 4) leaves its map
    else:
        A, B, grids, cls, solve_one = setup(E, case[:3], num_opt=2 if case.endswith("2") else 1)
        episodes = EPISODES
    seqs = [episode_grids(E, g, k, n) for k, (g, n) in enumerate(zip(grids, episodes))]
    batch = cls(A)
    with quiet():
        out = batch.run_trial_sequences(seqs, MAX_STEPS)
    print(case, "steps", out["steps"].tolist(), "status", out["status"])
    assert out["xhist"].shape == (5, 5, MAX_STEPS + 1, 3) and out["uhist"].shape == (5, 5, MAX_STEPS, 2)
    assert [len(s) for s in out["status"]] == episodes and [len(v) for v in out["logs"]] == episodes
    assert any("left_map" in s[:-1] and s[-1] == "not_run" for s in out["status"])
    # a later episode of one step: the last solve planned from the previous episode's final pose
    assert any(out["episodes_run"][k] > 1 and out["steps"][k, out["episodes_run"][k] - 1] == 1 for k in range(5))
    total = out["steps"].sum(axis=1).max()
    assert total <= batch.steps_issued <= total + 4
    replay_sequences(A, B, out, solve_one, reset_x0=False)


@pytest.mark.parametrize("reset_x0", [False, True])
def test_host_driven_sequences(eng, reset_x0):
    """Against host_sequence on the twins: the same status and steps, trajectories and logs within 1e-9."""
    E = eng
    A, B, grids, cls, _ = setup(E, "det")
    seqs = [episode_grids(E, g, k, n) for k, (g, n) in enumerate(zip(grids, EPISODES))]
    with quiet():
        out = cls(A).run_trial_sequences(seqs, MAX_STEPS, reset_x0=reset_x0)
        host = [host_sequence(p, s, MAX_STEPS, reset_x0=reset_x0) for p, s in zip(B, seqs)]
    for k, eps in enumerate(host):
        for e, h in enumerate(eps):
            if h is None:
                assert out["status"][k][e] == "not_run" and out["logs"][k][e] is None
                continue
            log, xh, uh, n, status = h
            assert out["status"][k][e] == status and out["steps"][k, e] == n, (k, e)
            assert np.allclose(out["xhist"][k, e], xh, rtol=0, atol=1e-9, equal_nan=True)
            assert np.allclose(out["uhist"][k, e], uh, rtol=0, atol=1e-9, equal_nan=True)
            for key, v in log.items():
                w = out["logs"][k][e][key]
                if isinstance(v, bool):
                    assert w == v
                else:
                    assert (np.isnan(v) and np.isnan(w)) or abs(w - v) <= 1e-9 * max(1.0, abs(v)), (k, e, key, w, v)
        assert np.allclose(A[k].params["x0"], B[k].params["x0"], rtol=0, atol=1e-9)


@pytest.mark.parametrize("mode,per_step", [("det", 5), ("tdm", 7)])
def test_launches_per_step_as_run_trials(eng, mode, per_step):
    E = eng
    A, _, grids, cls, _ = setup(E, mode)
    batch = cls(A)
    seqs = [episode_grids(E, g, k, n) for k, (g, n) in enumerate(zip(grids, EPISODES))]
    l0 = batch.launch_count()
    with quiet():
        out = batch.run_trial_sequences(seqs, MAX_STEPS)
    assert batch.launch_count() - l0 == per_step * batch.steps_issued
    total = int(out["steps"].sum(axis=1).max())
    assert total <= batch.steps_issued <= total + 4
