"""Closed-loop trials on the GPU (run with ``-m gpu``): MPPI_Batch.run_trials against the same episodes driven from the
host on identical twins -- replayed from the device's trajectory (controls and every planner buffer bit for bit), the
plant step recomputed in numpy, and a fully host-driven episode -- plus launch accounting and the batch solve left
as it was."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_batch import _quiet, assert_same, map_planner, map_scenario, snapshot
from tests.trial_loop import host_trial, plant_step

pytestmark = pytest.mark.gpu

K_EACH = 5
MAX_STEPS = 30


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    assert E.device_count() >= 1, "GPU tests need a CUDA device"
    return E


def trial_setup(E, mode, k):
    """Planner k of a mode (its own map, seed and warm start) and its ground-truth grid.  k = 0, 1: goal within a
    step or a few; k = 2: goal out of reach (runs to MAX_STEPS); k = 3: goal a metre away on a ground-truth grid that
    extends beyond the map (negative offsets); k = 4: an int8 grid (TractionGrid's use_int8 stores 100 x traction, so
    the robot is 100 times faster) that throws the robot off the padded map."""
    sc = map_scenario(mode, k, N=256, T=16, H=40, res=0.2, B=6)
    p = sc["params"]
    L = 40 * 0.2
    rng = np.random.default_rng(100 + k + (0 if mode == "det" else 50))
    if k == 0:
        p["xgoal"] = p["x0"][:2] + 0.3
    elif k == 1:
        p["xgoal"] = p["x0"][:2] + np.array([0.9, -0.4])
    elif k == 3:
        p["xgoal"] = p["x0"][:2] + np.array([-0.8, 0.7])
    elif k == 4:
        p["xgoal"] = p["x0"][:2] + np.array([-1.5, 1.2])
    pl = map_planner(E, sc, k)
    if k == 3:
        grid = E.TractionGrid(rng.uniform(0.6, 1.0, (60, 70)), rng.uniform(0.6, 1.0, (60, 70)), res=0.2,
                              xlimits=(-2.3, 11.7), ylimits=(-1.9, 10.1))
    else:
        grid = E.TractionGrid(rng.uniform(0.2, 1.0, (40, 40)), rng.uniform(0.2, 1.0, (40, 40)), res=0.2,
                              use_int8=(k == 4))
    return pl, grid


def twins(E, mode):
    with _quiet():
        A = [trial_setup(E, mode, k) for k in range(K_EACH)]
        B = [trial_setup(E, mode, k) for k in range(K_EACH)]
    return [a[0] for a in A], [b[0] for b in B], [a[1] for a in A]


@pytest.mark.parametrize("mode", ["det", "spd"])
def test_replay_equality(eng, mode):
    """run_trials == the host loop replayed with the device's trajectory: u[0] of every solve bit for bit, then every
    planner buffer, RNG stream, sampled map and params['x0'] -- and one more solve() on both sets is identical."""
    E = eng
    A, B, grids = twins(E, mode)
    batch = E.MPPI_Batch(A)
    with _quiet():
        out = batch.run_trials(grids, MAX_STEPS)
    steps, status = out["steps"], out["status"]
    print(mode, "steps", steps.tolist(), "status", status)
    assert status[0] == "goal" and steps[0] == 1
    assert status[1] == "goal" and status[3] == "goal"
    assert status[2] == "max_steps" and steps[2] == MAX_STEPS
    assert status[4] == "left_map"
    for k, p in enumerate(B):
        n = int(steps[k])
        with _quiet():
            for t in range(n):
                useq = p.solve()
                assert np.array_equal(useq[0], out["uhist"][k, t]), "planner %d step %d: u[0] differs" % (k, t)
                p.shift_and_update(out["xhist"][k, t + 1], useq, 1)
        assert np.isnan(out["xhist"][k, n + 1:]).all() and np.isnan(out["uhist"][k, n:]).all()
        assert not np.isnan(out["xhist"][k, :n + 1]).any()
        assert_same(snapshot(A[k]), snapshot(p), "planner %d" % k)
        assert np.array_equal(A[k].params["x0"], p.params["x0"]) and A[k].params["x0"].dtype == np.float64
    with _quiet():
        for k in range(K_EACH):
            ua, ub = A[k].solve(), B[k].solve()
            if status[k] == "left_map":
                assert ua is None and ub is None
            else:
                assert np.array_equal(ua, ub), "planner %d: the next solve differs" % k
                assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d after one more solve" % k)


def ulps(a, b):
    ia, ib = a.view(np.int64), b.view(np.int64)
    ia = np.where(ia < 0, np.int64(-2 ** 63) - ia, ia)
    ib = np.where(ib < 0, np.int64(-2 ** 63) - ib, ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize("mode", ["det", "spd"])
def test_plant_accuracy(eng, mode):
    """Every step of xhist recomputed in numpy from the device's xhist[t] and uhist[t]: the same traction cell, and
    states within 2 ulp (CUDA's double cos / sin are not correctly rounded)."""
    E = eng
    A, _, grids = twins(E, mode)
    with _quiet():
        out = E.MPPI_Batch(A).run_trials(grids, MAX_STEPS)
    differ, total, worst = 0, 0, 0
    for k, g in enumerate(grids):
        dt = float(A[k].params["dt"])
        for t in range(int(out["steps"][k])):
            x, u = out["xhist"][k, t], out["uhist"][k, t]
            want = plant_step(g, x, u, dt)
            got = out["xhist"][k, t + 1]
            u_ = ulps(want, got)
            worst = max(worst, int(u_.max()))
            differ += int((u_ > 0).any())
            total += 1
            assert (u_ <= 2).all(), "planner %d step %d: %s vs %s" % (k, t, got, want)
    print("%s: %d of %d plant steps differ from numpy in any bit (worst %d ulp)" % (mode, differ, total, worst))


@pytest.mark.parametrize("mode", ["det", "spd"])
def test_end_to_end_against_host_trial(eng, mode):
    """run_trials against a fully host-driven episode on twins: same status and step count, trajectories and the trial
    logs within 1e-9."""
    E = eng
    A, B, grids = twins(E, mode)
    with _quiet():
        out = E.MPPI_Batch(A).run_trials(grids, MAX_STEPS)
        host = [host_trial(p, g, MAX_STEPS) for p, g in zip(B, grids)]
    for k, (log, xh, uh, n, status) in enumerate(host):
        assert out["status"][k] == status and out["steps"][k] == n, "planner %d" % k
        assert np.allclose(out["xhist"][k], xh, rtol=0, atol=1e-9, equal_nan=True)
        assert np.array_equal(out["uhist"][k], uh, equal_nan=True)
        for key, v in log.items():
            w = out["logs"][k][key]
            if isinstance(v, bool):
                assert w == v
            else:
                assert (np.isnan(v) and np.isnan(w)) or abs(w - v) <= 1e-9 * max(1.0, abs(v)), (k, key, w, v)


def test_launch_accounting_and_batch_solve_unchanged(eng):
    """5 launches per issued step (num_opt = 1), nothing issued once every planner has stopped, and the batch solve's
    results and launch count are those of the same batch without trials."""
    E = eng
    A, B, grids = twins(E, "det")
    batch = E.MPPI_Batch(A)
    l0 = batch.launch_count()
    with _quiet():
        out = batch.run_trials(grids, MAX_STEPS)
    issued = batch.steps_issued
    assert batch.launch_count() - l0 == 5 * issued
    last = int(out["steps"].max())
    assert last <= issued <= min(MAX_STEPS, last + 4)       # the count of running planners is polled 4 steps behind
    # the batch solve after trials: the same launches and results as a fresh batch of twins in the same state
    with _quiet():
        ok = [k for k in range(K_EACH) if out["status"][k] != "left_map"]
        Ab = E.MPPI_Batch([A[k] for k in ok])
        for k, p in enumerate(B):
            n = int(out["steps"][k])
            for t in range(n):
                useq = p.solve()
                p.shift_and_update(out["xhist"][k, t + 1], useq, 1)
        Bb = E.MPPI_Batch([B[k] for k in ok])
        la, lb = Ab.launch_count(), Bb.launch_count()
        ua, ub = Ab.solve(), Bb.solve()
    assert np.array_equal(ua, ub)
    assert Ab.launch_count() - la == Bb.launch_count() - lb == 4


def test_refusals_name_the_planner(eng):
    E = eng
    A, _, grids = twins(E, "det")
    batch = E.MPPI_Batch(A)
    l0 = batch.launch_count()
    with pytest.raises(ValueError, match="4 traction grids for 5 planners"):
        batch.run_trials(grids[:4], 5)
    with pytest.raises(ValueError, match="max_steps 0 < 1"):
        batch.run_trials(grids, 0)
    A[2].params["num_opt"] = 0
    with pytest.raises(ValueError, match="planner 2 has num_opt 0"):
        batch.run_trials(grids, 5)
    A[2].params["num_opt"] = 1
    x0 = A[3].params["x0"].copy()
    A[3].params["x0"] = np.array([-50.0, 1.0, 0.0])
    with _quiet(), pytest.raises(ValueError, match="planner 3 cannot solve"):
        batch.run_trials(grids, 5)
    A[3].params["x0"] = x0
    # a pair that cannot join the one sampler launch: its two TDMs' streams diverged
    with _quiet():
        A[1].lin_tdm.sample_grids()
    with pytest.raises(E.B200MPPIError, match="planner 1: its TDM pair cannot join"):
        batch.run_trials(grids, 5)
    assert batch.launch_count() == l0
