"""Closed-loop trials of barebone planners on the GPU (run with ``-m gpu``): MPPI_Batch.run_barebone_trials against the
notebook's loop driven from the host on identical twins -- replayed from the device's trajectory (controls and every
planner buffer bit for bit), the plant step and the obstacle contacts recomputed in numpy, and a fully host-driven
episode -- plus launch accounting, the batch solve left as it was, and the C entry point's refusals."""
import ctypes as C
import functools

import numpy as np
import pytest

from tests.barebone_trial_loop import host_trial, in_contact, obstacles, plant_step
from tests.gpu_harness import assert_same, eng, quiet, replay, snapshot, twins, ulps  # noqa: F401

pytestmark = pytest.mark.gpu

K_EACH = 6
MAX_STEPS = 40


def bb_setup(E, k, num_opt=1):
    """Barebone planner k (its own seed, lambda and noise) and no ground-truth grid.  k = 0: goal within one step;
    k = 1: goal a few steps away; k = 2: goal out of reach (runs to MAX_STEPS); k = 3: an obstacle on the straight
    path with obs_penalty 0, so the planner drives through it; k = 4: a start inside an obstacle; k = 5: no obstacles."""
    from mppi_numba_b200 import barebone as BB
    pl = BB.MPPI_Numba(BB.Config(T=2.0, dt=0.1, num_control_rollouts=512, seed=3 + k))
    x0 = [np.array([0.0, 0.0, 0.0]), np.array([0.0, 0.0, np.pi / 4]), np.array([0.5, -0.5, 0.3]),
          np.array([0.0, 0.0, 0.0]), np.array([0.0, 0.0, 0.2]), np.array([1.0, 1.0, -0.5])][k]
    xgoal = [np.array([0.3, 0.0]), np.array([1.5, 0.8]), np.array([40.0, 40.0]), np.array([3.0, 0.0]),
             np.array([2.5, 1.0]), np.array([3.0, -0.5])][k]
    params = dict(dt=[0.1, 0.1, 0.08, 0.1, 0.12, 0.1][k], x0=x0, xgoal=xgoal, goal_tolerance=0.5, dist_weight=10,
                  lambda_weight=[1.0, 0.5, 2.0, 1.0, 0.8, 1.3][k], num_opt=num_opt,
                  u_std=np.array([1.0, 1.0]) * (1.0 + 0.1 * k), vrange=np.array([0.0, 2.0]),
                  wrange=np.array([-np.pi, np.pi]), obs_penalty=1e6)
    if k == 3:
        params.update(obstacle_positions=np.array([[1.5, 0.0]]), obstacle_radius=np.array([0.4]), obs_penalty=0.0)
    elif k == 4:
        params.update(obstacle_positions=np.array([[0.1, 0.0], [4.0, 4.0]]), obstacle_radius=np.array([0.5, 1.0]))
    elif k != 5:
        params.update(obstacle_positions=np.array([[5.0, 4.5], [2.0, 1.0]]), obstacle_radius=np.array([1.5, 1.0]))
    pl.setup(params)
    return pl, None


def bb_twins(E, num_opt=1):
    A, B, _ = twins(functools.partial(bb_setup, E, num_opt=num_opt), K_EACH)
    return A, B


@pytest.mark.parametrize("num_opt", [1, 2])
def test_replay_equality(eng, num_opt):
    """run_barebone_trials == the host loop replayed with the device's trajectory: u[0] of every solve bit for bit,
    then every planner buffer and params['x0'] -- and one more solve() on both sets is identical."""
    E = eng
    A, B = bb_twins(E, num_opt)
    with quiet():
        out = E.MPPI_Batch(A).run_barebone_trials(MAX_STEPS)
    steps, status, contacts = out["steps"], out["status"], out["contact_steps"]
    print("num_opt", num_opt, "steps", steps.tolist(), "status", status, "contacts", contacts.tolist())
    assert status[0] == "goal" and steps[0] == 1
    assert status[1] == "goal" and 1 < steps[1] < MAX_STEPS
    assert status[2] == "max_steps" and steps[2] == MAX_STEPS
    assert status[3] == "goal" and contacts[3] > 0
    assert contacts[4] > 0 and contacts[5] == 0
    assert set(status) <= {"goal", "max_steps"}
    replay(A, B, out, lambda p: p.solve())


def test_plant_accuracy_and_contacts(eng):
    """Every step of xhist recomputed in numpy from the device's xhist[t] and uhist[t] within 2 ulp (CUDA's double
    cos / sin are not correctly rounded), and the contact counts exactly those of numpy's rule on the device's
    xhist."""
    E = eng
    A, _ = bb_twins(E)
    with quiet():
        out = E.MPPI_Batch(A).run_barebone_trials(MAX_STEPS)
    differ, total, worst = 0, 0, 0
    for k, p in enumerate(A):
        dt, obs, n = float(p.params["dt"]), obstacles(p), int(out["steps"][k])
        for t in range(n):
            want = plant_step(out["xhist"][k, t], out["uhist"][k, t], dt)
            u_ = ulps(want, out["xhist"][k, t + 1])
            worst = max(worst, int(u_.max()))
            differ += int((u_ > 0).any())
            total += 1
            assert (u_ <= 2).all(), "planner %d step %d: %s vs %s" % (k, t, out["xhist"][k, t + 1], want)
        touched = sum(in_contact(out["xhist"][k, t], obs) for t in range(1, n + 1))
        assert out["contact_steps"][k] == touched == out["logs"][k]["contact_steps"], k
    print("%d of %d plant steps differ from numpy in any bit (worst %d ulp)" % (differ, total, worst))


def test_end_to_end_against_the_notebook_loop(eng):
    """run_barebone_trials against the notebook's loop driven from the host on twins: same status, steps and contacts,
    trajectories and the trial logs within 1e-9."""
    E = eng
    A, B = bb_twins(E)
    with quiet():
        out = E.MPPI_Batch(A).run_barebone_trials(MAX_STEPS)
        host = [host_trial(p, MAX_STEPS) for p in B]
    for k, (log, xh, uh, n, status, contacts) in enumerate(host):
        assert out["status"][k] == status and out["steps"][k] == n, "planner %d" % k
        assert out["contact_steps"][k] == contacts, "planner %d" % k
        assert np.allclose(out["xhist"][k], xh, rtol=0, atol=1e-9, equal_nan=True)
        assert_same(dict(uhist=out["uhist"][k]), dict(uhist=uh), "planner %d" % k)
        assert out["logs"][k].keys() == log.keys()
        for key, v in log.items():
            w = out["logs"][k][key]
            if isinstance(v, (bool, int)):
                assert w == v, (k, key, w, v)
            else:
                assert (np.isnan(v) and np.isnan(w)) or abs(w - v) <= 1e-9 * max(1.0, abs(v)), (k, key, w, v)


@pytest.mark.parametrize("num_opt", [1, 2])
def test_launch_accounting_and_batch_solve_unchanged(eng, num_opt):
    """3 num_opt + 1 launches per issued step, nothing issued once every planner has stopped, and the batch solve's
    results, planner state and launch count after trials are those of a batch of twins in the same state."""
    E = eng
    A, B = bb_twins(E, num_opt)
    batch = E.MPPI_Batch(A)
    l0 = batch.launch_count()
    with quiet():
        out = batch.run_barebone_trials(MAX_STEPS)
    issued = batch.steps_issued
    assert batch.launch_count() - l0 == (3 * num_opt + 1) * issued
    last = int(out["steps"].max())
    assert last <= issued <= min(MAX_STEPS, last + 4)       # the count of running planners is polled 4 steps behind
    with quiet():
        for k, p in enumerate(B):
            for t in range(int(out["steps"][k])):
                useq = p.solve()
                p.shift_and_update(out["xhist"][k, t + 1], useq, 1)
        Bb = E.MPPI_Batch(B)
        la, lb = batch.launch_count(), Bb.launch_count()
        ua, ub = batch.solve(), Bb.solve()
    assert_same(dict(u=ua), dict(u=ub), "batch solve after trials")
    for k in range(K_EACH):
        assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d after the batch solve" % k)
    assert batch.launch_count() - la == Bb.launch_count() - lb == 3 * num_opt


def test_c_refusals_name_the_planner_and_issue_nothing(eng):
    """b200mppi_batch_run_barebone_trials refuses before issuing anything: a non-barebone batch, max_steps < 1,
    num_opt < 1, grids, a non-finite x0, xgoal or goal_tolerance, a dt that is not finite and positive; and the
    one-map and stochastic trial calls still refuse a barebone batch."""
    E = eng
    L = E._lib
    A, _ = bb_twins(E)
    batch = E.MPPI_Batch(A)
    with quiet():
        for p in A:
            p.move_mppi_task_vars_to_device()
    K, S = len(A), 5
    xh, uh = np.empty((K, S + 1, 3)), np.empty((K, S, 2), np.float32)
    con = np.zeros(K, np.int32)
    grid = np.ones((2, 2))

    def descs(**bad):
        d = (L.TrialDesc * K)()
        for i, p in enumerate(A):
            d[i].x0[:] = [float(v) for v in p.params["x0"]]
            d[i].xgoal[:] = [float(v) for v in p.params["xgoal"]]
            d[i].goal_tolerance, d[i].dt = float(p.params["goal_tolerance"]), float(p.params["dt"])
        for key, (i, v) in bad.items():
            if key == "lin":
                d[i].lin = grid.ctypes.data
            elif key in ("x0", "xgoal"):
                getattr(d[i], key)[0] = v
            else:
                setattr(d[i], key, v)
        return d

    def refused(b, d, steps, match, entry=L.lib.b200mppi_batch_run_barebone_trials):
        res = (L.TrialResult * K)()
        extra = (L.ptr(con),) if entry is L.lib.b200mppi_batch_run_barebone_trials else ()
        rc = entry(b._handle, d, steps, L.ptr(xh), L.ptr(uh), res, *extra, None)
        msg = L.lib.b200mppi_last_error().decode()
        assert rc != 0 and match in msg, (rc, msg)

    l0 = batch.launch_count()
    refused(batch, descs(), 0, "run_barebone_trials: max_steps < 1")
    refused(batch, descs(lin=(1, None)), S, "run_barebone_trials: planner 1: traction grids given")
    refused(batch, descs(x0=(2, np.nan)), S, "run_barebone_trials: planner 2: start pose, goal or goal_tolerance")
    refused(batch, descs(xgoal=(3, np.inf)), S, "run_barebone_trials: planner 3: start pose, goal or goal_tolerance")
    refused(batch, descs(goal_tolerance=(4, np.nan)), S, "planner 4: start pose, goal or goal_tolerance not finite")
    refused(batch, descs(dt=(5, 0.0)), S, "run_barebone_trials: planner 5: dt not finite and positive")
    refused(batch, descs(dt=(0, np.inf)), S, "run_barebone_trials: planner 0: dt not finite and positive")
    refused(batch, descs(), S, "run_trials: planner 0 is MODE_BAREBONE", L.lib.b200mppi_batch_run_trials)
    refused(batch, descs(), S, "run_stochastic_trials: planner 0 is MODE_BAREBONE",
            L.lib.b200mppi_batch_run_stochastic_trials)
    A[1].params["num_opt"] = 0
    with quiet():
        A[1].move_mppi_task_vars_to_device()
    refused(batch, descs(), S, "planner 1 has num_opt 0")
    assert batch.launch_count() == l0
    from tests.gpu_harness import tdm_planner
    from tests.scenarios import make_scenario
    with quiet():
        det = E.MPPI_Batch([tdm_planner(E, make_scenario("det", N=256, M=1, T=16, H=40, W=40, res=0.2, B=6, seed=4))])
    res = (L.TrialResult * 1)()
    d1 = descs()
    rc = L.lib.b200mppi_batch_run_barebone_trials(det._handle, d1, S, L.ptr(xh), L.ptr(uh), res, L.ptr(con), None)
    assert rc != 0 and "run_barebone_trials: planner 0 is MODE_DET_DYN" in L.lib.b200mppi_last_error().decode()
    assert det.launch_count() == 0
