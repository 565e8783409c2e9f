"""Closed-loop trials of stochastic (use_tdm) batches on the GPU (run with ``-m gpu``): run_stochastic_trials against
the same episodes driven from the host on identical twins -- replayed from the device's trajectory (controls, every
planner buffer, the reach box and the next solve bit for bit), the plant step recomputed in numpy, a fully host-driven
episode -- in every box mode and at the reference benchmark's shape; launch accounting; every refusal."""

import numpy as np
import pytest

from tests.test_gpu_stochastic_batch import _quiet, assert_same, planner_launches, snapshot, tdm_planner, tdm_scenario
from tests.test_gpu_trials import ulps
from tests.trial_loop import host_trial, plant_step

pytestmark = pytest.mark.gpu

MAX_STEPS = 20


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    assert E.device_count() >= 1, "GPU tests need a CUDA device"
    return E


def trial_setup(E, k, num_opt=1, **shape):
    """Planner k and its ground-truth grid.  k = 0, 1: goal within a step, and a nearby goal; k = 2: goal out of reach (runs to
    max_steps); k = 3: start near the map's corner (every box leaves the map: whole maps); k = 4: an int8 grid
    (TractionGrid's use_int8 stores 100 x traction) that throws the robot off the padded map."""
    sc = tdm_scenario(k, num_opt=num_opt, edge=(k == 3), **shape)
    p = sc["params"]
    n, res = shape.get("H", 64), shape.get("res", 0.2)
    x0 = np.asarray(p["x0"], dtype=np.float64)
    if k == 0:
        p["xgoal"] = x0[:2] + 0.3
    elif k == 1:
        p["xgoal"] = x0[:2] + np.array([0.9, -0.4])
    elif k == 2:
        p["xgoal"] = x0[:2] + 50.0
    elif k == 3:
        p["xgoal"] = x0[:2] + np.array([1.5, 1.0])
    elif k == 4:
        p["xgoal"] = x0[:2] + np.array([-1.5, 1.2])
    pl = tdm_planner(E, sc, k)
    rng = np.random.default_rng(300 + k)
    grid = E.TractionGrid(rng.uniform(0.2, 1.0, (n, n)), rng.uniform(0.2, 1.0, (n, n)), res=res, use_int8=(k == 4))
    return pl, grid


def twins(E, K=5, **kw):
    with _quiet():
        A = [trial_setup(E, k, **kw) for k in range(K)]
        B = [trial_setup(E, k, **kw) for k in range(K)]
    return [a[0] for a in A], [b[0] for b in B], [a[1] for a in A]


def replay(E, A, B, out, check_next=True):
    """The host loop fed with the device's trajectory, on the twins B: u[0] of every step, then every buffer of the
    planner (snapshot, sample_box and costs_nm included) and params['x0'], then one more solve on both."""
    for k, p in enumerate(B):
        n = int(out["steps"][k])
        one = E.MPPI_StochasticBatch([p])
        with _quiet():
            for t in range(n):
                useq = one.solve()[0]
                assert np.array_equal(useq[0], out["uhist"][k, t]), "planner %d step %d: u[0] differs" % (k, t)
                p.shift_and_update(out["xhist"][k, t + 1], useq, 1)
        assert np.isnan(out["xhist"][k, n + 1:]).all() and np.isnan(out["uhist"][k, n:]).all()
        assert_same(snapshot(A[k]), snapshot(p), "planner %d" % k)
        assert np.array_equal(A[k].params["x0"], p.params["x0"])
    if not check_next:
        return
    with _quiet():
        for k in range(len(A)):
            ua, ub = A[k].solve(), B[k].solve()
            if out["status"][k] == "left_map":
                assert ua is None and ub is None
            else:
                assert np.array_equal(ua, ub), "planner %d: the next solve differs" % k
                assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d after one more solve" % k)


def test_replay_equality(eng):
    E = eng
    A, B, grids = twins(E)
    batch = E.MPPI_StochasticBatch(A)
    with _quiet():
        out = batch.run_stochastic_trials(grids, MAX_STEPS)
    steps, status = out["steps"], out["status"]
    print("steps", steps.tolist(), "status", status, "boxes", [list(p.sample_box()) for p in A])
    assert status[0] == "goal" and steps[0] == 1
    assert status[2] == "max_steps" and steps[2] == MAX_STEPS
    assert status[4] == "left_map"
    assert A[2].sample_box()[0] == 2                           # the dynamic box, decided on the device
    assert batch.launch_count() == 7 * batch.steps_issued
    replay(E, A, B, out)


def test_host_driven_episode_and_plant(eng):
    """A fully host-driven episode on the twins: the same status, steps and logs; every plant step of the device within
    2 ulp of numpy's (CUDA's double cos / sin are not correctly rounded)."""
    E = eng
    A, B, grids = twins(E)
    with _quiet():
        out = E.MPPI_StochasticBatch(A).run_stochastic_trials(grids, MAX_STEPS)
    worst = 0
    for k, g in enumerate(grids):
        dt = float(A[k].params["dt"])
        for t in range(int(out["steps"][k])):
            worst = max(worst, int(ulps(plant_step(g, out["xhist"][k, t], out["uhist"][k, t], dt),
                                        out["xhist"][k, t + 1]).max()))
        with _quiet():
            log, xh, uh, n, st = host_trial(B[k], g, MAX_STEPS)
        assert (n, st) == (int(out["steps"][k]), out["status"][k]), "planner %d" % k
        for key, v in log.items():
            w = out["logs"][k][key]
            assert (np.isnan(v) and np.isnan(w)) if isinstance(v, float) and np.isnan(v) else np.isclose(v, w, rtol=1e-9), \
                "planner %d: log %s %r vs %r" % (k, key, w, v)
    assert worst <= 2, worst


@pytest.mark.parametrize("case", ["num_opt2", "box_off"])
def test_box_modes(eng, case, monkeypatch):
    """num_opt 2 (the static box: the reach of one iteration's controls does not bound the next) and
    B200MPPI_SAMPLE_BOX=off (whole maps every step), set before the planners are created."""
    E = eng
    if case == "box_off":
        monkeypatch.setenv("B200MPPI_SAMPLE_BOX", "off")
    A, B, grids = twins(E, num_opt=2 if case == "num_opt2" else 1)
    batch = E.MPPI_StochasticBatch(A)
    with _quiet():
        out = batch.run_stochastic_trials(grids, 6)
    want = (0, 1) if case == "num_opt2" else (0,)
    boxes = [list(p.sample_box()) for p in A]
    assert all(b[0] in want for b in boxes), boxes
    assert batch.launch_count() == (4 * (2 if case == "num_opt2" else 1) + 3) * batch.steps_issued
    replay(E, A, B, out)


def test_reference_shape_and_config3(eng):
    """The reference benchmark's shape (M 1024, T 100, a 9 x 9-cell map at 1 m: every box leaves it) with K = 4, and
    config 3's shape with K = 32, over a few steps."""
    E = eng
    A, B, grids = twins(E, K=4, N=256, M=1024, T=100, H=9, res=1.0)
    with _quiet():
        out = E.MPPI_StochasticBatch(A).run_stochastic_trials(grids, 3)
    assert all(p.sample_box()[0] == 0 for p in A)
    replay(E, A, B, out, check_next=False)
    with _quiet():
        A = [trial_setup(E, 2 if k % 2 else 1, N=1024, M=64, T=64, H=512, res=0.1)[0] for k in range(32)]
        B = [trial_setup(E, 2 if k % 2 else 1, N=1024, M=64, T=64, H=512, res=0.1)[0] for k in range(32)]
        grids = [E.TractionGrid(np.full((512, 512), 0.8), np.full((512, 512), 0.9), res=0.1) for _ in range(32)]
        out = E.MPPI_StochasticBatch(A).run_stochastic_trials(grids, 3)
    replay(E, A[:4] + A[-2:], B[:4] + B[-2:], dict(out, steps=np.concatenate([out["steps"][:4], out["steps"][-2:]]),
                                                   uhist=np.concatenate([out["uhist"][:4], out["uhist"][-2:]]),
                                                   xhist=np.concatenate([out["xhist"][:4], out["xhist"][-2:]]),
                                                   status=out["status"][:4] + out["status"][-2:]), check_next=False)


def test_refusals_issue_nothing(eng):
    E = eng
    A, _, grids = twins(E, K=3)
    batch = E.MPPI_StochasticBatch(A)
    before = [snapshot(p) for p in A]
    with pytest.raises(ValueError, match="trials run det-dynamics or speed-map"):
        batch.run_trials(grids, 5)
    with pytest.raises(ValueError, match="2 traction grids for 3 planners"):
        batch.run_stochastic_trials(grids[:2], 5)
    with pytest.raises(ValueError, match="max_steps 0 < 1"):
        batch.run_stochastic_trials(grids, 0)
    A[1].params["num_opt"] = 0
    with pytest.raises(ValueError, match="planner 1 has num_opt 0 < 1"):
        batch.run_stochastic_trials(grids, 5)
    A[1].params["num_opt"] = 1
    with _quiet():
        A[2].lin_tdm.sample_grids()                              # diverged lin / ang streams
    before[2] = snapshot(A[2])
    with pytest.raises(E.B200MPPIError, match="planner 2: its TDM pair cannot join"):
        batch.run_stochastic_trials(grids, 5)
    with _quiet():
        A[2].setup(A[2].params, A[2].lin_tdm, A[2].lin_tdm)      # lin == ang
    with pytest.raises(E.B200MPPIError, match="planner 2: its TDM pair cannot join"):
        batch.run_stochastic_trials(grids, 5)
    assert batch.launch_count() == 0
    for k, (p, b) in enumerate(zip(A[:2], before[:2])):
        assert_same(snapshot(p), b, "refused planner %d" % k)
    assert all(planner_launches(E, p) == 0 for p in A[:2])
    det = E.MPPI_Batch([trial_setup_det(E)])
    res = (E._lib.TrialResult * 1)()
    rc = E._lib.lib.b200mppi_batch_run_stochastic_trials(det._handle, (E._lib.TrialDesc * 1)(), 5, None, None, res, None)
    assert rc != 0 and "planner 0 is MODE_DET_DYN" in E._lib.lib.b200mppi_last_error().decode()
    assert det.launch_count() == 0


def trial_setup_det(E):
    from tests.scenarios import make_scenario
    det = make_scenario("det", N=200, M=1, T=20, H=64, W=64, res=0.2, B=5, seed=3)
    with _quiet():
        cfg = E.Config(**det["cfg"])
        lin, ang = E.TDM_Numba(cfg), E.TDM_Numba(cfg)
        lin.set_TDM_from_PMF_grid(det["pmf_lin"], det["tdm_dict"], det["obstacle"], det["unknown"])
        ang.set_TDM_from_PMF_grid(det["pmf_ang"], det["tdm_dict"], det["obstacle"], det["unknown"])
        dp = E.MPPI_Numba(cfg)
        dp.setup(det["params"], lin, ang)
    return dp
