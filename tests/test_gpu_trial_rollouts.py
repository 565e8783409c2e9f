"""Visualisation rollouts of batches and device trials on the GPU (run with ``-m gpu``): MPPI_Batch.get_state_rollout
against each twin's get_state_rollout() (every planner kind, a use_tdm batch right after solves whose boxes were
partial), and the records of run_trials / run_stochastic_trials / run_barebone_trials with record_every against the host
loop that calls get_state_rollout() after solve() and before shift_and_update -- bit for bit, NaN after each planner's
last step -- while everything else equals the same call without recording; launch accounting; the C refusals."""
import ctypes as C
import functools

import numpy as np
import pytest

from tests.gpu_harness import (assert_same, eng, quiet, snapshot, solve_in_batch_of_one, tdm_planner,  # noqa: F401
                               tdm_trial_setup, vary)
from tests.scenarios import make_scenario

pytestmark = pytest.mark.gpu

MAX_STEPS = 10


def map_setup(E, mode, k):
    """det / spd planner k (own map, seed, warm start) and its ground-truth grid: k = 0 reaches its goal in one step,
    k = 1 in a few, k = 2 runs to max_steps, k = 3 is thrown off the padded map by an int8 (100 x) grid."""
    sc = make_scenario(mode, N=256, M=1, T=16, H=40, W=40, res=0.2, B=6, seed=11 + 7 * k, warm_start=(k % 2 == 1))
    p = sc["params"]
    p["xgoal"] = p["x0"][:2] + [np.array([0.3, 0.3]), np.array([0.9, -0.4]), np.array([50.0, 50.0]),
                                np.array([-1.5, 1.2])][k]
    pl = tdm_planner(E, vary(sc, k))
    rng = np.random.default_rng(100 + k + (0 if mode == "det" else 50))
    grid = E.TractionGrid(rng.uniform(0.2, 1.0, (40, 40)), rng.uniform(0.2, 1.0, (40, 40)), res=0.2,
                          use_int8=(k == 3))
    return pl, grid


def bb_setup(E, k, V=20):
    """Barebone planner k and no grid: k = 0 reaches its goal in one step, k = 1 in a few, k = 2 runs to max_steps."""
    from mppi_numba_b200 import barebone as BB
    pl = BB.MPPI_Numba(BB.Config(T=2.0, dt=0.1, num_control_rollouts=512, num_vis_state_rollouts=V, seed=3 + k))
    pl.setup(dict(dt=[0.1, 0.1, 0.08][k], x0=np.array([0.0, 0.0, 0.1 * k]),
                  xgoal=[np.array([0.3, 0.0]), np.array([1.5, 0.8]), np.array([40.0, 40.0])][k], goal_tolerance=0.5,
                  dist_weight=10, lambda_weight=[1.0, 0.5, 2.0][k], num_opt=1, u_std=np.array([1.0, 1.0]) * (1 + 0.1 * k),
                  vrange=np.array([0.0, 2.0]), wrange=np.array([-np.pi, np.pi]), obs_penalty=1e6,
                  obstacle_positions=np.array([[5.0, 4.5], [2.0, 1.0]]), obstacle_radius=np.array([1.5, 1.0])))
    return pl, None


# kind -> (setup(E, k), K, batch class name, trial method, traction grids taken, host solve, launches per step)
KINDS = {
    "det": (functools.partial(map_setup, mode="det"), 4, "MPPI_Batch", "run_trials", True, None, 5),
    "spd": (functools.partial(map_setup, mode="spd"), 4, "MPPI_Batch", "run_trials", True, None, 5),
    "barebone": (bb_setup, 3, "MPPI_Batch", "run_barebone_trials", False, None, 4),
    "tdm": (tdm_trial_setup, 5, "MPPI_StochasticBatch", "run_stochastic_trials", True, solve_in_batch_of_one, 7),
    "tdm_whole": (functools.partial(tdm_trial_setup, N=256, M=64, T=20, H=9, res=1.0), 4, "MPPI_StochasticBatch",
                  "run_stochastic_trials", True, solve_in_batch_of_one, 7),
}


def sets(E, kind, n):
    """n identical sets of the kind's planners (and one list of grids)."""
    setup, K = KINDS[kind][0], KINDS[kind][1]
    with quiet():
        made = [[setup(E, k=k) for k in range(K)] for _ in range(n)]
    return [[m[0] for m in s] for s in made], [m[1] for m in made[0]]


def with_vis(p):
    d = snapshot(p)
    d["state_rollout"] = p.state_rollout_batch_d.copy_to_host()
    return d


def run(E, kind, planners, grids, steps, **kw):
    cls, method, takes_grids = getattr(E, KINDS[kind][2]), KINDS[kind][3], KINDS[kind][4]
    batch = cls(planners)
    with quiet():
        out = getattr(batch, method)(*((grids,) if takes_grids else ()), steps, **kw)
    return batch, out


@pytest.mark.parametrize("kind", ["det", "spd", "barebone", "tdm"])
def test_batch_get_state_rollout(eng, kind):
    """batch.get_state_rollout() == each twin's get_state_rollout() after equal solves, bit for bit, and the planners
    (snapshots and state_rollout_batch_d) equal afterwards.  For use_tdm the solves' boxes are partial."""
    E = eng
    (A, B), _ = sets(E, kind, 2)
    batch = getattr(E, KINDS[kind][2])(A)
    with quiet():
        for r in range(2):
            ua = batch.solve()
            ub = np.stack([p.solve() for p in B])
            assert_same(dict(u=ua), dict(u=ub), "round %d" % r)
    if kind == "tdm":
        assert sum(p.sample_box()[0] != 0 for p in A) >= 2, [list(p.sample_box()) for p in A]
    before = batch.launch_count()
    got = batch.get_state_rollout()
    assert batch.launch_count() == before + 1
    with quiet():
        want = np.stack([p.get_state_rollout() for p in B])
    assert got.dtype == np.float32 and got.shape == (len(A), A[0].num_vis_state_rollouts, A[0].num_steps + 1, 3)
    assert not np.isnan(got).any()
    assert_same(dict(r=got), dict(r=want), kind)
    for k in range(len(A)):
        assert_same(with_vis(A[k]), with_vis(B[k]), "planner %d" % k)


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("kind", ["det", "spd", "barebone", "tdm", "tdm_whole"])
def test_trial_records(eng, kind, every):
    """The records == get_state_rollout() of the host loop replayed on twins with the device trajectory, at the same
    steps (after solve(), before shift_and_update), bit for bit and NaN after each planner's last step; xhist, uhist,
    logs, steps, status and every planner's final state == the same call without recording; launch accounting."""
    E = eng
    (A, B, Cw), grids = sets(E, kind, 3)
    batch, out = run(E, kind, A, grids, MAX_STEPS, record_every=every)
    plain_batch, plain = run(E, kind, Cw, grids, MAX_STEPS)
    K, R = len(A), -(-MAX_STEPS // every)
    V, T = A[0].num_vis_state_rollouts, A[0].num_steps
    print(kind, every, "steps", out["steps"].tolist(), "status", out["status"])
    if kind == "tdm":
        assert any(p.sample_box()[0] != 0 for p in A)
    if kind == "tdm_whole":
        assert all(p.sample_box()[0] == 0 for p in A)
    else:                                              # records after a planner's last step exist, and are NaN
        assert out["steps"][0] == 1 and out["steps"].max() == MAX_STEPS
    assert out["steps"].max() > every
    # without recording: everything else identical
    assert set(out) == set(plain) | {"state_rollouts", "rollout_steps"}
    for key in ("xhist", "uhist", "steps") + (("contact_steps",) if kind == "barebone" else ()):
        assert_same({key: out[key]}, {key: plain[key]}, "%s vs plain" % key)
    assert out["status"] == plain["status"] and batch.steps_issued == plain_batch.steps_issued
    for k in range(K):
        assert out["logs"][k].keys() == plain["logs"][k].keys()
        assert_same({x: np.float64(v) for x, v in out["logs"][k].items()},
                    {x: np.float64(v) for x, v in plain["logs"][k].items()}, "planner %d: log" % k)
        assert_same(snapshot(A[k]), snapshot(Cw[k]), "planner %d vs plain" % k)
    # launches: the plain call's, plus 1 per recorded step (2 for a stochastic batch)
    recorded = -(-batch.steps_issued // every)
    assert batch.launch_count() == plain_batch.launch_count() + recorded * (2 if kind.startswith("tdm") else 1)
    assert plain_batch.launch_count() == KINDS[kind][6] * plain_batch.steps_issued
    # the records against the host loop
    rec = out["state_rollouts"]
    assert rec.dtype == np.float32 and rec.shape == (K, R, V, T + 1, 3)
    assert out["rollout_steps"].tolist() == [r * every for r in range(R)]
    solve_one = KINDS[kind][5] or (lambda p: p.solve())
    for k, p in enumerate(B):
        n = int(out["steps"][k])
        with quiet():
            for t in range(n):
                u = solve_one(p)
                assert_same({"u[0]": u[0]}, {"u[0]": out["uhist"][k, t]}, "planner %d step %d" % (k, t))
                if t % every == 0:
                    want = p.get_state_rollout()
                    assert not np.isnan(want).any()
                    assert_same(dict(r=rec[k, t // every]), dict(r=want), "planner %d step %d: record" % (k, t))
                p.shift_and_update(out["xhist"][k, t + 1], u, 1)
        done = -(-n // every)
        assert np.isnan(rec[k, done:]).all(), "planner %d: records after step %d" % (k, n)
        assert_same(with_vis(A[k]), with_vis(p), "planner %d after the host loop" % k)


def test_refusals_issue_nothing(eng):
    """Refused before any work: record_every < 1 (Python and C), a wrong byte count, an unknown kind, unequal V."""
    E = eng
    from mppi_numba_b200 import _lib as L
    (A,), _ = sets(E, "barebone", 1)
    batch = E.MPPI_Batch(A)
    before = [with_vis(p) for p in A]
    with pytest.raises(ValueError, match="record_every 0 < 1"):
        batch.run_barebone_trials(5, record_every=0)
    K, V, T = len(A), A[0].num_vis_state_rollouts, A[0].num_steps
    descs = (L.TrialDesc * K)()
    for i, p in enumerate(A):
        p.move_mppi_task_vars_to_device()              # what the Python calls do before the C call
        descs[i].x0[:] = [float(v) for v in p.params["x0"]]
        descs[i].xgoal[:] = [float(v) for v in p.params["xgoal"]]
        descs[i].goal_tolerance, descs[i].dt = float(p.params["goal_tolerance"]), float(p.params["dt"])
    xh, uh = np.empty((K, 6, 3)), np.empty((K, 5, 2), np.float32)
    res, con, issued = (L.TrialResult * K)(), np.empty(K, np.int32), C.c_int32(-1)
    good = np.empty((K, 2, V, T + 1, 3), np.float32)
    for kind, every, nbytes, msg in ((L.TRIALS_BAREBONE, 0, good.nbytes, "record_every 0 < 1"),
                                     (L.TRIALS_BAREBONE, 3, good.nbytes - 4, "rollouts buffer of"),
                                     (7, 3, good.nbytes, "unknown trial kind 7"),
                                     (L.TRIALS_MAP, 3, good.nbytes, "MODE_BAREBONE")):
        rc = L.lib.b200mppi_batch_run_trials_recorded(batch._handle, kind, descs, 5, L.ptr(xh), L.ptr(uh), res,
                                                      L.ptr(con), every, L.ptr(good), nbytes, C.byref(issued))
        assert rc != 0 and msg in L.lib.b200mppi_last_error().decode(), (msg, L.lib.b200mppi_last_error())
    assert issued.value == -1 and batch.launch_count() == 0
    with quiet():
        odd = bb_setup(E, 2, V=7)[0]
    mixed = E.MPPI_Batch(A[:2] + [odd])
    with pytest.raises(ValueError, match="planner 2 has num_vis_state_rollouts 7, planner 0 20"):
        mixed.get_state_rollout()
    with pytest.raises(ValueError, match="planner 2 has num_vis_state_rollouts 7"):
        mixed.run_barebone_trials(5, record_every=2)
    out = np.empty((3, V, T + 1, 3), np.float32)
    odd.move_mppi_task_vars_to_device()
    assert L.lib.b200mppi_batch_get_state_rollout(mixed._handle, L.ptr(out), out.nbytes) != 0
    assert "planner 2 has num_vis_state_rollouts 7, planner 0 20" in L.lib.b200mppi_last_error().decode()
    assert L.lib.b200mppi_batch_get_state_rollout(batch._handle, L.ptr(out), out.nbytes - 4) != 0
    assert "size mismatch" in L.lib.b200mppi_last_error().decode()
    assert mixed.launch_count() == 0 and batch.launch_count() == 0
    for p, b in zip(A, before):
        assert_same(with_vis(p), b, "untouched")
