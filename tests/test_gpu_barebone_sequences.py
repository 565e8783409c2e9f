"""Barebone trial sequences on the GPU (run with ``-m gpu``): MPPI_Batch.run_barebone_trial_sequences against the
barebone notebook's loop per episode replayed on identical twins with the device trajectory -- u[0] of every solve,
contact counts per episode (tests/barebone_trial_loop.py's rule), records at each episode's steps t % n == 0, and every
planner's snapshot and state_rollout_batch_d bit for bit -- with and without reset_x0; one-episode sequences against
run_barebone_trials; launches; refusals."""
import numpy as np
import pytest

from tests.barebone_trial_loop import in_contact, obstacles
from tests.gpu_harness import assert_same, eng, quiet, snapshot  # noqa: F401
from tests.test_gpu_trial_rollouts import bb_setup

pytestmark = pytest.mark.gpu

S = 12


def with_vis(p):
    d = snapshot(p)
    d["state_rollout"] = p.state_rollout_batch_d.copy_to_host()
    return d


def through_obstacle(E):
    """A planner whose start lies inside an obstacle it is barely penalised for: its first steps touch it."""
    from mppi_numba_b200 import barebone as BB
    pl = BB.MPPI_Numba(BB.Config(T=2.0, dt=0.1, num_control_rollouts=512, num_vis_state_rollouts=20, seed=9))
    pl.setup(dict(dt=0.1, x0=np.array([0.0, 0.0, 0.0]), xgoal=np.array([3.0, 0.0]), goal_tolerance=0.3,
                  dist_weight=10, lambda_weight=1.0, num_opt=1, u_std=np.array([1.0, 1.0]), vrange=np.array([0.0, 2.0]),
                  wrange=np.array([-np.pi, np.pi]), obs_penalty=1.0, obstacle_positions=np.array([[0.2, 0.0]]),
                  obstacle_radius=np.array([0.5])))
    return pl


def planners(E, n=3):
    """n identical sets: bb_setup's three planners (goal in one step, in a few, out of reach) and through_obstacle."""
    with quiet():
        return [[bb_setup(E, k)[0] for k in range(3)] + [through_obstacle(E)] for _ in range(n)]


@pytest.mark.parametrize("every", [None, 1, 5])
@pytest.mark.parametrize("reset_x0", [False, True])
def test_against_host_loop(eng, reset_x0, every):
    E = eng
    A, B, Cw = planners(E)
    episodes = [3, 2, 4, 2]
    ba = E.MPPI_Batch(A)
    with quiet():
        out = ba.run_barebone_trial_sequences(episodes, S, reset_x0=reset_x0, record_every=every)
        plain = E.MPPI_Batch(Cw).run_barebone_trial_sequences(episodes, S, reset_x0=reset_x0)
    print(reset_x0, every, "steps", out["steps"].tolist(), "contacts", out["contact_steps"].tolist())
    assert out["episodes_run"].tolist() == episodes
    assert all(set(s) <= {"goal", "max_steps"} for s in out["status"])
    assert out["contact_steps"].shape == (4, 4) and (out["contact_steps"][3, :2] > 0).all()
    assert (out["steps"] == 1).any() and (out["steps"] == S).any()
    for key in ("xhist", "uhist", "steps", "contact_steps"):
        assert_same({key: out[key]}, {key: plain[key]}, "%s vs plain" % key)
    per_step = 4 + (1 if every else 0)                 # noise, rollout, update, plant step (+ the gated record)
    assert ba.launch_count() == per_step * ba.steps_issued
    rec = out.get("state_rollouts")
    for k, p in enumerate(B):
        x_start = np.array(p.params["x0"], dtype=np.float64)
        obs = obstacles(p)
        with quiet():
            for e in range(episodes[k]):
                n = int(out["steps"][k, e])
                assert np.array_equal(out["xhist"][k, e, 0], x_start)
                if reset_x0:
                    p.params["x0"] = x_start.copy()
                for t in range(n):
                    u = p.solve()
                    assert_same({"u[0]": u[0]}, {"u[0]": out["uhist"][k, e, t]}, "planner %d ep %d step %d" % (k, e, t))
                    if every and t % every == 0:
                        assert_same(dict(r=rec[k, e, t // every]), dict(r=p.get_state_rollout()),
                                    "planner %d episode %d step %d: record" % (k, e, t))
                    p.shift_and_update(out["xhist"][k, e, t + 1], u, 1)
                want = sum(in_contact(out["xhist"][k, e, t + 1], obs) for t in range(n))
                assert out["contact_steps"][k, e] == want == out["logs"][k][e]["contact_steps"], (k, e)
                if every:
                    assert np.isnan(rec[k, e, -(-n // every):]).all()
        assert out["contact_steps"][k, episodes[k]:].tolist() == [0] * (4 - episodes[k])
        if every:
            assert np.isnan(rec[k, episodes[k]:]).all()
            assert_same(with_vis(A[k]), with_vis(p), "planner %d" % k)
        else:
            assert_same(snapshot(A[k]), snapshot(p), "planner %d" % k)
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=p.params["x0"]), "planner %d: x0" % k)


def test_one_episode_equals_run_barebone_trials(eng):
    E = eng
    A, B, _ = planners(E)
    with quiet():
        out = E.MPPI_Batch(A).run_barebone_trial_sequences(1, S, record_every=2)
        want = E.MPPI_Batch(B).run_barebone_trials(S, record_every=2)
    assert_same(dict(r=out["state_rollouts"][:, 0], x=out["xhist"][:, 0], c=out["contact_steps"][:, 0]),
                dict(r=want["state_rollouts"], x=want["xhist"], c=want["contact_steps"]), "outputs")
    for k in range(4):
        assert_same(with_vis(A[k]), with_vis(B[k]), "planner %d" % k)


def test_refusals_issue_nothing(eng):
    E = eng
    from tests.test_gpu_trials import trial_setup
    A, _, _ = planners(E)
    batch = E.MPPI_Batch(A)
    before = [with_vis(p) for p in A]
    with pytest.raises(ValueError, match="planner 1: episode count 0 < 1"):
        batch.run_barebone_trial_sequences([1, 0, 2, 1], S)
    with pytest.raises(ValueError, match="record_every 0 < 1"):
        batch.run_barebone_trial_sequences(2, S, record_every=0)
    with pytest.raises(ValueError, match="planner 0 is a barebone planner"):
        batch.run_trial_sequences([[None]] * 4, S)
    with quiet():
        det = E.MPPI_Batch([trial_setup(E, "det", k)[0] for k in range(2)])
    with pytest.raises(ValueError, match="run_barebone_trial_sequences: planner 0 is a det planner"):
        det.run_barebone_trial_sequences(2, S)
    assert batch.launch_count() == 0 and det.launch_count() == 0
    for p, b in zip(A, before):
        assert_same(with_vis(p), b, "untouched")
