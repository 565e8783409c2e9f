"""The map-free ("barebone") planner on the GPU against the exact oracle with the device provider (oracle/arith.py:
this GPU's approximate operations and .ftz flushes), every element equal: raw C-ABI planners over the edge-case table
of tests/barebone_edge_cases.py (costs, visualisation states, and the cost rollout's own states where a visualisation
row retraces it), the obstacle and goal boundaries built with this GPU's cos / sin, get_state_rollout of one planner
and of a batch, one MPPI_Batch solve with the update checked by tests/reduce_bounds.py, a device trial whose plant poses
land exactly on an obstacle's circle, and a solve whose every cost is +inf."""
import ctypes as C

import numpy as np
import pytest

from tests import barebone_edge_cases as BE
from tests import reduce_bounds as RB
from tests.barebone_trial_loop import in_contact, obstacles
from tests.gpu_harness import assert_all_equal, dev, eng, quiet   # noqa: F401

pytestmark = pytest.mark.gpu

F32 = np.float32
OBSTACLE_KINDS = ["up", "up_ahead", "down", "on_circle"]
GOAL_KINDS = ["on_tol", "split"]


class RawBarebone:
    """A MODE_BAREBONE planner driven through the C entry points: N below the Python Config's clamp, any V <= N."""

    def __init__(self, E, c, V):
        L = self.L = E._lib
        pod = L.ConfigPOD(num_steps=c["T"], num_control_rollouts=c["N"], num_grid_samples=1, max_map_rows=1,
                          max_map_cols=1, tdm_thread_x=1, tdm_thread_y=1, num_vis_state_rollouts=V, mode=L.MODE_BAREBONE,
                          device=0, rank=0, world_size=1, seed=1)
        self.h = C.c_void_p()
        L.check(L.lib.b200mppi_planner_create(C.byref(pod), C.byref(self.h)))
        self.c, self.V = c, V
        p = L.ParamsPOD()
        p.dt = c["dt"]
        p.x0 = L.c_floats(np.asarray(c["x0"], F32), 3)
        p.xgoal = L.c_floats(np.asarray(c["goal"], F32), 2)
        p.goal_tolerance, p.lambda_weight, p.cvar_alpha, p.num_opt, p.alpha_dyn = c["tol"], c["lam"], 1.0, 1, 1.0
        p.u_std = L.c_floats(np.asarray(c["u_std"], F32), 2)
        p.vrange = L.c_floats(np.asarray(c["vrange"], F32), 2)
        p.wrange = L.c_floats(np.asarray(c["wrange"], F32), 2)
        p.obs_penalty, p.dist_weight, p.v_post_rollout, p.unknown_penalty = c["obs_cost"], c["dist_weight"], 0.0, 0.0
        L.check(L.lib.b200mppi_planner_set_params(self.h, C.byref(p)))
        ob = c["obstacles"]
        pos, rad = np.ascontiguousarray(ob[:, :2]), np.ascontiguousarray(ob[:, 2])
        L.check(L.lib.b200mppi_planner_set_obstacles(self.h, L.ptr(pos) if len(ob) else None,
                                                     L.ptr(rad) if len(ob) else None, len(ob)))

    def copy_in(self, buf, a):
        a = np.ascontiguousarray(a, F32)
        self.L.check(self.L.lib.b200mppi_planner_copy_in(self.h, buf, self.L.ptr(a), a.nbytes))

    def rollout(self, noise, u_cur):
        self.copy_in(self.L.BUF_NOISE, noise)
        self.copy_in(self.L.BUF_U_CUR, u_cur)
        self.L.check(self.L.lib.b200mppi_planner_rollout(self.h))
        out = np.empty(self.c["N"], F32)
        self.L.check(self.L.lib.b200mppi_planner_copy_out(self.h, self.L.BUF_COSTS, self.L.ptr(out), out.nbytes))
        return out

    def states(self, u_prev):
        self.copy_in(self.L.BUF_U_PREV, u_prev)
        out = np.empty((self.V, self.c["T"] + 1, 3), F32)
        self.L.check(self.L.lib.b200mppi_planner_get_state_rollout(self.h, self.L.ptr(out), out.nbytes))
        return out

    def close(self):
        self.L.lib.b200mppi_planner_destroy(self.h)


def _run_case(E, dev, c, noise, u_cur, u_prev):
    """Costs, visualisation states (u_prev as given, then u_prev = u_cur) against the oracle; returns the costs."""
    V = BE.vis_count(c)
    rp = RawBarebone(E, c, V)
    try:
        costs = rp.rollout(noise, u_cur)
        vis = rp.states(u_prev)
        vis_alias = rp.states(u_cur)
    finally:
        rp.close()
    want, st = BE.oracle_costs(c, noise, u_cur, dev, return_states=True)
    assert_all_equal(costs, want, c["name"] + " costs")
    assert_all_equal(vis, BE.oracle_states(c, V, noise, u_cur, u_prev, dev), c["name"] + " states")
    assert_all_equal(vis_alias, BE.oracle_states(c, V, noise, u_cur, u_cur, dev), c["name"] + " states, u_prev = u_cur")
    for b in range(1, V):                  # a noisy row retraces cost rollout b up to its goal step
        frozen = np.nonzero((st[b, 1:] == st[b, :-1]).all(-1))[0]
        stop = c["T"] if not len(frozen) else int(frozen[0])
        assert_all_equal(vis_alias[b, :stop + 1], st[b, :stop + 1], "%s row %d" % (c["name"], b))
    return costs


@pytest.mark.parametrize("name", [c["name"] for c in BE.CASES])
def test_raw_planner_sweep(eng, dev, name):
    c = next(c for c in BE.CASES if c["name"] == name)
    _run_case(eng, dev, c, *BE.inputs(c))


@pytest.mark.parametrize("kind", OBSTACLE_KINDS)
def test_obstacle_boundary(eng, dev, kind):
    """Inputs built with this GPU's cos / sin so that the first step ends at distance exactly r from the obstacle's
    centre in float32: the kernel decides inside / outside as FFMA(-r, r, q) > 0 does, not as a split difference or >=."""
    case = BE.obstacle_boundary_case(dev, kind)
    assert case["alt_outside"] != case["exact_outside"]
    c, noise, u, _ = BE.directed_inputs(case)
    costs = _run_case(eng, dev, c, noise, u, u)
    paid = costs - BE.oracle_costs(c, noise, u, dev, obstacles=[])
    assert ((paid > 0.5 * c["obs_cost"]) == (not case["exact_outside"])).all()


@pytest.mark.parametrize("kind", GOAL_KINDS)
def test_goal_boundary(eng, dev, kind):
    """The goal test of the first step on its boundary (d2 == tol2, and a fused d2 on the other side of tol2 from the
    split one): the kernel decides as d2 = FFMA(dx, dx, dy*dy) <= tol2 does."""
    case = BE.goal_boundary_case(dev, kind)
    assert case["alt_reached"] != case["exact_reached"]
    c, noise, u, _ = BE.directed_inputs(case)
    costs = _run_case(eng, dev, c, noise, u, u)
    unreached = BE.oracle_costs(dict(c, tol=0.0), noise, u, dev)
    assert ((costs < unreached) == case["exact_reached"]).all()


# ----------------------------------------------------------------------------- Python planners and batches
def _planner(k, V=5, N=256, steps=24, nobs=3, **over):
    from mppi_numba_b200 import barebone as BB
    with quiet():
        pl = BB.MPPI_Numba(BB.Config(T=steps * 0.1 + 0.05, dt=0.1, num_control_rollouts=N, num_vis_state_rollouts=V,
                                     seed=11 + k))
    rng = np.random.default_rng(70 + k)
    p = dict(dt=[0.1, 0.08, 0.12, 0.1, 0.15][k % 5], x0=np.array([0.2 * k, -0.1 * k, 0.3 - 0.2 * k]),
             xgoal=np.array([3.0 - k, 2.0 + 0.5 * k]), goal_tolerance=0.3 + 0.05 * k, lambda_weight=[1.0, 0.3, 5.0, 0.05, 2.0][k % 5],
             num_opt=1, u_std=np.array([1.0 + 0.3 * k, 1.5 - 0.2 * k]), vrange=np.array([0.1 * k, 2.0]),
             wrange=np.array([-np.pi, np.pi]))
    if nobs:
        p.update(obstacle_positions=rng.uniform(-0.5, 3.0, (nobs, 2)), obstacle_radius=rng.uniform(0.05, 0.5, nobs))
    p.update(over)
    pl.setup(p)
    u0 = np.stack([rng.uniform(-0.3, 2.3, pl.num_steps), rng.uniform(-3.5, 3.5, pl.num_steps)], 1).astype(F32)
    pl.u_cur_d.copy_to_device(u0)
    return pl, u0


def _case_of(pl):
    """The planner's parameters as an edge-case dict (for the oracle helpers)."""
    p = pl.params
    ob = obstacles(pl)
    return BE._base("planner", pl.num_control_rollouts, pl.num_steps, x0=tuple(np.asarray(p["x0"], F32)),
                    goal=tuple(np.asarray(p["xgoal"], F32)), tol=p["goal_tolerance"], dt=p["dt"], lam=p["lambda_weight"],
                    u_std=tuple(p["u_std"]), vrange=tuple(p["vrange"]), wrange=tuple(p["wrange"]),
                    obs_cost=p.get("obs_penalty", 1e3), dist_weight=p.get("dist_weight", 10), obstacles=ob)


def _vis_oracle(pl, dev):
    c = _case_of(pl)
    return BE.oracle_states(c, pl.num_vis_state_rollouts, pl.noise_samples_d.copy_to_host(), pl.u_cur_d.copy_to_host(),
                            pl.u_prev_d.copy_to_host(), dev)


@pytest.mark.parametrize("V", [1, 5, 32, 33, 100])
def test_get_state_rollout(eng, dev, V):
    """One planner after a solve and a shift (u_cur != u_prev): row 0 the shifted optimal sequence, rows b > 0 the
    solve's noisy samples; V > 32 spans several blocks."""
    pl, _ = _planner(1, V=V)
    with quiet():
        u = pl.solve()
        pl.shift_and_update(np.array([0.15, -0.05, 0.4]), u, 1)
    assert not (pl.u_cur_d.copy_to_host() == pl.u_prev_d.copy_to_host()).all()
    with quiet():
        got = pl.get_state_rollout()
    assert_all_equal(got, _vis_oracle(pl, dev), "get_state_rollout, V %d" % V)


def test_batch_get_state_rollout(eng, dev):
    """state_rollout_batch_kernel: K = 3 planners with their own obstacles, starts, dt and bounds, V = 33."""
    from mppi_numba_b200 import MPPI_Batch
    pls = [_planner(k, V=33, nobs=[0, 4, 9][k])[0] for k in range(3)]
    batch = MPPI_Batch(pls)
    with quiet():
        u = batch.solve()
        for k, pl in enumerate(pls):
            pl.shift_and_update(np.asarray(pl.params["x0"]) + [0.05 * k, 0.02, -0.1], u[k], 1)
        got = batch.get_state_rollout()
    for k, pl in enumerate(pls):
        assert_all_equal(got[k], _vis_oracle(pl, dev), "batch get_state_rollout, planner %d" % k)


def test_batch_solve(eng, dev):
    """One MPPI_Batch.solve() of 5 planners with 0, 1, 3, 64 and 300 obstacles and their own goals, dt, lambda and
    u_std: every cost against the oracle from the planner's u before the solve and the noise it drew; u and the weights
    within the update's bounds."""
    from mppi_numba_b200 import MPPI_Batch
    made = [_planner(k, nobs=n, N=512) for k, n in enumerate([0, 1, 3, 64, 300])]
    pls = [m[0] for m in made]
    with quiet():
        u = MPPI_Batch(pls).solve()
    for k, (pl, u0) in enumerate(made):
        c = _case_of(pl)
        noise, costs = pl.noise_samples_d.copy_to_host(), pl.costs_d.copy_to_host()
        assert_all_equal(costs, BE.oracle_costs(c, noise, u0, dev), "batch planner %d costs" % k)
        RB.check_update(u[k], pl.weights_d.copy_to_host(), costs, noise, u0, c["lam"], c["vrange"], c["wrange"],
                        label="batch planner %d" % k)
        assert (pl.u_cur_d.copy_to_host() == u[k]).all()


def test_device_trial_contacts_on_the_circle(eng):
    """A barebone device trial with fixed controls (vrange [2, 2], wrange [0, 0], heading 0, dt 0.125: every plant step
    moves x by exactly 0.25).  Pose x = 0.75 lies exactly on the circle of the obstacle (0.8125, 0, 0.0625) in float64,
    and poses 1.75, 2.0 and 2.25 inside (2, 0, 0.3): contact_steps counts the boundary step, as in_contact does."""
    from mppi_numba_b200 import MPPI_Batch
    from mppi_numba_b200 import barebone as BB
    steps = 12
    with quiet():
        pl = BB.MPPI_Numba(BB.Config(T=1.0, dt=0.125, num_control_rollouts=128, seed=5))
    pl.setup(dict(dt=0.125, x0=np.array([0.0, 0.0, 0.0]), xgoal=np.array([100.0, 0.0]), goal_tolerance=0.5,
                  lambda_weight=1.0, num_opt=1, u_std=np.array([1.0, 1.0]), vrange=np.array([2.0, 2.0]),
                  wrange=np.array([0.0, 0.0]), obstacle_positions=np.array([[0.8125, 0.0], [2.0, 0.0]]),
                  obstacle_radius=np.array([0.0625, 0.3])))
    with quiet():
        out = MPPI_Batch([pl]).run_barebone_trials(steps)
    assert out["status"][0] == "max_steps" and out["steps"][0] == steps
    xh = out["xhist"][0]
    assert (xh[:, 0] == 0.25 * np.arange(steps + 1)).all() and (xh[:, 1:] == 0).all()
    obs = obstacles(pl)
    touched = [t for t in range(1, steps + 1) if in_contact(xh[t], obs)]
    assert touched == [3, 7, 8, 9]
    strict = [t for t in touched if not any((xh[t, 0] - o[0]) ** 2 + (xh[t, 1] - o[1]) ** 2 == float(o[2]) ** 2
                                            for o in obs.astype(np.float64))]
    assert strict == [7, 8, 9]                           # the boundary step is the one a strict test would drop
    assert out["contact_steps"][0] == len(touched) == out["logs"][0]["contact_steps"]


# ----------------------------------------------------------------------------- every cost +inf
def test_solve_with_every_cost_inf(eng, dev):
    """obs_penalty 1e38 and a start inside a 50 m obstacle: four steps inside overflow float32, so every cost is +inf.
    The update takes a zero step -- u == clip(u0), with u0 outside the bounds in places -- and every weight is 0, in the
    planner's own solve and in a batch next to a planner with finite costs (whose update stays within its bounds)."""
    from mppi_numba_b200 import MPPI_Batch
    big = dict(obs_penalty=1e38, obstacle_positions=np.array([[0.0, 0.0]]), obstacle_radius=np.array([50.0]),
               vrange=np.array([0.0, 1.0]), wrange=np.array([-1.0, 1.0]), x0=np.array([0.1, 0.2, 0.3]))
    for label, batched in (("solve", False), ("batch", True)):
        pl, u0 = _planner(0, nobs=0, steps=10, **big)
        other, u0o = _planner(2, nobs=3, steps=10)
        with quiet():
            u = MPPI_Batch([pl, other]).solve() if batched else pl.solve()[None]
        c = _case_of(pl)
        noise, costs = pl.noise_samples_d.copy_to_host(), pl.costs_d.copy_to_host()
        assert np.isposinf(costs).all(), label
        assert_all_equal(costs, BE.oracle_costs(c, noise, u0, dev), label + " costs")
        RB.check_update(u[0], pl.weights_d.copy_to_host(), costs, noise, u0, c["lam"], c["vrange"], c["wrange"],
                        label=label)
        assert not (u0 == u[0]).all()                    # the clip moved u0
        if batched:
            co = _case_of(other)
            RB.check_update(u[1], other.weights_d.copy_to_host(), other.costs_d.copy_to_host(),
                            other.noise_samples_d.copy_to_host(), u0o, co["lam"], co["vrange"], co["wrange"],
                            label="batch, finite planner")
