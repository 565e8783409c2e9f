"""The plant-step kernel of closed-loop trials (csrc/reduce.cu, ``[emu:... trial]``) emulated on the host against a
numpy restatement of one step of the benchmark's trial() (tests/trial_loop.py), bit for bit: the traction lookup at
cell edges, negative offsets and just outside the grid, int8 grids, the float64 state update, the shift of u, the
float32 x0 of the next rollout, the metrics and the stopping rules."""
import ctypes as C

import numpy as np
import pytest

from mppi_numba_b200.terrain import TractionGrid
from tests import emu_trial
from tests.trial_loop import plant_step

GOAL, MAX_STEPS, LEFT_MAP = 1, 2, 3


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_trial.build(str(tmp_path_factory.mktemp("trial_emu")))


class Planner(object):
    def __init__(self, grid, x, u, xgoal, tol=0.5, dt=0.1, pxlim=(-1e9, 1e9), pylim=(-1e9, 1e9), cum=(0.0, 0.0)):
        self.grid, self.x, self.u = grid, np.asarray(x, dtype=np.float64), np.ascontiguousarray(u, dtype=np.float32)
        self.xgoal, self.tol, self.dt, self.pxlim, self.pylim, self.cum = np.asarray(xgoal, float), tol, dt, pxlim, pylim, cum


def run(emu, pls, step, max_steps):
    K, T = len(pls), pls[0].u.shape[0]
    lin = [np.ascontiguousarray(p.grid.lin_traction, dtype=np.float64) for p in pls]
    ang = [np.ascontiguousarray(p.grid.ang_traction, dtype=np.float64) for p in pls]
    g = np.array([[p.grid.xlimits[0], p.grid.ylimits[0], p.grid.res, p.dt, p.xgoal[0], p.xgoal[1], p.tol,
                   p.pxlim[0], p.pxlim[1], p.pylim[0], p.pylim[1]] for p in pls], dtype=np.float64)
    u = [p.u.copy() for p in pls]
    x0 = [np.zeros(3, np.float32) for _ in pls]
    nbytes = emu.emu_state_bytes()
    assert nbytes == 56
    state = np.zeros((K, 7), dtype=np.float64)
    for k, p in enumerate(pls):
        state[k, :3] = p.x
        state[k, 3:5] = p.cum
    active = np.ones(K, dtype=np.int32)
    count = np.array([K], dtype=np.int32)
    xh = np.full((K, max_steps + 1, 3), -7.0)
    uh = np.full((K, max_steps, 2), -7.0, dtype=np.float32)
    P = lambda arrs: (C.c_void_p * K)(*[a.ctypes.data for a in arrs])      # noqa: E731
    Hs, Ws = np.array([a.shape[0] for a in lin], np.int32), np.array([a.shape[1] for a in lin], np.int32)
    emu.emu_plant(K, T, max_steps, step, P(lin), P(ang), Hs.ctypes.data, Ws.ctypes.data, g.ctypes.data, P(u), P(x0),
                  state.ctypes.data, active.ctypes.data, count.ctypes.data, xh.ctypes.data, uh.ctypes.data)
    ints = state[:, 6].copy().view(np.int32).reshape(K, 2)
    return dict(u=u, x0=x0, x=state[:, :3], cum_obj=state[:, 3], cum_dist=state[:, 4], dist=state[:, 5],
                steps=ints[:, 0], status=ints[:, 1], active=active, count=int(count[0]), xh=xh, uh=uh)


def expect(p, step, max_steps):
    """numpy restatement of one trial() step and of the stopping rules."""
    xn = plant_step(p.grid, p.x, p.u[0], p.dt)
    dx, dy = xn[0] - p.xgoal[0], xn[1] - p.xgoal[1]
    d = np.sqrt(dx * dx + dy * dy) - p.tol
    if d <= 0:
        status = GOAL
    elif not (p.pxlim[0] <= xn[0] <= p.pxlim[1] and p.pylim[0] <= xn[1] <= p.pylim[1]):
        status = LEFT_MAP
    elif step + 1 >= max_steps:
        status = MAX_STEPS
    else:
        status = 0
    u = p.u.copy()
    u[:-1] = u[1:]
    return dict(x=xn, d=d, cum_obj=p.cum[0] + (p.dt + d), cum_dist=p.cum[1] + d, status=status, u=u)


def check(emu, pls, step=0, max_steps=10):
    got = run(emu, pls, step, max_steps)
    stopped = 0
    for k, p in enumerate(pls):
        w = expect(p, step, max_steps)
        assert np.array_equal(got["x"][k], w["x"]), (k, got["x"][k], w["x"])
        assert np.array_equal(got["xh"][k, step + 1], w["x"]) and np.array_equal(got["uh"][k, step], p.u[0])
        assert np.array_equal(got["x0"][k], w["x"].astype(np.float32))
        assert np.array_equal(got["u"][k], w["u"]), k
        assert got["dist"][k] == w["d"] and got["cum_obj"][k] == w["cum_obj"] and got["cum_dist"][k] == w["cum_dist"]
        assert got["steps"][k] == step + 1 and got["status"][k] == w["status"], (k, got["status"][k], w["status"])
        assert got["active"][k] == (w["status"] == 0)
        stopped += w["status"] != 0
    assert got["count"] == len(pls) - stopped
    return got


def grid(rng, H=12, W=15, res=0.25, xlo=0.0, ylo=0.0, int8=False):
    return TractionGrid(rng.uniform(0.1, 1.0, (H, W)), rng.uniform(0.1, 1.0, (H, W)), res=res, use_int8=int8,
                        xlimits=(xlo, xlo + W * res), ylimits=(ylo, ylo + H * res))


def controls(rng, T):
    return np.stack([rng.uniform(-1, 3, T), rng.uniform(-2, 2, T)], 1)


def test_lookup_on_cell_edges_negative_offsets_and_just_outside(emu):
    rng = np.random.default_rng(1)
    pls = []
    for res, xlo, ylo in ((0.25, 0.0, 0.0), (0.1, -1.3, -0.7), (0.3, -2.05, 1.15)):
        g = grid(rng, res=res, xlo=xlo, ylo=ylo)
        W, H = g.width, g.height
        xs = [xlo + i * res for i in range(W + 1)] + [xlo - 1e-12, xlo + W * res - 1e-12, xlo + W * res + 1e-12,
                                                       np.nextafter(xlo, -np.inf), xlo + 0.5 * res]
        ys = [ylo + j * res for j in range(H + 1)] + [ylo - 1e-12, np.nextafter(ylo + H * res, -np.inf)]
        for x in xs:
            for y in ys[::3] + ys[-2:]:
                pls.append(Planner(g, [x, y, rng.uniform(-4, 4)], controls(rng, 6), xgoal=[100.0, 100.0]))
    got = check(emu, pls)
    zero = sum(p.grid.get(p.x[0], p.x[1]) == (0, 0) for p in pls)
    assert 0 < zero < len(pls)                                   # both sides of the grid's edges are exercised
    assert got["count"] == len(pls)


def test_int8_grids(emu):
    rng = np.random.default_rng(2)
    pls = [Planner(grid(rng, int8=True, xlo=-0.4), [rng.uniform(-0.5, 3.8), rng.uniform(-0.2, 3.2), rng.uniform(-3, 3)],
                   controls(rng, 5), xgoal=[500.0, 0.0], dt=0.05) for _ in range(40)]
    assert pls[0].grid.lin_traction.dtype == np.int8
    check(emu, pls)


def test_goal_on_first_and_last_step_max_steps_and_leaving_the_map(emu):
    rng = np.random.default_rng(3)
    g = grid(rng)
    near = Planner(g, [1.0, 1.0, 0.3], controls(rng, 4), xgoal=[1.1, 1.05], cum=(0.0, 0.0))
    far = Planner(g, [1.0, 1.0, 0.3], controls(rng, 4), xgoal=[9.0, 9.0], cum=(1.25, -0.5))
    u = np.tile([[3.0, 0.0]], (4, 1))
    out = Planner(g, [3.7, 1.0, 0.0], u, xgoal=[90.0, 1.0], pxlim=(-0.75, 3.71), pylim=(-0.75, 3.75))
    got = check(emu, [near, far, out], step=0, max_steps=5)
    assert got["status"].tolist() == [GOAL, 0, LEFT_MAP]
    last = Planner(g, [1.0, 1.0, 0.3], controls(rng, 4), xgoal=[1.1, 1.05], cum=(3.0, 2.0))
    got = check(emu, [last, far], step=4, max_steps=5)
    assert got["status"].tolist() == [GOAL, MAX_STEPS] and got["steps"].tolist() == [5, 5]


def test_shift_of_one_row_and_long_sequences(emu):
    rng = np.random.default_rng(4)
    g = grid(rng)
    for T in (1, 2, 17, 33, 100):
        pls = [Planner(g, [rng.uniform(0, 3.7), rng.uniform(0, 2.9), rng.uniform(-3, 3)], controls(rng, T),
                       xgoal=[50.0, 50.0]) for _ in range(3)]
        check(emu, pls, step=2, max_steps=8)


def test_stopped_planners_are_left_alone(emu):
    rng = np.random.default_rng(5)
    g = grid(rng)
    p = Planner(g, [1.0, 1.0, 0.0], controls(rng, 5), xgoal=[50.0, 50.0])
    K, T = 2, 5
    lin = np.ascontiguousarray(g.lin_traction, dtype=np.float64)
    arrs = [lin, lin]
    gg = np.tile(np.array([0, 0, g.res, 0.1, 50, 50, 0.5, -9, 9, -9, 9], np.float64), (K, 1))
    u = [p.u.copy(), p.u.copy()]
    x0 = [np.zeros(3, np.float32), np.zeros(3, np.float32)]
    state = np.zeros((K, 7))
    state[:, :3] = p.x
    active = np.array([0, 1], np.int32)
    count = np.array([1], np.int32)
    xh, uh = np.zeros((K, 4, 3)), np.zeros((K, 3, 2), np.float32)
    P = lambda a: (C.c_void_p * K)(*[x.ctypes.data for x in a])      # noqa: E731
    hw = np.array([g.height, g.height], np.int32), np.array([g.width, g.width], np.int32)
    emu.emu_plant(K, T, 3, 0, P(arrs), P(arrs), hw[0].ctypes.data, hw[1].ctypes.data, gg.ctypes.data, P(u), P(x0),
                  state.ctypes.data, active.ctypes.data, count.ctypes.data, xh.ctypes.data, uh.ctypes.data)
    assert np.array_equal(u[0], p.u) and not x0[0].any() and not xh[0].any() and not uh[0].any()
    assert np.array_equal(state[0, :3], p.x) and not state[0, 3:].any()
    assert not np.array_equal(u[1], p.u) and xh[1, 1].any()
