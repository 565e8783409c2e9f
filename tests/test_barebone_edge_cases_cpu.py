"""The barebone (map-free) edge cases of tests/barebone_edge_cases.py on the host: the tables reach what they claim, each
directed boundary case separates the exact rule from its alternative (libm provider), and the REAL source of the
barebone rollout kernel and of the visualisation kernels (tests/emu_rollout.py, tests/emu_vis_batch.py) equals the
exact oracle bit for bit on every case."""
import ctypes as C

import numpy as np
import pytest

from tests import barebone_edge_cases as BE
from tests import emu_rollout, emu_vis_batch
from tests.test_exact_oracle_cpu import EXACT

F32 = np.float32
MODE_BAREBONE = 3
OBSTACLE_KINDS = ["up", "up_ahead", "down", "on_circle"]
GOAL_KINDS = ["on_tol", "split"]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_rollout.build(str(tmp_path_factory.mktemp("emu_bb_rollout")))


@pytest.fixture(scope="module")
def emu_vis(tmp_path_factory):
    return emu_vis_batch.build(str(tmp_path_factory.mktemp("emu_bb_vis")))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def fparams(c):
    """The 23 floats of tests/emu_cuda.h's params for a barebone case (no map: res 1, origin 0, bounds 0)."""
    x0, g, us, vr, wr = c["x0"], c["goal"], c["u_std"], c["vrange"], c["wrange"]
    return np.ascontiguousarray([1.0, 0.0, 0.0, c["dt"], x0[0], x0[1], x0[2], g[0], g[1], c["tol"], 0.0, c["lam"], us[0],
                                 us[1], vr[0], vr[1], wr[0], wr[1], c["obs_cost"], 0.0, c["dist_weight"], 0.0, 0.0], F32)


def emu_costs(emu, c, noise, u_cur):
    N, T = c["N"], c["T"]
    geo = np.ascontiguousarray([1, 1, 1, 1, 1, 1, T, N, 1], np.int32)
    ob = np.ascontiguousarray(c["obstacles"], F32)
    costs = np.zeros(N, F32)
    emu.emu_rollout(MODE_BAREBONE, _p(fparams(c)), _p(geo), _p(np.array([0.0, 0.0])), None, None, None, None, None,
                    _p(np.ascontiguousarray(noise)), _p(np.ascontiguousarray(u_cur)), None, _p(costs),
                    _p(ob) if len(ob) else None, len(ob))
    return costs


def emu_states(emu, c, V, noise, u_cur, u_prev):
    geo = np.ascontiguousarray([1, 1, 1, 1, 1, 1, c["T"], c["N"], 1], np.int32)
    out = np.zeros((V, c["T"] + 1, 3), F32)
    emu.emu_state_rollout(MODE_BAREBONE, V, _p(fparams(c)), _p(geo), _p(np.array([0.0, 0.0])), None, None,
                          _p(np.ascontiguousarray(noise)), _p(np.ascontiguousarray(u_cur)),
                          _p(np.ascontiguousarray(u_prev)), _p(out))
    return out


def bits_equal(got, want, what):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, "%s: %d of %d differ; first: %s" % (what, len(bad), got.size,
                                                             [(tuple(map(int, ix)), float(got[tuple(ix)]),
                                                               float(want[tuple(ix)])) for ix in bad[:4]])


def _inside(states, ob):
    """(N, T+1) count of obstacles each state lies in, by the rollout's rule (FFMA(-r, r, q) <= 0), libm arithmetic."""
    x, y = states[..., 0][..., None], states[..., 1][..., None]
    ddx, ddy = EXACT.sub32(x, ob[:, 0]), EXACT.sub32(y, ob[:, 1])
    diff = EXACT.fma32(-ob[:, 2], ob[:, 2], EXACT.fma32(ddx, ddx, EXACT.mul32(ddy, ddy)))
    return (diff <= 0).sum(-1)


# ----------------------------------------------------------------------------- the tables
def test_tables_reach_what_they_claim():
    by = {c["name"]: c for c in BE.CASES}
    assert {c["N"] for c in BE.CASES} >= set(BE.SHAPE_N) and {c["T"] for c in BE.CASES} >= set(BE.SHAPE_T)
    assert any(c["N"] < 100 for c in BE.CASES) and any(c["N"] % 128 and c["N"] > 128 for c in BE.CASES)
    counts = {len(c["obstacles"]) for c in BE.CASES}
    assert counts >= set(BE.OBSTACLE_COUNTS)
    for c in BE.CASES:
        if len(c["obstacles"]) >= 256:
            assert c["N"] * c["T"] <= 1000, c["name"]
    runs = {}
    for name in ("overlapping", "x0-inside", "goal-inside", "radius-0", "goal-step-1", "obstacles-4096"):
        c = by[name]
        noise, u_cur, _ = BE.inputs(c)
        runs[name] = (c, BE.oracle_costs(c, noise, u_cur, EXACT, return_states=True))
    # one step pays the penalty once per obstacle: some state lies in several
    c, (_, st) = runs["overlapping"]
    assert _inside(st[:, 1:], c["obstacles"]).max() >= 3
    assert _inside(runs["obstacles-4096"][1][1][:, 1:], by["obstacles-4096"]["obstacles"]).max() >= 1
    c = by["x0-inside"]
    assert _inside(np.asarray(c["x0"], F32)[None, None], c["obstacles"])[0, 0] == 1
    c, (costs, st) = runs["goal-inside"]
    assert _inside(np.array([[c["goal"]]], F32), c["obstacles"])[0, 0] == 1
    d2 = ((st[..., 0] - F32(c["goal"][0])) ** 2 + (st[..., 1] - F32(c["goal"][1])) ** 2)
    assert (d2 <= F32(c["tol"]) ** 2).any()                     # some rollouts reach it (and stop there)
    # radius 0 on a visited point: row 0 stands on the centre after step 1, which counts as inside (diff = 0)
    c, (_, st) = runs["radius-0"]
    assert tuple(st[0, 1, :2]) == tuple(c["obstacles"][0, :2]) and c["obstacles"][0, 2] == 0
    assert _inside(st[:1, 1:2], c["obstacles"][:1])[0, 0] == 1
    # goal reached at step 1 inside an obstacle: row 0 stops there and has paid that step's penalty
    c, (costs, st) = runs["goal-step-1"]
    assert tuple(st[0, 1, :2]) == (F32(c["goal"][0]), F32(c["goal"][1])) and (st[0, 2:] == st[0, 1]).all()
    assert costs[0] >= F32(c["obs_cost"])
    c = by["subnormal-theta0"]
    th = F32(c["x0"][2])
    assert th != 0 and abs(th) < np.finfo(F32).tiny
    assert any(c["vrange"][0] > 0 for c in BE.CASES) and any(c["lam"] < 0.1 for c in BE.CASES)
    assert any(c["lam"] > 10 for c in BE.CASES) and len({c["u_std"] for c in BE.CASES}) >= 3
    # the noisy controls leave vrange and wrange on both sides, so the clip is exercised
    noise, u_cur, _ = BE.inputs(by["values-a"])
    v = u_cur[None, :, 0] + noise[..., 0]
    assert (v < F32(0.3)).any() and (v > F32(1.7)).any()


@pytest.mark.parametrize("kind", OBSTACLE_KINDS)
def test_obstacle_boundary_cases_separate_the_alternative(kind):
    case = BE.obstacle_boundary_case(EXACT, kind)
    assert case["exact_outside"] == (kind in ("up", "up_ahead"))
    assert case["alt_outside"] != case["exact_outside"], case
    # and the exact oracle's cost shows that decision: the penalty is paid exactly when the rule says inside
    c, noise, u, _ = BE.directed_inputs(case)
    with_ob = BE.oracle_costs(c, noise, u, EXACT, return_states=True)
    without = BE.oracle_costs(c, noise, u, EXACT, obstacles=[])
    assert tuple(with_ob[1][0, 1, :2]) == case["x1"]
    paid = with_ob[0] - without
    assert ((paid > 0.5 * c["obs_cost"]) == (not case["exact_outside"])).all()


@pytest.mark.parametrize("kind", GOAL_KINDS)
def test_goal_boundary_cases_separate_the_alternative(kind):
    case = BE.goal_boundary_case(EXACT, kind)
    assert case["alt_reached"] != case["exact_reached"], case
    c, noise, u, _ = BE.directed_inputs(case)
    costs = BE.oracle_costs(c, noise, u, EXACT)
    far = dict(c, tol=0.0)                                         # the same rollout with the goal never reached
    d2_term = costs - BE.oracle_costs(far, noise, u, EXACT)
    assert ((d2_term < 0) == case["exact_reached"]).all()           # reached: no terminal cost d2


# ----------------------------------------------------------------------------- emulated kernels against the oracle
def _directed():
    out = [BE.directed_inputs(BE.obstacle_boundary_case(EXACT, k)) for k in OBSTACLE_KINDS]
    return out + [BE.directed_inputs(BE.goal_boundary_case(EXACT, k)) for k in GOAL_KINDS]


@pytest.mark.parametrize("name", [c["name"] for c in BE.CASES] + ["directed"])
def test_emulated_kernels_equal_the_oracle(emu, name):
    """Every cost of the barebone rollout kernel and every state of the visualisation kernel's mode 3 (V <= 33 rows, u_prev
    != u_cur) equal the exact oracle (libm provider), and the noisy visualisation rows equal the cost rollout's states
    up to each row's goal step when u_prev = u_cur (the solve's alias)."""
    runs = _directed() if name == "directed" else [(c, *BE.inputs(c)) for c in BE.CASES if c["name"] == name]
    for c, noise, u_cur, u_prev in runs:
        want, st = BE.oracle_costs(c, noise, u_cur, EXACT, return_states=True)
        bits_equal(emu_costs(emu, c, noise, u_cur), want, c["name"] + " costs")
        V = BE.vis_count(c)
        bits_equal(emu_states(emu, c, V, noise, u_cur, u_prev), BE.oracle_states(c, V, noise, u_cur, u_prev, EXACT),
                   c["name"] + " states")
        vis = emu_states(emu, c, V, noise, u_cur, u_cur)
        bits_equal(vis, BE.oracle_states(c, V, noise, u_cur, u_cur, EXACT), c["name"] + " states, u_prev = u_cur")
        for b in range(1, V):
            frozen = np.nonzero((st[b, 1:] == st[b, :-1]).all(-1))[0]
            stop = c["T"] if not len(frozen) else int(frozen[0])    # after the goal step the cost rollout stands still
            bits_equal(vis[b, :stop + 1], st[b, :stop + 1], "%s row %d" % (c["name"], b))


def test_emulated_batched_vis_equals_the_oracle(emu_vis):
    """state_rollout_batch_kernel over K = 3 barebone planners (own starts, dt, bounds, noise, u_cur and u_prev; V = 33,
    two blocks): every state equals the oracle."""
    names = ["values-a", "values-b", "shape-N129-T1024"]
    cs = [dict(c) for c in BE.CASES if c["name"] in names]
    T = 40
    V = 33
    f, g, noise, u_cur, u_prev, outs = [], [], [], [], [], []
    for k, c in enumerate(cs):
        c.update(T=T, N=V + 4, x0=(0.1 * k, -0.3 * k, 0.2 - 0.4 * k))
        n, uc, up = BE.inputs(c)
        f.append(fparams(c))
        g.append([1, 1, 1, 1, 1, 1, T, c["N"], 1])
        noise.append(np.ascontiguousarray(n))
        u_cur.append(np.ascontiguousarray(uc))
        u_prev.append(np.ascontiguousarray(up))
        outs.append(np.zeros((V, T + 1, 3), F32))
    K = len(cs)
    ptrs = lambda arrs: (C.c_void_p * K)(*[a.ctypes.data if a is not None else None for a in arrs])   # noqa: E731
    f, g = np.ascontiguousarray(f, F32), np.ascontiguousarray(g, np.int32)
    emu_vis.emu_vis(K, 1, _p(np.full(K, MODE_BAREBONE, np.int32)), V, _p(f), _p(g), _p(np.zeros(2 * K)),
                    ptrs([None] * K), ptrs([None] * K), ptrs(noise), ptrs(u_cur), ptrs(u_prev), ptrs(outs), None,
                    C.c_size_t(0))
    for k, c in enumerate(cs):
        bits_equal(outs[k], BE.oracle_states(c, V, noise[k], u_cur[k], u_prev[k], EXACT), "planner %d" % k)
