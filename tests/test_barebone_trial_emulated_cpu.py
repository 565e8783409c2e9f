"""The plant step of barebone closed-loop trials (csrc/reduce.cu, ``[emu:... trial]`` with TrialDev::lin null and
PlantArgs::contacts set) emulated on the host against the numpy restatement of the notebook's loop
(tests/barebone_trial_loop.py), bit for bit: the nominal unicycle step, the goal and step-limit stops with no map to
leave, and the obstacle contacts -- poses exactly on a circle and one float64 ulp either side of it, overlapping
obstacles, none at all, a start inside one.  Stopped planners are left alone, and a map trial with obstacles in its
descriptor but no contact buffer is the map trial of tests/test_trial_emulated_cpu.py."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_trial
from tests.barebone_trial_loop import in_contact, plant_step
from tests.test_trial_emulated_cpu import Planner as MapPlanner
from tests.test_trial_emulated_cpu import controls, expect, grid

GOAL, MAX_STEPS = 1, 2

HARNESS = r'''
// emu_plant with each planner's obstacles (obs[i]: nobs[i] rows x, y, r; null for none) and the per-planner contact
// counts (null: a map trial's PlantArgs); lin[i] null: a barebone planner
extern "C" void emu_plant_obs(int K, int T, int max_steps, int step, const double** lin, const double** ang, const int* H,
                              const int* W, const double* g, float** u_cur, float** x0_out, const float** obs,
                              const int* nobs, void* state, int* active, int* count, double* xhist, float* uhist,
                              int* contacts) {
  std::vector<TrialDev> d(K);
  for (int i = 0; i < K; ++i) {
    const double* q = g + 11 * i;
    d[i] = TrialDev{lin[i], ang[i], H[i], W[i], q[0], q[1], q[2], q[3], {q[4], q[5]}, q[6], {q[7], q[8]}, {q[9], q[10]},
                    u_cur[i], x0_out[i]};
    d[i].obstacles = obs[i];
    d[i].num_obstacles = nobs[i];
  }
  PlantArgs a{d.data(), reinterpret_cast<TrialState*>(state), active, count, xhist, uhist, K, T, max_steps, step,
              contacts};
  emu::launch({(unsigned)K, 1, 1}, 32, [&] { plant_step_body(a, (int)blockIdx.x, (int)threadIdx.x); });
}
'''


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_trial.build(str(tmp_path_factory.mktemp("bb_trial_emu")), extra=HARNESS)


class Planner(object):
    """A barebone planner's trial state: pose x, controls u, goal, obstacles (n, 3) float32."""

    def __init__(self, x, u, xgoal, obs=(), tol=0.5, dt=0.1, cum=(0.0, 0.0), contacts=0):
        self.x, self.u = np.asarray(x, dtype=np.float64), np.ascontiguousarray(u, dtype=np.float32)
        self.xgoal, self.tol, self.dt, self.cum = np.asarray(xgoal, float), tol, dt, cum
        self.obs = np.ascontiguousarray(np.asarray(obs, dtype=np.float32).reshape(-1, 3))
        self.contacts = contacts


def run(emu, pls, step, max_steps, active=None, contacts=True):
    """One launch of the plant step over pls (barebone Planners, or MapPlanners whose obstacles are ``p.obs``)."""
    K, T = len(pls), pls[0].u.shape[0]
    maps = [getattr(p, "grid", None) for p in pls]
    lin = [None if g is None else np.ascontiguousarray(g.lin_traction, dtype=np.float64) for g in maps]
    ang = [None if g is None else np.ascontiguousarray(g.ang_traction, dtype=np.float64) for g in maps]
    g = np.array([[0.0, 0.0, 0.0, p.dt, p.xgoal[0], p.xgoal[1], p.tol, 0.0, 0.0, 0.0, 0.0] if m is None else
                  [m.xlimits[0], m.ylimits[0], m.res, p.dt, p.xgoal[0], p.xgoal[1], p.tol, p.pxlim[0], p.pxlim[1],
                   p.pylim[0], p.pylim[1]] for p, m in zip(pls, maps)], dtype=np.float64)
    u = [p.u.copy() for p in pls]
    x0 = [np.zeros(3, np.float32) for _ in pls]
    obs = [p.obs for p in pls]
    state = np.zeros((K, 7), dtype=np.float64)
    for k, p in enumerate(pls):
        state[k, :3] = p.x
        state[k, 3:5] = p.cum
    act = np.ones(K, dtype=np.int32) if active is None else np.array(active, dtype=np.int32)
    count = np.array([int(act.sum())], dtype=np.int32)
    xh = np.full((K, max_steps + 1, 3), -7.0)
    uh = np.full((K, max_steps, 2), -7.0, dtype=np.float32)
    con = np.array([getattr(p, "contacts", 0) for p in pls], dtype=np.int32)
    P = lambda arrs: (C.c_void_p * K)(*[None if a is None or not a.size else a.ctypes.data for a in arrs])  # noqa: E731
    Hs = np.array([0 if a is None else a.shape[0] for a in lin], np.int32)
    Ws = np.array([0 if a is None else a.shape[1] for a in lin], np.int32)
    nobs = np.array([len(o) for o in obs], np.int32)
    emu.emu_plant_obs(K, T, max_steps, step, P(lin), P(ang), Hs.ctypes.data, Ws.ctypes.data, g.ctypes.data, P(u),
                      P(x0), P(obs), nobs.ctypes.data, state.ctypes.data, act.ctypes.data, count.ctypes.data,
                      xh.ctypes.data, uh.ctypes.data, con.ctypes.data if contacts else None)
    ints = state[:, 6].copy().view(np.int32).reshape(K, 2)
    return dict(u=u, x0=x0, x=state[:, :3], cum_obj=state[:, 3], cum_dist=state[:, 4], dist=state[:, 5],
                steps=ints[:, 0], status=ints[:, 1], active=act, count=int(count[0]), xh=xh, uh=uh, contacts=con)


def bits(a):
    a = np.asarray(a)
    return a.dtype, a.shape, a.tobytes()


def check(emu, pls, step=0, max_steps=10):
    """One step of every planner against numpy, bit for bit; returns the kernel's outputs."""
    got = run(emu, pls, step, max_steps)
    stopped = 0
    for k, p in enumerate(pls):
        xn = plant_step(p.x, p.u[0], p.dt)
        dx, dy = xn[0] - p.xgoal[0], xn[1] - p.xgoal[1]
        d = np.sqrt(dx * dx + dy * dy) - p.tol
        status = GOAL if d <= 0 else MAX_STEPS if step + 1 >= max_steps else 0
        u = p.u.copy()
        u[:-1] = u[1:]
        assert bits(got["x"][k]) == bits(xn) and bits(got["xh"][k, step + 1]) == bits(xn), (k, got["x"][k], xn)
        assert bits(got["uh"][k, step]) == bits(p.u[0]) and bits(got["u"][k]) == bits(u), k
        assert bits(got["x0"][k]) == bits(xn.astype(np.float32)), k
        assert bits(got["dist"][k]) == bits(np.float64(d)), k
        assert bits(got["cum_obj"][k]) == bits(np.float64(p.cum[0] + (p.dt + d))), k
        assert bits(got["cum_dist"][k]) == bits(np.float64(p.cum[1] + d)), k
        assert got["steps"][k] == step + 1 and got["status"][k] == status, (k, got["status"][k], status)
        assert got["active"][k] == (status == 0)
        assert got["contacts"][k] == p.contacts + in_contact(xn, p.obs), (k, got["contacts"][k])
        stopped += status != 0
    assert got["count"] == len(pls) - stopped
    return got


def still(x, obs, contacts=0):
    """A planner that stays at pose x (v = w = 0: x + dt cos(th) 0 == x) next to obstacles obs."""
    return Planner(x, np.zeros((3, 2)), xgoal=[1e3, 1e3], obs=obs, contacts=contacts)


def test_nominal_steps(emu):
    rng = np.random.default_rng(1)
    obs = [[5.0, 4.5, 1.5], [2.0, 1.0, 1.0]]                      # the notebook's obstacles
    touched = total = 0
    for T in (1, 2, 17, 33, 50):
        pls = [Planner([rng.uniform(-1, 8), rng.uniform(-1, 6), rng.uniform(-4, 4)], controls(rng, T),
                       xgoal=[7.0, 5.0], obs=obs, dt=dt, cum=(rng.uniform(0, 5), rng.uniform(0, 5)))
               for dt in (0.1, 0.05, 0.3) for _ in range(8)]
        touched += int(check(emu, pls, step=3, max_steps=20)["contacts"].sum())
        total += len(pls)
    assert 0 < touched < total                                      # both sides of the obstacles' edges are exercised


def test_contact_on_the_circle_and_one_ulp_either_side(emu):
    pls, want = [], []
    for ox, oy, r in ((5.0, 4.5, 1.5), (2.0, 1.0, 1.0), (np.float32(1.1), np.float32(-0.7), np.float32(0.3)),
                      (np.float32(-3.3), np.float32(2.9), np.float32(0.05))):
        o = np.array([[ox, oy, r]], np.float32)
        X, Y, R = (float(v) for v in o[0])
        for sx, sy in ((1, 0), (-1, 0), (0, 1), (0, -1)):
            c = 0 if sx else 1
            on = np.array([X + sx * R, Y + sy * R, 0.3])
            assert in_contact(on, o)                                 # exactly on the circle: touching
            inward = on.copy()
            inward[c] = np.nextafter(on[c], (X, Y)[c])
            assert in_contact(inward, o)
            # outward: the offset from the centre one ulp of r beyond r at a time (the pose has coarser ulps than a
            # small r, and x - ox may round back onto r); the last pose that still touches and the first that does not
            last, out, off = on.copy(), on.copy(), R
            for _ in range(1024):
                off = np.nextafter(off, np.inf)
                out[c] = (X, Y)[c] + (sx + sy) * off
                if not in_contact(out, o):
                    break
                last = out.copy()
            assert not in_contact(out, o) and in_contact(last, o)
            pls += [still(on, o), still(inward, o), still(last, o), still(out, o)]
            want += [True, True, True, False]
    got = check(emu, pls)
    assert got["contacts"].astype(bool).tolist() == want


def test_overlapping_obstacles_count_once_and_no_obstacles(emu):
    overlap = [[0.0, 0.0, 1.0], [0.2, 0.1, 1.0], [-0.1, 0.3, 0.8], [9.0, 9.0, 0.5]]
    pls = [still([0.05, 0.1, 0.0], overlap), still([0.05, 0.1, 0.0], overlap, contacts=4),
           still([5.0, 5.0, 0.0], overlap), still([0.05, 0.1, 0.0], ())]
    got = check(emu, pls)
    assert got["contacts"].tolist() == [1, 5, 0, 0]


def test_start_inside_an_obstacle(emu):
    o = [[1.0, 1.0, 0.5]]
    stay = Planner([1.1, 0.9, 0.0], np.tile([[0.5, 0.0]], (4, 1)), xgoal=[9.0, 9.0], obs=o)      # 5 cm: still inside
    leave = Planner([1.1, 0.9, 0.0], np.tile([[6.0, 0.0]], (4, 1)), xgoal=[9.0, 9.0], obs=o)     # 60 cm: out
    got = check(emu, [stay, leave])
    assert got["contacts"].tolist() == [1, 0]


def test_goal_on_the_first_and_last_step_max_steps_and_no_map_to_leave(emu):
    rng = np.random.default_rng(3)
    near = Planner([1.0, 1.0, 0.3], controls(rng, 4), xgoal=[1.1, 1.05])
    far = Planner([1.0, 1.0, 0.3], controls(rng, 4), xgoal=[9.0, 9.0], cum=(1.25, -0.5))
    away = Planner([1e6, -3e5, 0.0], np.tile([[2.0, 0.0]], (4, 1)), xgoal=[0.0, 0.0])   # far from any map
    got = check(emu, [near, far, away], step=0, max_steps=5)
    assert got["status"].tolist() == [GOAL, 0, 0]
    last = Planner([1.0, 1.0, 0.3], controls(rng, 4), xgoal=[1.1, 1.05], cum=(3.0, 2.0))
    got = check(emu, [last, far, away], step=4, max_steps=5)
    assert got["status"].tolist() == [GOAL, MAX_STEPS, MAX_STEPS] and got["steps"].tolist() == [5, 5, 5]


def test_stopped_planners_are_left_alone(emu):
    rng = np.random.default_rng(5)
    o = [[1.0, 1.0, 5.0]]
    pls = [Planner([1.0, 1.0, 0.0], controls(rng, 5), xgoal=[50.0, 50.0], obs=o, contacts=3) for _ in range(2)]
    got = run(emu, pls, 0, 3, active=[0, 1])
    assert bits(got["u"][0]) == bits(pls[0].u) and not got["x0"][0].any()
    assert (got["xh"][0] == -7.0).all() and (got["uh"][0] == -7.0).all()
    assert bits(got["x"][0]) == bits(pls[0].x) and not got["cum_obj"][0] and got["steps"][0] == 0
    assert got["contacts"].tolist() == [3, 4] and got["count"] == 1


def test_map_trial_without_a_contact_buffer_is_unchanged(emu):
    """A map trial (lin set) whose descriptor also carries obstacles, with PlantArgs::contacts null: the map trial's
    step, lookup and stop rules (LEFT_MAP included), bit for bit."""
    rng = np.random.default_rng(6)
    g = grid(rng)
    pls = [MapPlanner(g, [rng.uniform(0, 3.7), rng.uniform(0, 2.9), rng.uniform(-3, 3)], controls(rng, 6),
                      xgoal=[50.0, 50.0]) for _ in range(12)]
    pls.append(MapPlanner(g, [3.7, 1.0, 0.0], np.tile([[3.0, 0.0]], (6, 1)), xgoal=[90.0, 1.0], pxlim=(-0.75, 3.71),
                          pylim=(-0.75, 3.75)))
    pls.append(MapPlanner(g, [1.0, 1.0, 0.3], controls(rng, 6), xgoal=[1.1, 1.05]))
    for p in pls:
        p.obs = np.array([[p.x[0], p.x[1], 2.0]], np.float32)
    got = run(emu, pls, 2, 8, contacts=False)
    for k, p in enumerate(pls):
        w = expect(p, 2, 8)
        assert bits(got["x"][k]) == bits(w["x"]) and bits(got["u"][k]) == bits(w["u"]), k
        assert bits(got["dist"][k]) == bits(np.float64(w["d"])) and got["status"][k] == w["status"], k
    assert got["status"][-2:].tolist() == [3, GOAL]
