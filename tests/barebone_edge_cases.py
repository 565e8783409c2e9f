"""Edge cases of the map-free ("barebone") planner's rollout and visualisation kernels (TEST INFRASTRUCTURE, importable
without a GPU).

``CASES``: the sweep.  Shapes N in {1, 31, 32, 33, 127, 128, 129, 1000} (128-thread blocks, a ragged last block, N
below the Python Config's clamp of 100) and T in {1, 2, 3, 100, 1024} (T = 1024: 8 KB of staged controls); obstacle
counts 0, 1, 2, 17, 256 and 4096 (N * T kept small for the large ones: the oracle adds the penalties one obstacle at a
time); overlapping obstacles (one step pays once per obstacle); an obstacle that contains x0 and one that contains the
goal; radius 0 on a visited point; the goal reached at step 1 inside an obstacle; a subnormal theta0; vrange with a
low end above 0, narrow wrange, and small and large u_std and lambda.  ``inputs(case)`` gives its noise, u_cur and
u_prev.

Directed cases, built with the arithmetic ``A`` of the kernel under test (its cos / sin decide the first step):

* ``obstacle_boundary_case(A, kind)``: one step to (x1, y1), an obstacle at (x1 - r, y1) (kind "up", or x1 + r for
  "up_ahead") with both subtractions exact, so ddx = +-r and ddy = 0, and q = f32(r*r).  The kernel decides inside /
  outside from diff = FFMA(-r, r, q) > 0:
    "up", "up_ahead"  f32(r*r) > r*r: the FFMA gives diff > 0 (outside); q - f32(r*r) rounded twice gives 0 (inside);
    "down"            f32(r*r) < r*r: the FFMA gives diff < 0 (inside); the split difference with >= says outside;
    "on_circle"       r*r exact: diff = 0 exactly, inside; >= says outside.
* ``goal_boundary_case(A, kind)``: the goal test d2 <= tol2 of that step:
    "on_tol"  d2 == tol2 exactly: reached; < says not reached;
    "split"   d2 = FFMA(dx, dx, dy*dy) and f32(dx*dx) + f32(dy*dy) on either side of tol2.
Each case records the decision of the exact rule and of the alternative it separates (``alt``).  ``directed_inputs``
turns a case into a one-step scenario whose cost shows the decision: an obstacle penalty, or the terminal cost d2.
"""
import numpy as np

F32, F64 = np.float32, np.float64
PI = float(np.pi)

SHAPE_N = (1, 31, 32, 33, 127, 128, 129, 1000)
SHAPE_T = (1, 2, 3, 100, 1024)
SHAPES = [(1, 1024), (31, 3), (32, 100), (33, 2), (127, 1), (128, 100), (129, 1024), (1000, 3), (1000, 100)]
OBSTACLE_COUNTS = (0, 1, 2, 17, 256, 4096)
THREE = [(1.0, 0.5, 0.6), (2.0, 1.2, 0.5), (0.6, 1.5, 0.4)]


def _base(name, N, T, **kw):
    c = dict(name=name, N=N, T=T, x0=(0.2, -0.1, 0.3), goal=(3.0, 2.0), tol=0.3, dt=0.1, lam=1.0, u_std=(1.0, 1.5),
             vrange=(0.0, 2.0), wrange=(-PI, PI), obs_cost=1e3, dist_weight=1.0, obstacles=THREE, seed=N * 7 + T,
             row0=None, w_zero=False)
    c.update(kw)
    c["obstacles"] = np.asarray(c["obstacles"], dtype=F32).reshape(-1, 3)
    return c


def _random_obstacles(k, seed, lo=-0.5, hi=2.5, rmax=0.6):
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(lo, hi, k), rng.uniform(lo, hi, k), rng.uniform(0.02, rmax, k)], 1)


def _first_x(x0, v, dt):
    """float32 x after one step from heading 0 with speed v: cos(0) = 1 on every provider, so x1 = f32(x0 + f32(v*dt))."""
    return F32(F64(F32(x0)) + F64(F32(F32(v) * F32(dt))))


def _cases():
    cs = [_base("shape-N%d-T%d" % (N, T), N, T) for N, T in SHAPES]
    for k in OBSTACLE_COUNTS:
        N, T = (129, 100) if k <= 17 else (33, 20) if k == 256 else (33, 3)
        rmax = 0.6 if k <= 17 else 0.25 if k == 256 else 0.08
        cs.append(_base("obstacles-%d" % k, N, T, obstacles=_random_obstacles(k, 40 + k, rmax=rmax) if k else []))
    ring = [(0.8 + 0.1 * np.cos(a), 0.3 + 0.1 * np.sin(a), 0.5 + 0.05 * i) for i, a in enumerate(np.linspace(0, 6, 6))]
    cs.append(_base("overlapping", 129, 40, obstacles=ring))
    cs.append(_base("x0-inside", 129, 30, obstacles=[(0.25, -0.05, 0.5)] + THREE))
    cs.append(_base("goal-inside", 129, 60, goal=(1.2, 0.8), tol=0.5, obstacles=[(1.25, 0.8, 0.4), (3.0, 3.0, 0.5)]))
    x1 = _first_x(0.5, 1.0, 0.1)
    cs.append(_base("radius-0", 40, 4, x0=(0.5, 0.25, 0.0), obstacles=[(x1, 0.25, 0.0), (2.0, 2.0, 0.3)],
                    row0=(1.0, 0.0)))
    g1 = _first_x(0.0, 1.5, 0.1)
    cs.append(_base("goal-step-1", 40, 8, x0=(0.0, 0.0, 0.0), goal=(g1, 0.0), tol=0.05, row0=(1.5, 0.0),
                    obstacles=[(g1, 0.0, 0.1)]))
    cs.append(_base("subnormal-theta0", 65, 12, x0=(0.1, 0.2, 1e-40), w_zero=True))
    cs.append(_base("values-a", 129, 50, vrange=(0.3, 1.7), wrange=(-0.5, 0.8), u_std=(0.4, 2.5), lam=0.05,
                    dist_weight=10.0, obs_cost=1e5))
    cs.append(_base("values-b", 129, 50, vrange=(0.5, 0.6), wrange=(-0.05, 0.05), u_std=(3.0, 0.2), lam=30.0,
                    dt=0.25, goal=(-2.0, 4.0), tol=1.0))
    return cs


CASES = _cases()


def inputs(case):
    """(noise (N, T, 2), u_cur (T, 2), u_prev (T, 2)) float32 of a case: noise N(0, u_std); controls that reach past
    vrange and wrange on both sides, so the clip of the noisy rows matters.  ``row0`` = (v, w): row 0's first control
    (u_cur[0] + noise[0, 0]) is exactly (v, w).  ``w_zero``: u_cur's angular controls and row 0's noise are 0."""
    rng = np.random.default_rng(case["seed"])
    N, T = case["N"], case["T"]
    us, vr, wr = np.asarray(case["u_std"]), case["vrange"], case["wrange"]
    noise = (rng.standard_normal((N, T, 2)) * us).astype(F32)

    def ctrl():
        v = rng.uniform(vr[0] - 0.3, vr[1] + 0.3, T)
        w = rng.uniform(wr[0] - 0.3, wr[1] + 0.3, T)
        return np.stack([v, w], 1).astype(F32)
    u_cur, u_prev = ctrl(), ctrl()
    if case["row0"] is not None:
        u_cur[0] = case["row0"]
        noise[0, 0] = 0.0
    if case["w_zero"]:
        u_cur[:, 1] = 0.0
        noise[0] = 0.0
    return noise, u_cur, u_prev


# ----------------------------------------------------------------------------- directed cases
def _step(A, x0, v, dt):
    dv = A.mul32(np.array([v], F32), F32(dt))
    th = np.array([x0[2]], F32)
    x1 = A.fma32(dv, A.cos32(th), np.array([x0[0]], F32))[0]
    y1 = A.fma32(dv, A.sin32(th), np.array([x0[1]], F32))[0]
    return F32(x1), F32(y1)


DIRECTED_X0 = (0.3, -0.2, 0.6)
DIRECTED_V = 1.25
DIRECTED_DT = 0.1


def obstacle_boundary_case(A, kind):
    assert kind in ("up", "up_ahead", "down", "on_circle")
    x1, y1 = _step(A, DIRECTED_X0, DIRECTED_V, DIRECTED_DT)
    if kind == "on_circle":
        rs = np.array([0.375], F32)
    else:
        rs = np.nextafter(F32(0.3), F32(1)) + np.arange(4096, dtype=F32) * np.spacing(F32(0.3))
        rs = rs.astype(F32)
    for r in rs:
        sq = F64(r) * F64(r)                                          # exact
        rn = F64(F32(sq))
        if (kind in ("up", "up_ahead") and not rn > sq) or (kind == "down" and not rn < sq):
            continue
        ox = F32(x1 + r) if kind == "up_ahead" else F32(x1 - r)
        ddx = F32(x1 - ox)
        if F64(ox) != F64(x1) + (F64(r) if kind == "up_ahead" else -F64(r)) or abs(ddx) != r:
            continue
        q = F32(F64(ddx) * F64(ddx))                                  # FFMA(ddx, ddx, 0 * 0)
        diff = F32(F64(q) - sq)                                       # FFMA(-r, r, q): one rounding
        split = F32(q - F32(r * r))
        exact_outside = bool(diff > 0)
        alt = dict(up="split", up_ahead="split", down="split_ge", on_circle="ge")[kind]
        alt_outside = bool(split > 0) if alt == "split" else bool(split >= 0) if alt == "split_ge" else bool(diff >= 0)
        return dict(kind=kind, obstacle=(float(ox), float(y1), float(r)), x1=(x1, y1), exact_outside=exact_outside,
                    alt=alt, alt_outside=alt_outside)
    raise AssertionError("no %s obstacle boundary case" % kind)


def goal_boundary_case(A, kind):
    assert kind in ("on_tol", "split")
    x1, y1 = _step(A, DIRECTED_X0, DIRECTED_V, DIRECTED_DT)
    if kind == "on_tol":
        tol = F32(0.375)
        gx = F32(x1 + tol)
        assert A.sub32(gx, x1) == tol
        d2 = F32(tol * tol)                                           # exact
        return dict(kind=kind, goal=(float(gx), float(y1)), tol=float(tol), exact_reached=True, alt="lt",
                    alt_reached=bool(d2 < F32(tol * tol)))
    gx = np.full(8192, F32(x1 + F32(0.2718)), F32)
    gy = (F32(y1 + F32(0.2)) + np.arange(8192, dtype=F32) * np.spacing(F32(0.2))).astype(F32)
    dx, dy = A.sub32(gx, np.full_like(gx, x1)), A.sub32(gy, np.full_like(gy, y1))
    e = A.fma32(dx, dx, A.mul32(dy, dy))
    s = A.add32(A.mul32(dx, dx), A.mul32(dy, dy))
    for i in np.nonzero(e != s)[0]:
        lo2, hi2 = min(e[i], s[i]), max(e[i], s[i])
        tol = F32(np.sqrt(F64(lo2)))
        for _ in range(8):                                            # tol2 = f32(tol * tol) in [lo2, hi2)
            tol2 = F32(tol * tol)
            if tol2 < lo2:
                tol = np.nextafter(tol, F32(np.inf))
            elif tol2 >= hi2:
                tol = np.nextafter(tol, F32(-np.inf))
            else:
                break
        tol2 = F32(tol * tol)
        if not lo2 <= tol2 < hi2:
            continue
        return dict(kind=kind, goal=(float(gx[i]), float(gy[i])), tol=float(tol), exact_reached=bool(e[i] <= tol2),
                    alt="split", alt_reached=bool(s[i] <= tol2))
    raise AssertionError("no split goal boundary case")


def directed_inputs(case, N=40):
    """A one-step scenario (a _base case with its inputs) for a directed case: noise 0, u = (v, 0), the case's obstacle
    (with obs_cost 1e4) or goal and tolerance, otherwise a far goal and no obstacle."""
    kw = dict(x0=DIRECTED_X0, dt=DIRECTED_DT, vrange=(0.0, 3.0), goal=(5.0, 5.0), tol=0.1, obs_cost=1e4, obstacles=[])
    if "obstacle" in case:
        kw["obstacles"] = [case["obstacle"]]
    else:
        kw.update(goal=case["goal"], tol=case["tol"])
    c = _base("directed-" + case["kind"], N, 1, **kw)
    noise = np.zeros((N, 1, 2), F32)
    u = np.array([[DIRECTED_V, 0.0]], F32)
    return c, noise, u, u.copy()


# ----------------------------------------------------------------------------- the oracle on a case
def oracle_costs(case, noise, u_cur, arith, return_states=False, obstacles=None):
    from oracle import mppi_ref as MR
    ob = case["obstacles"] if obstacles is None else np.asarray(obstacles, F32).reshape(-1, 3)
    return MR.rollout_costs_barebone(ob[:, :2], ob[:, 2], case["vrange"], case["wrange"], case["goal"], case["obs_cost"],
                                     case["tol"], case["lam"], case["u_std"], case["x0"], case["dt"], case["dist_weight"],
                                     noise, u_cur, return_states=return_states, arith=arith)


def oracle_states(case, V, noise, u_cur, u_prev, arith):
    from oracle import mppi_ref as MR
    return MR.state_rollouts_barebone(V, case["x0"], case["dt"], u_cur, u_prev, noise, case["vrange"], case["wrange"],
                                      arith=arith)


def vis_count(case):
    """The visualisation rollouts checked on a case: at most 33 (two 32-thread blocks), at most N."""
    return min(case["N"], 33)
