"""What the GPU tests (run with ``-m gpu``) share: the engine and exact-oracle fixtures, the planner builders, the
snapshot of everything a solve writes and its bit-for-bit comparison, and the drivers that hold a batch or a trial
against the same work done one planner at a time on identical twins.  A test module takes the fixtures with
``from tests.gpu_harness import eng, dev  # noqa: F401``; module scope gives each module its own instance.
Importing this module neither builds nor loads the library: the ``eng`` fixture does."""
import contextlib
import ctypes as C
import io

import numpy as np
import pytest


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    assert E.device_count() >= 1, "GPU tests need a CUDA device"
    return E


@pytest.fixture(scope="module")
def dev(eng):
    """The exact oracle's arithmetic with this GPU's approximate operations and .ftz flushes."""
    from oracle import arith as AR
    return AR.Exact(AR.DeviceProvider(eng._lib), ftz=True)


def quiet():
    return contextlib.redirect_stdout(io.StringIO())


# ----------------------------------------------------------------------------- planners
def tdm_pair(E, cfg, pmf_lin, pmf_ang, tdm_dict, obstacle=None, unknown=None, **kw):
    """(lin, ang): two TDMs set from their PMF grids and the shared masks; ``kw`` (rank, world_size) goes to
    TDM_Numba."""
    lin, ang = E.TDM_Numba(cfg, **kw), E.TDM_Numba(cfg, **kw)
    lin.set_TDM_from_PMF_grid(pmf_lin, tdm_dict, obstacle, unknown)
    ang.set_TDM_from_PMF_grid(pmf_ang, tdm_dict, obstacle, unknown)
    return lin, ang


def tdm_planner(E, sc, params=None, box=None, monkeypatch=None, diverged=False, **kw):
    """The set-up MPPI_Numba of a scenario (the keys of tests/scenarios.make_scenario), warm-started from sc["u0"] when
    the scenario has one; its TDMs are pl.lin_tdm and pl.ang_tdm.  ``params`` replaces sc["params"]; ``box`` sets
    B200MPPI_SAMPLE_BOX through ``monkeypatch``, which the planner handle reads when it is created; ``diverged``: one
    public lin.sample_grids() first, so the pair's streams differ and each TDM is sampled on its own; ``kw`` (rank,
    world_size) goes to TDM_Numba and MPPI_Numba."""
    if box is not None:
        monkeypatch.setenv("B200MPPI_SAMPLE_BOX", box)
    cfg = E.Config(**sc["cfg"])
    lin, ang = tdm_pair(E, cfg, sc["pmf_lin"], sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"], **kw)
    if diverged:
        lin.sample_grids()
    pl = E.MPPI_Numba(cfg, **kw)
    pl.setup(sc["params"] if params is None else params, lin, ang)
    if "u0" in sc:
        pl.u_cur_d.copy_to_device(sc["u0"])
    return pl


def tdm_scenario(k, N=200, M=24, T=20, H=64, res=0.2, num_opt=1, edge=False, masks03=False):
    """Stochastic (use_tdm) scenario k of the batch and trial tests, with its own seed, CVaR alpha, penalties and dt."""
    from tests.scenarios import make_scenario
    sc = make_scenario("tdm", N=N, M=M, T=T, H=H, W=H, res=res, B=5, seed=23 + 5 * k, warm_start=(k % 2 == 1),
                       cvar_alpha=[0.5, 0.25, 1.0, 0.1][k % 4])
    p = sc["params"]
    p["num_opt"] = num_opt
    p["obs_penalty"], p["unknown_penalty"] = 1e3 + 10 * k, 50.0 + k
    p["dt"] = [0.1, 0.08, 0.12][k % 3]
    if edge:                                             # the reach box would leave the map: whole maps
        p["x0"] = np.array([0.15, 0.3, 0.4])
    if masks03:                                          # mask values 0..3: the general penalty variant
        rng = np.random.default_rng(90 + k)
        sc["obstacle"] = (rng.integers(0, 4, sc["obstacle"].shape) * (rng.random(sc["obstacle"].shape) < 0.05)).astype(np.int8)
    return sc


def tdm_trial_setup(E, k, num_opt=1, **shape):
    """Stochastic trial planner k and its ground-truth grid.  k = 0, 1: goal within a step, and a nearby goal; k = 2:
    goal out of reach (runs to max_steps); k = 3: start near the map's corner (every box leaves the map: whole maps);
    k = 4: an int8 grid (TractionGrid's use_int8 stores 100 x traction) that throws the robot off the padded map."""
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
    pl = tdm_planner(E, vary(sc, k))
    rng = np.random.default_rng(300 + k)
    grid = E.TractionGrid(rng.uniform(0.2, 1.0, (n, n)), rng.uniform(0.2, 1.0, (n, n)), res=res, use_int8=(k == 4))
    return pl, grid


def vary(sc, k):
    """Scenario sc with planner k's own lambda and u_std."""
    p = dict(sc["params"])
    p["lambda_weight"] = [1.0, 0.5, 2.0, 0.8, 1.3][k % 5]
    p["u_std"] = np.array([2.0, 3.0]) * (1.0 + 0.1 * (k % 7))
    return dict(sc, params=p)


def staged_rollout(E, sc):
    """The planner of scenario sc after the stages of one solve up to the rollout, through the C entry points: both
    TDMs sampled whole (alpha 1), the noise drawn, the rollout run."""
    pl = tdm_planner(E, sc)
    pl.move_mppi_task_vars_to_device()
    L = E._lib
    pl.lin_tdm.sample_grids(1.0)
    pl.ang_tdm.sample_grids(1.0)
    L.check(L.lib.b200mppi_planner_sample_noise(pl._handle))
    L.check(L.lib.b200mppi_planner_rollout(pl._handle))
    return pl


class RawPlanner:
    """Drives libb200mppi.so directly (no Python API objects): what a foreign-language binding would do."""

    def __init__(self, E, mode, N, M, T, Rmax, Cmax, seed=1, thread_dim=(4, 4), V=1, rank=0, world=1):
        L = E._lib
        self.L, self.lib = L, L.lib
        self.pod = L.ConfigPOD(num_steps=T, num_control_rollouts=N, num_grid_samples=M, max_map_rows=Rmax,
                               max_map_cols=Cmax, tdm_thread_x=thread_dim[0], tdm_thread_y=thread_dim[1],
                               num_vis_state_rollouts=V, mode=mode, device=0, rank=rank, world_size=world, seed=seed)
        self.lin, self.ang, self.pl = C.c_void_p(), C.c_void_p(), C.c_void_p()
        L.check(self.lib.b200mppi_tdm_create(C.byref(self.pod), C.byref(self.lin)))
        L.check(self.lib.b200mppi_tdm_create(C.byref(self.pod), C.byref(self.ang)))
        L.check(self.lib.b200mppi_planner_create(C.byref(self.pod), C.byref(self.pl)))
        self.N, self.M, self.T, self.Rmax, self.Cmax = N, (M if mode == 0 else 1), T, Rmax, Cmax
        self.n_local = N * (rank + 1) // world - N * rank // world

    def close(self):
        self.lib.b200mppi_planner_destroy(self.pl)
        self.lib.b200mppi_tdm_destroy(self.lin)
        self.lib.b200mppi_tdm_destroy(self.ang)

    def set_map(self, which, pmf_padded, bin_values, bounds, res, pxl, pyl, obs=None, unk=None, risk=None):
        L, t = self.L, (self.lin if which == "lin" else self.ang)
        pmf = np.ascontiguousarray(pmf_padded, dtype=np.int8)
        bv = np.ascontiguousarray(bin_values, dtype=np.float32)
        bb = np.ascontiguousarray(bounds, dtype=np.float32)
        xl = np.ascontiguousarray(pxl, dtype=np.float32)
        yl = np.ascontiguousarray(pyl, dtype=np.float32)
        L.check(self.lib.b200mppi_tdm_set_pmf(t, L.ptr(pmf), pmf.shape[0], pmf.shape[1], pmf.shape[2], L.ptr(bv),
                                              L.ptr(bb), np.float32(res), L.ptr(xl), L.ptr(yl)))
        if obs is not None:
            o = np.ascontiguousarray(obs, dtype=np.int8)
            u = np.ascontiguousarray(unk, dtype=np.int8)
            L.check(self.lib.b200mppi_tdm_set_masks(t, L.ptr(o), L.ptr(u), o.shape[0], o.shape[1]))
        if risk is not None:
            r = np.ascontiguousarray(risk, dtype=np.int8)
            L.check(self.lib.b200mppi_tdm_set_risk_map(t, L.ptr(r), r.shape[0], r.shape[1]))

    def set_grids(self, which, g):
        g = np.ascontiguousarray(g, dtype=np.int8)
        self.L.check(self.lib.b200mppi_tdm_set_sample_grids(self.lin if which == "lin" else self.ang,
                                                            self.L.ptr(g), g.nbytes))

    def get_grids(self, which):
        maps = self.M
        out = np.empty((maps, self.Rmax, self.Cmax), dtype=np.int8)
        self.L.check(self.lib.b200mppi_tdm_get_sample_grids(self.lin if which == "lin" else self.ang,
                                                            self.L.ptr(out), out.nbytes))
        return out

    def set_params(self, **kw):
        L = self.L
        p = L.ParamsPOD()
        d = dict(dt=0.1, x0=[0, 0, 0], xgoal=[0, 0], goal_tolerance=0.5, v_post_rollout=0.01, cvar_alpha=1.0,
                 lambda_weight=1.0, u_std=[2, 3], vrange=[0, 3], wrange=[-np.pi, np.pi], obs_penalty=1e5,
                 unknown_penalty=1e2, dist_weight=1.0, num_opt=1, alpha_dyn=1.0)
        d.update(kw)
        for k, v in d.items():
            if k in ("x0", "xgoal", "u_std", "vrange", "wrange"):
                setattr(p, k, L.c_floats(np.asarray(v, dtype=np.float32), len(v)))
            else:
                setattr(p, k, v)
        L.check(self.lib.b200mppi_planner_set_tdms(self.pl, self.lin, self.ang))
        L.check(self.lib.b200mppi_planner_set_params(self.pl, C.byref(p)))

    def copy_in(self, buf, arr):
        arr = np.ascontiguousarray(arr)
        self.L.check(self.lib.b200mppi_planner_copy_in(self.pl, buf, self.L.ptr(arr), arr.nbytes))

    def copy_out(self, buf, shape, dtype=np.float32):
        out = np.empty(shape, dtype=dtype)
        self.L.check(self.lib.b200mppi_planner_copy_out(self.pl, buf, self.L.ptr(out), out.nbytes))
        return out

    def call(self, name, *args):
        self.L.check(getattr(self.lib, "b200mppi_planner_" + name)(self.pl, *args))


def run_directed(eng, s, mode, states=False):
    """A directed case (tests/directed_cases.py) through the C-ABI planner: uniform grids set directly, its bounds.
    ``states``: the planner's visualisation rollout instead (V = 1: u_cur without noise, on map 0), (1, T + 1, 3)."""
    N, T, R, Cc = s["N"], s["T"], s["R"], s["Cc"]
    rp = RawPlanner(eng, mode, N, s["M"], T, R, Cc)
    try:
        lim = np.array([s["xlo"], s["xlo"] + Cc * s["res"]], np.float32)
        dummy = np.zeros((2, R, Cc), np.int8)
        dummy[1] = 100
        rp.set_map("lin", dummy, [0.0, 1.0], s["lb"], s["res"], lim, lim, s["obs"], s["unk"], s["risk"] if mode == 2 else None)
        rp.set_map("ang", dummy, [0.0, 1.0], s["ab"], s["res"], lim, lim, s["obs"], s["unk"], None)
        rp.set_grids("lin", s["lin"][:rp.M])
        rp.set_grids("ang", s["ang"][:rp.M])
        rp.copy_in(eng._lib.BUF_NOISE, s["noise"])
        rp.copy_in(eng._lib.BUF_U_CUR, s["u_cur"])
        rp.set_params(x0=list(s["x0"]), xgoal=list(s["goal"]), goal_tolerance=s["tol"], dt=s["dt"])
        if states:
            out = np.empty((1, T + 1, 3), np.float32)
            rp.call("get_state_rollout", eng._lib.ptr(out), out.nbytes)
            return out
        rp.call("rollout")
        return rp.copy_out(eng._lib.BUF_COSTS_NM, (N, rp.M)) if mode == 0 else rp.copy_out(eng._lib.BUF_COSTS, (N,))[:, None]
    finally:
        rp.close()


def directed_oracle(s, mode, arith):
    from oracle import mppi_ref as MR
    lim = [s["xlo"], s["xlo"] + s["Cc"] * s["res"]]
    return MR.rollout_costs(mode, s["lin"] if mode == 0 else s["lin"][:1], s["ang"] if mode == 0 else s["ang"][:1],
                            s["lb"], s["ab"], s["obs"], s["unk"], s["res"], lim, lim, [0, 3], [-np.pi, np.pi], s["goal"],
                            0.01, 1e5, 1e2, s["tol"], 1.0, [2, 3], s["x0"], s["dt"], 1.0, s["noise"], s["u_cur"],
                            risk_map=s["risk"][None], arith=arith, ctrl_order="presummed" if mode == 0 else "sequential",
                            wrap_clamp=True)


# ----------------------------------------------------------------------------- comparisons
def planner_launches(p):
    """Kernel launches issued through planner p's own handle (a batch counts the launches it issues itself)."""
    from mppi_numba_b200 import _lib as L
    n = C.c_int64()
    L.check(L.lib.b200mppi_planner_launch_count(p._handle, C.byref(n)))
    return int(n.value)


def snapshot(p):
    """Everything a solve() writes: controls, noise, costs, weights, RNG states and, for planners with maps, both TDMs'
    RNG states and sampled maps (reading them completes a boxed sampling).  Stochastic planners add sample_box() and
    the per-(m, n) costs -- those only once a rollout ran: with num_opt = 0 no solve writes them and the buffer holds
    whatever its allocation held."""
    stochastic = getattr(p, "use_tdm", False)
    d = dict(u_cur=p.u_cur_d.copy_to_host(), u_prev=p.u_prev_d.copy_to_host(), noise=p.noise_samples_d.copy_to_host(),
             costs=p.costs_d.copy_to_host())
    if stochastic and int(p.params["num_opt"]) >= 1:
        d["costs_nm"] = p.costs_nm_d.copy_to_host()
    d.update(weights=p.weights_d.copy_to_host(), rng=p.rng_states_d.copy_to_host())
    if stochastic:
        d["box"] = np.asarray(p.sample_box())
    if getattr(p, "lin_tdm", None) is not None:
        for name, t in (("lin", p.lin_tdm), ("ang", p.ang_tdm)):
            d[name + "_rng"] = t.rng_states_d.copy_to_host()
            d[name + "_map"] = t.sample_grid_batch_d.copy_to_host()
    return d


def assert_same(a, b, what):
    """Bit for bit: the same keys and, per key, the same dtype, shape and bytes.  So -0.0 differs from +0.0, and an
    untouched buffer's NaN patterns (whatever its allocation held), which == never equates, compare equal."""
    assert a.keys() == b.keys(), (what, list(a), list(b))
    for key in a:
        x, y = np.asarray(a[key]), np.asarray(b[key])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), "%s: %s differs" % (what, key)


def assert_all_equal(got, want, what):
    """Every element of got equals want's as float32 bits; a mismatch reports its count and the first indices."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    print("\n[%s] %d mismatches of %d" % (what, len(bad), got.size))
    assert bad.size == 0, "%s: %d of %d differ; first: %s" % (
        what, len(bad), got.size, [(tuple(int(i) for i in ix), float(got[tuple(ix)]), float(want[tuple(ix)]))
                                   for ix in bad[:5]])


def ulps(a, b):
    """Distance in float64 ulps, element by element."""
    ia, ib = a.view(np.int64), b.view(np.int64)
    ia = np.where(ia < 0, np.int64(-2 ** 63) - ia, ia)
    ib = np.where(ib < 0, np.int64(-2 ** 63) - ib, ib)
    return np.abs(ia - ib)


# ----------------------------------------------------------------------------- batches and trials against twins
def batch_vs_sequential(batch_cls, make, K, rounds=3, check_every=True):
    """Twins built by make(k): a batch_cls (MPPI_Batch or MPPI_StochasticBatch) solve on one set against K solve()
    calls on the other, over `rounds` closed-loop rounds; u every round, every snapshot every round (or only the last
    round's without check_every).  Returns (A, B, batch)."""
    with quiet():
        A = [make(k) for k in range(K)]
        B = [make(k) for k in range(K)]
        batch = batch_cls(A)
        for r in range(rounds):
            ub = batch.solve()
            us = np.stack([p.solve() for p in B])
            assert ub.dtype == np.float32
            assert_same(dict(u=ub), dict(u=us), "round %d" % r)
            for k in range(K):                           # the Python layer leaves u_prev_d as solve() does
                assert (A[k].u_prev_d is A[k]._u_prev_buf) == (B[k].u_prev_d is B[k]._u_prev_buf)
            if check_every or r == rounds - 1:
                for k in range(K):
                    assert_same(snapshot(A[k]), snapshot(B[k]), "round %d planner %d" % (r, k))
            for k in range(K):
                x0 = np.asarray(A[k].params["x0"], dtype=np.float64) + np.array([0.03 * (k + 1), -0.02 * r, 0.05])
                A[k].shift_and_update(x0.copy(), ub[k], 1)
                B[k].shift_and_update(x0.copy(), us[k], 1)
    return A, B, batch


def expected_batch_launches(B, rounds, num_opt):
    """A stochastic batch's launches: 1 noise + 1 rollout + 1 CVaR + 1 update per iteration, plus every planner's own
    sampler launches (its solve() issues those same sampler launches next to its 4 per iteration)."""
    per_iter = 4 * num_opt * rounds
    return per_iter + sum(planner_launches(p) - per_iter for p in B)


def twins(setup, K, **kw):
    """(A, B, grids): K planners and their ground-truth grids from setup(k, **kw), twice."""
    with quiet():
        A = [setup(k, **kw) for k in range(K)]
        B = [setup(k, **kw) for k in range(K)]
    return [a[0] for a in A], [b[0] for b in B], [a[1] for a in A]


def solve_in_batch_of_one(p):
    """u of one stochastic planner's solve through MPPI_StochasticBatch, the solve its device trial repeats."""
    from mppi_numba_b200 import MPPI_StochasticBatch
    return MPPI_StochasticBatch([p]).solve()[0]


def replay(A, B, out, solve_one, check_next=True):
    """The host loop fed with the device trials' trajectory `out` (of the planners A) on the twins B, u = solve_one(p)
    per step: u[0] of every step bit for bit, the histories NaN after each planner's last step and only there, then
    every buffer of the planner (snapshot) and params['x0'] (float64) bit for bit; with check_next, one more solve() on
    both sets."""
    for k, p in enumerate(B):
        n = int(out["steps"][k])
        with quiet():
            for t in range(n):
                useq = solve_one(p)
                assert_same({"u[0]": useq[0]}, {"u[0]": out["uhist"][k, t]}, "planner %d step %d" % (k, t))
                p.shift_and_update(out["xhist"][k, t + 1], useq, 1)
        assert np.isnan(out["xhist"][k, n + 1:]).all() and np.isnan(out["uhist"][k, n:]).all()
        assert not np.isnan(out["xhist"][k, :n + 1]).any()
        assert_same(snapshot(A[k]), snapshot(p), "planner %d" % k)
        assert A[k].params["x0"].dtype == np.float64
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=p.params["x0"]), "planner %d" % k)
    if not check_next:
        return
    with quiet():
        for k in range(len(A)):
            ua, ub = A[k].solve(), B[k].solve()
            if out["status"][k] == "left_map":
                assert ua is None and ub is None
            else:
                assert_same(dict(u=ua), dict(u=ub), "planner %d: the next solve" % k)
                assert_same(snapshot(A[k]), snapshot(B[k]), "planner %d after one more solve" % k)
