"""The windowed stochastic rollout (rollout_win_kernel, rollout_win_batch_kernel) and its fused noise kernel
(noise_prepare_kernel) against the exact oracle with the device provider, at the inputs where a kernel goes wrong
without the existing comparisons noticing: every work-share regime of the persistent grid, reached by shape on this
device's SM count (a ragged last warp, one CTA walking every map, shares that cross maps, a map split between CTAs,
a fractional pass count), both window heights, maps smaller than, equal to and just larger than the window with the
robot at the centre, the corners and in the padding, rollouts that random-walk across a cell corner about one ulp per
step (cell indices small, near +-2^20 and beyond 2^21), and batches of planners on different maps.  Every per-(n, m) cost
equals the oracle's in the windowed kernel's order (ctrl_order="presummed", wrap_clamp=True); the CVaR of the same
costs is checked against its high-precision reference.  tests/rollout_edge_cases.py holds the launch rules and the
tables; tests/test_rollout_edge_cases_cpu.py checks that the tables reach every regime."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import mppi_ref as MR           # noqa: E402
from oracle import xoroshiro as X           # noqa: E402
from tests import reduce_bounds as RB       # noqa: E402
from tests import rollout_edge_cases as EC  # noqa: E402
from tests.gpu_harness import RawPlanner, assert_all_equal, dev, eng, quiet, tdm_planner   # noqa: E402,F401
from tests.scenarios import make_scenario, oracle_rollout_costs   # noqa: E402

F32, F64 = np.float32, np.float64


@pytest.fixture(scope="module")
def sms(eng):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------- raw C-ABI driver and its oracle
def _run(eng, s):
    """Case s through the C-ABI planner: its maps, masks, risk, noise and u_cur set directly, one rollout (+ CVaR in
    mode 0).  Returns (costs (N, M), CVaR costs (N,) or None).  Mode 0 must take the windowed kernel: the rollout stage
    then issues 3 launches (controls from the outside noise, windowed rollout, CVaR) where the generic kernel, which
    the stage falls back to if the tensor maps cannot be encoded, issues 2."""
    N, T, R, C, mode = s["N"], s["T"], s["R"], s["C"], s["mode"]
    rp = RawPlanner(eng, mode, N, s["M"], T, R, C)
    try:
        pxl = np.array([s["xlo"], F64(s["xlo"]) + C * F64(s["res"])], F32)
        pyl = np.array([s["ylo"], F64(s["ylo"]) + R * F64(s["res"])], F32)
        dummy = np.zeros((2, R, C), np.int8)
        dummy[1] = 100
        rp.set_map("lin", dummy, [0.0, 1.0], s["lb"], s["res"], pxl, pyl, s["obs"], s["unk"], s["risk"] if mode == 2 else None)
        rp.set_map("ang", dummy, [0.0, 1.0], s["ab"], s["res"], pxl, pyl, s["obs"], s["unk"], None)
        rp.set_grids("lin", s["lin"])
        rp.set_grids("ang", s["ang"])
        rp.copy_in(eng._lib.BUF_NOISE, s["noise"])
        rp.copy_in(eng._lib.BUF_U_CUR, s["u_cur"])
        rp.set_params(x0=list(s["x0"]), xgoal=list(s["goal"]), goal_tolerance=s["tol"], vrange=list(s["vrange"]),
                      dt=float(s["dt"]), cvar_alpha=s.get("alpha", 1.0))
        before = _launches(rp)
        rp.call("rollout")
        if mode != 0:
            return rp.copy_out(eng._lib.BUF_COSTS, (N,))[:, None], None
        assert _launches(rp) - before == 3, "the rollout stage did not take the windowed kernel"
        return rp.copy_out(eng._lib.BUF_COSTS_NM, (N, rp.M)), rp.copy_out(eng._lib.BUF_COSTS, (N,))
    finally:
        rp.close()


def _launches(rp):
    n = ctypes.c_int64()
    rp.L.check(rp.lib.b200mppi_planner_launch_count(rp.pl, ctypes.byref(n)))
    return int(n.value)


def _oracle(s, arith, maps=None, return_states=False, ctrl_order=None):
    mode, R, C = s["mode"], s["R"], s["C"]
    lin, ang = (s["lin"], s["ang"]) if maps is None else (s["lin"][maps], s["ang"][maps])
    pxl = [s["xlo"], F64(s["xlo"]) + C * F64(s["res"])]
    pyl = [s["ylo"], F64(s["ylo"]) + R * F64(s["res"])]
    return MR.rollout_costs(mode, lin, ang, s["lb"], s["ab"], s["obs"], s["unk"], s["res"], pxl, pyl, s["vrange"],
                            [-np.pi, np.pi], s["goal"], 0.01, 1e5, 1e2, s["tol"], 1.0, [2, 3], s["x0"], s["dt"], 1.0,
                            s["noise"], s["u_cur"], risk_map=s["risk"][None], return_states=return_states, arith=arith,
                            ctrl_order=ctrl_order or ("presummed" if mode == 0 else "sequential"), wrap_clamp=True)


def _random_case(N, M, T, seed, cells=128, res=0.1, vr=(0.0, 3.0), alpha=0.5):
    """Mode 0 on a cells x cells map at res from the origin, robot near the centre, random maps, masks, noise, u_cur."""
    rng = np.random.default_rng(seed)
    c = cells * res / 2
    return dict(mode=0, N=N, M=M, T=T, R=cells, C=cells, res=F32(res), xlo=F32(0.0), ylo=F32(0.0), lb=[0.2, 1.3],
                ab=[0.15, 0.9], obs=(rng.random((cells, cells)) < 0.03).astype(np.int8),
                unk=(rng.random((cells, cells)) < 0.03).astype(np.int8), risk=np.zeros((cells, cells), np.int8),
                lin=rng.integers(0, 101, (M, cells, cells)).astype(np.int8),
                ang=rng.integers(0, 101, (M, cells, cells)).astype(np.int8),
                noise=(rng.standard_normal((N, T, 2)) * [2, 3]).astype(F32),
                u_cur=np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(F32),
                x0=[c + 0.37 * res, c - 0.21 * res, float(rng.uniform(-np.pi, np.pi))], goal=[c + 4.0, c - 3.0],
                tol=0.5, dt=F32(0.1), vrange=list(vr), alpha=alpha)


# ----------------------------------------------------------------------------- 1. every share regime, by shape
@pytest.mark.parametrize("N,M,T,grid,unit,what", EC.REGIME_CASES, ids=["N%d-M%d-T%d" % c[:3] for c in EC.REGIME_CASES])
def test_share_regimes(eng, dev, sms, N, M, T, grid, unit, what):
    r = EC.share_regime(N, M, sms)
    assert (r["grid"], r["unit"]) == (grid, unit), (
        "on %d SMs N %d, M %d gets grid %d, unit %d, not the %s case (grid %d, unit %d) of a 132-SM H100 SXM"
        % (sms, N, M, r["grid"], r["unit"], what, grid, unit))
    vr = (0.0, 0.3) if T > 100 else (0.0, 3.0)
    s = _random_case(N, M, T, seed=100 + N + M + T, vr=vr)
    got, cvar = _run(eng, s)
    maps = EC.oracle_maps(N, M, T, sms)
    assert_all_equal(got[:, maps], _oracle(s, dev, maps),
                     "%s (N %d, M %d, T %d, grid %d, unit %d)" % (what, N, M, T, grid, unit))
    RB.check_cvar(cvar, got, s["alpha"], label=what)


# ----------------------------------------------------------------------------- 2. small maps, edges and padding
def _map_scenario(rows, cols, res, spot, N=256, M=8, T=100, seed=0):
    sc = make_scenario("tdm", N=N, M=M, T=T, H=rows, W=cols, res=res, B=5, seed=31 + seed, warm_start=True)
    x, y = EC.map_spot(spot, rows, cols, res, EC.pad_cells(res))
    sc["params"]["x0"] = np.array([x, y, 0.7 - 0.4 * seed])
    return sc


def _staged(eng, sc):
    """staged_rollout with the robot placed as shift_and_update places it: setup() takes x0 only inside the map, a
    closed loop also moves it into the padding."""
    p = sc["params"]
    pl = tdm_planner(eng, sc, params=dict(p, x0=np.array([np.mean(sc["tdm_dict"]["xlimits"]),
                                                          np.mean(sc["tdm_dict"]["ylimits"]), 0.0])))
    pl.params["x0"] = p["x0"].copy()
    pl.move_mppi_task_vars_to_device()
    L = eng._lib
    pl.lin_tdm.sample_grids(1.0)
    pl.ang_tdm.sample_grids(1.0)
    L.check(L.lib.b200mppi_planner_sample_noise(pl._handle))
    L.check(L.lib.b200mppi_planner_rollout(pl._handle))
    return pl


def _check_staged(eng, dev, sc, what, maps=None):
    pl = _staged(eng, sc)
    lin, ang = pl.lin_tdm, pl.ang_tdm
    got = pl.costs_nm_d.copy_to_host()
    gl, ga = lin.sample_grid_batch_d.copy_to_host(), ang.sample_grid_batch_d.copy_to_host()
    if maps is not None:
        gl, ga, got_m = gl[maps], ga[maps], got[:, maps]
    else:
        got_m = got
    want = oracle_rollout_costs(sc, lin, ang, pl.noise_samples_d.copy_to_host(), pl.u_cur_d.copy_to_host(), grids=(gl, ga),
                                arith=dev, ctrl_order="presummed", wrap_clamp=True)
    assert_all_equal(got_m, want, what)
    RB.check_cvar(pl.costs_d.copy_to_host(), got, sc["params"]["cvar_alpha"], label=what)
    return pl


@pytest.mark.parametrize("rows,cols,res", EC.MAP_CASES, ids=["grid%dx%d" % EC.padded_grid(*c) for c in EC.MAP_CASES])
def test_map_sizes_edges_and_padding(eng, dev, rows, cols, res):
    """Per map size -- a padded grid smaller than the 240 x 232 window, equal to it, one row and column larger, and
    larger -- the robot at the centre, near each corner (the window's clamped, 16-aligned origin at each edge; past the
    window the last rows and columns go through the global path) and in the padding; T 100 at up to 3 m/s leaves the
    map from every spot but the centre of the large maps (wrap + clamp)."""
    R, C = EC.padded_grid(rows, cols, res)
    for k, spot in enumerate(EC.MAP_SPOTS):
        sc = _map_scenario(rows, cols, res, spot, seed=k)
        pl = _check_staged(eng, dev, sc, "%d x %d grid at %g m, %s" % (R, C, res, spot))
        assert pl.lin_tdm.sample_grid_batch_d.copy_to_host().shape[1:] == (R, C)


def test_noisy_dyn_shape(eng, dev, sms):
    """The reference benchmark's noisy_dyn shape: N 1024, M 1024, T 100 on 9 x 9 cells at 1 m (grid = SMs, unit 32:
    7.75 passes per CTA on 132 SMs); the oracle checks the maps where CTA shares begin and end."""
    sc = _map_scenario(9, 9, 1.0, "centre", N=1024, M=1024, T=100)
    r = EC.share_regime(1024, 1024, sms)
    assert r["unit"] == 32 and r["grid"] == sms
    _check_staged(eng, dev, sc, "noisy_dyn", maps=EC.share_edge_maps(1024, 1024, sms, limit=8))


# ----------------------------------------------------------------------------- 3. cell corners on the hardware
def _corner_walk(s, states, arith):
    """(fraction of lane-steps with x or y within 2 ulps of the corner's cell edge, x cells visited, y cells visited)
    from the oracle's states."""
    xs, ys = states[..., 1:, 0].ravel(), states[..., 1:, 1].ravel()
    near = ((np.abs(xs.astype(F64) - s["edge"][0]) <= 2 * s["ulp"][0]) |
            (np.abs(ys.astype(F64) - s["edge"][1]) <= 2 * s["ulp"][1]))
    xi = MR.floor_div_f32(arith.sub32(xs, s["xlo"]), s["res"], arith)
    yi = MR.floor_div_f32(arith.sub32(ys, s["ylo"]), s["res"], arith)
    return float(np.mean(near)), set(xi.tolist()), set(yi.tolist())


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("kind", EC.CORNER_KINDS)
def test_cell_corners(eng, dev, kind, mode):
    """Rollouts that random-walk across a four-cell corner about one float32 ulp per step, res 0.1, 0.05, 0.3, 1, 1/16
    and 0.7: the windowed kernel's magic-number interval decision (mode 0) and cell_index_exact of the generic kernels
    (modes 1, 2) on the real instructions.  The oracle's states show that most lane-steps lie within 2 ulps of an edge
    and that the rollouts cross both edges."""
    for k, res in enumerate(EC.CORNER_RES):
        s = EC.corner_case(res, kind, mode, seed=10 * k + mode)
        got, _ = _run(eng, s)
        want, states = _oracle(s, dev, return_states=True)
        near, xs, ys = _corner_walk(s, states, dev)
        assert near > 0.5, "res %g, %s: only %.2f of the lane-steps within 2 ulps of an edge" % (res, kind, near)
        assert {s["i"] - 1, s["i"]} <= xs and {s["j"] - 1, s["j"]} <= ys, (res, kind, xs, ys)
        if mode == 0:       # the generic kernel's control-cost order would give other costs
            assert (_oracle(s, dev, ctrl_order="sequential") != want).any()
        assert_all_equal(got, want, "corner %s, res %g, mode %d" % (kind, res, mode))


# ----------------------------------------------------------------------------- 4. the fused noise kernel
@pytest.mark.parametrize("T", EC.NOISE_T)
@pytest.mark.parametrize("N", EC.NOISE_N)
def test_fused_noise_kernel(eng, dev, N, T):
    """The noise a stochastic planner's noise stage draws (noise_prepare_kernel) equals the oracle's Box-Muller."""
    seed = 7 + N + T
    rp = RawPlanner(eng, 0, N, 2, T, 16, 16, seed=seed)
    try:
        rp.copy_in(eng._lib.BUF_U_CUR, np.zeros((T, 2), F32))
        rp.set_params(u_std=[1.5, 0.7])
        rp.call("sample_noise")
        got = rp.copy_out(eng._lib.BUF_NOISE, (N, T, 2))
    finally:
        rp.close()
    assert_all_equal(got, MR.sample_noise(X.create_states(N * T, seed), [1.5, 0.7], N, T, arith=dev),
                     "fused noise, N %d, T %d" % (N, T))


# ----------------------------------------------------------------------------- 5. the batched kernel
@pytest.mark.parametrize("N,M,T", EC.BATCH_CASES, ids=["N%d-M%d-T%d" % c for c in EC.BATCH_CASES])
def test_batched_kernel_against_oracle(eng, dev, sms, N, M, T):
    """One MPPI_StochasticBatch.solve() of 3 planners on 9 x 9 cells at 1 m, 64 x 64 at 0.2 m and 300 x 300 at 0.05 m
    (the last near a corner): each planner's per-(n, m) costs from its u_cur before the solve, the noise it drew and
    its maps as read after the solve.  N 200: CTA shares switch planner mid-share; at T 702 the batched launch runs
    the 224-row window where the single launch runs 232."""
    assert EC.mid_share_switches(N, M, sms, len(EC.BATCH_MAPS)), "no CTA switches planner on %d SMs" % sms
    scs = []
    for k, (n, res) in enumerate(EC.BATCH_MAPS):
        sc = make_scenario("tdm", N=N, M=M, T=T, H=n, W=n, res=res, B=5, seed=61 + k, warm_start=True)
        if k == 2:
            sc["params"]["x0"] = np.array([1.3 * res, n * res - 2.2 * res, 2.4])
        if T > 100:
            sc["params"]["vrange"] = np.array([0.0, 0.5])
        scs.append(sc)
    with quiet():
        pls = [tdm_planner(eng, sc) for sc in scs]
        u0 = [p.u_cur_d.copy_to_host() for p in pls]
        eng.MPPI_StochasticBatch(pls).solve()
    for k, (sc, p) in enumerate(zip(scs, pls)):
        lin, ang = p.lin_tdm, p.ang_tdm
        gl, ga = lin.sample_grid_batch_d.copy_to_host(), ang.sample_grid_batch_d.copy_to_host()
        want = oracle_rollout_costs(sc, lin, ang, p.noise_samples_d.copy_to_host(), u0[k], grids=(gl, ga), arith=dev,
                                    ctrl_order="presummed", wrap_clamp=True)
        got = p.costs_nm_d.copy_to_host()
        assert_all_equal(got, want, "batch T %d, planner %d" % (T, k))
        RB.check_cvar(p.costs_d.copy_to_host(), got, sc["params"]["cvar_alpha"], label="batch planner %d" % k)
