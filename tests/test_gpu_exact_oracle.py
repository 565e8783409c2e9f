"""Every per-rollout cost, state and noise value of the GPU kernels against the exact oracle (oracle/arith.py) with the
device provider -- the GPU's own sin.approx / cos.approx / sqrt.approx / div.approx / div.full and libdevice logf / cosf,
evaluated by b200mppi_debug_device_math -- and the .ftz flushes: equality of every element, no tolerance.  The windowed
kernel is compared in its control-cost order (pre-summed), the generic kernels in the reference's (sequential);
out-of-map cells follow the engine's wrap + clamp (DESIGN.md 2).  A mismatch reports its count and the first (n, m)
with both values."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import arith as AR              # noqa: E402
from oracle import mppi_ref as MR           # noqa: E402
from oracle import xoroshiro as X           # noqa: E402
from tests.scenarios import make_scenario, oracle_rollout_costs   # noqa: E402

F32 = np.float32


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    assert E.device_count() >= 1, "GPU tests need a CUDA device"
    return E


@pytest.fixture(scope="module")
def dev(eng):
    return AR.Exact(AR.DeviceProvider(eng._lib), ftz=True)


def assert_all_equal(got, want, what):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    print("\n[%s] %d mismatches of %d" % (what, len(bad), got.size))
    assert bad.size == 0, "%s: %d of %d differ; first: %s" % (
        what, len(bad), got.size, [(tuple(int(i) for i in ix), float(got[tuple(ix)]), float(want[tuple(ix)]))
                                   for ix in bad[:5]])


def test_device_math_entry_point(eng):
    """The provider itself: finite results, sqrt.approx of perfect squares exact, and errors (not faults) for an
    unknown op or n < 0."""
    L = eng._lib
    a = np.array([0.0, 1.0, 4.0, 9.0, 0.5, -2.0], F32)
    out = np.zeros_like(a)
    L.check(L.lib.b200mppi_debug_device_math(2, L.ptr(a), None, L.ptr(out), a.size))
    assert (out[:4] == [0, 1, 2, 3]).all()
    assert L.lib.b200mppi_debug_device_math(7, L.ptr(a), None, L.ptr(out), a.size) != 0
    assert L.lib.b200mppi_debug_device_math(-1, L.ptr(a), None, L.ptr(out), a.size) != 0
    assert L.lib.b200mppi_debug_device_math(0, L.ptr(a), None, L.ptr(out), -1) != 0
    assert L.lib.b200mppi_debug_device_math(3, L.ptr(a), None, L.ptr(out), a.size) != 0      # division without b
    assert L.lib.b200mppi_debug_device_math(0, None, None, None, 0) == 0


def _planner_rollout(eng, sc):
    cfg = eng.Config(**sc["cfg"])
    lin, ang = eng.TDM_Numba(cfg), eng.TDM_Numba(cfg)
    lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    pl = eng.MPPI_Numba(cfg)
    pl.setup(sc["params"], lin, ang)
    if "u0" in sc:
        pl.u_cur_d.copy_to_device(sc["u0"])
    pl.move_mppi_task_vars_to_device()
    L = eng._lib
    lin.sample_grids(1.0)
    ang.sample_grids(1.0)
    L.check(L.lib.b200mppi_planner_sample_noise(pl._handle))
    L.check(L.lib.b200mppi_planner_rollout(pl._handle))
    return pl, lin, ang


def test_generic_stochastic_kernel_without_window(eng, dev, monkeypatch):
    """B200MPPI_NO_WINDOW: the generic kernel on the res 0.05 row (rollouts leave the window region)."""
    monkeypatch.setenv("B200MPPI_NO_WINDOW", "1")
    sc = make_scenario("tdm", N=512, M=16, T=128, H=900, W=900, res=0.05, B=12, seed=4, warm_start=True)
    pl, lin, ang = _planner_rollout(eng, sc)
    want = oracle_rollout_costs(sc, lin, ang, pl.noise_samples_d.copy_to_host(), pl.u_cur_d.copy_to_host(), arith=dev,
                                wrap_clamp=True)
    assert_all_equal(pl.costs_nm_d.copy_to_host(), want, "generic kernel, no window")


@pytest.mark.parametrize("maskmax", [1, 3])
def test_windowed_kernel_both_mask_variants(eng, dev, maskmax):
    sc = make_scenario("tdm", N=512, M=16, T=128, H=900, W=900, res=0.05, B=12, seed=8, warm_start=True)
    if maskmax > 1:
        rng = np.random.default_rng(3)
        sc["obstacle"] = (sc["obstacle"].astype(np.int64) * rng.integers(1, maskmax + 1, sc["obstacle"].shape)).astype(np.int8)
    pl, lin, ang = _planner_rollout(eng, sc)
    want = oracle_rollout_costs(sc, lin, ang, pl.noise_samples_d.copy_to_host(), pl.u_cur_d.copy_to_host(), arith=dev,
                                ctrl_order="presummed", wrap_clamp=True)
    assert_all_equal(pl.costs_nm_d.copy_to_host(), want, "windowed kernel, mask max %d" % maskmax)


# ----------------------------------------------------------------------------- raw C-ABI cases: any bounds, any origin
def _raw_case(eng, dev, mode, N, M, T, cells, res, origin, lb, ab, x0, goal, seed, tol=0.5, vr=(0, 3)):
    from tests.test_gpu_parity import RawPlanner
    rng = np.random.default_rng(seed)
    rp = RawPlanner(eng, mode, N, M, T, cells, cells)
    try:
        lim = np.array([origin, origin + cells * res], F32)
        obs = (rng.random((cells, cells)) < 0.02).astype(np.int8)
        unk = (rng.random((cells, cells)) < 0.02).astype(np.int8)
        risk = rng.integers(0, 101, (cells, cells)).astype(np.int8)
        dummy = np.zeros((2, cells, cells), np.int8)
        dummy[1] = 100
        rp.set_map("lin", dummy, [0.0, 1.0], lb, res, lim, lim, obs, unk, risk if mode == 2 else None)
        rp.set_map("ang", dummy, [0.0, 1.0], ab, res, lim, lim, obs, unk, None)
        lin = rng.integers(0, 101, (rp.M, cells, cells)).astype(np.int8)
        ang = rng.integers(0, 101, (rp.M, cells, cells)).astype(np.int8)
        rp.set_grids("lin", lin)
        rp.set_grids("ang", ang)
        noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(F32)
        u = np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(F32)
        rp.copy_in(eng._lib.BUF_NOISE, noise)
        rp.copy_in(eng._lib.BUF_U_CUR, u)
        rp.set_params(x0=list(x0), xgoal=list(goal), goal_tolerance=tol, vrange=list(vr))
        rp.call("rollout")
        got = rp.copy_out(eng._lib.BUF_COSTS_NM, (N, M)) if mode == 0 else rp.copy_out(eng._lib.BUF_COSTS, (N,))[:, None]
    finally:
        rp.close()
    want = MR.rollout_costs(mode, lin, ang, lb, ab, obs, unk, F32(res), lim, lim, list(vr), [-np.pi, np.pi], goal, 0.01,
                            1e5, 1e2, tol, 1.0, [2, 3], x0, 0.1, 1.0, noise, u, risk_map=risk[None], arith=dev,
                            ctrl_order="presummed" if mode == 0 else "sequential", wrap_clamp=True)
    return got, want


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("lb,ab", [([0.2, 1.3], [0.15, 0.9]), ([-0.4, 1.0], [-0.5, 0.8])])
def test_nonzero_traction_lower_bounds(eng, dev, mode, lb, ab):
    got, want = _raw_case(eng, dev, mode, 1024, 8 if mode == 0 else 1, 48, 300, 0.1, 0.0, lb, ab, [15.03, 14.91, 0.4],
                          [18.0, 17.0], seed=21 + mode)
    assert_all_equal(got, want, "mode %d, bounds %s / %s" % (mode, lb, ab))


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("origin,res,cells,T,vr", [(4096.0, 0.01, 600, 256, (0.0025, 0.3)), (4.0e5, 0.1, 300, 64, (0, 3))])
def test_far_origins(eng, dev, mode, origin, res, cells, T, vr):
    """The far-origin geometries of the reach-box tests (4096 m at 1 cm, 4e5 m at 10 cm): every step rounds the float32
    state to a whole ulp."""
    c = origin + cells * res / 2
    got, want = _raw_case(eng, dev, mode, 512, 8 if mode == 0 else 1, T, cells, res, origin, [0.0, 1.0], [0.0, 1.0],
                          [c, c + 0.37 * res, 1.2], [c + 50.0, c + 50.0], seed=5, vr=vr)
    assert_all_equal(got, want, "origin %g, mode %d" % (origin, mode))


@pytest.mark.parametrize("mode", ["tdm", "det", "spd"])
def test_state_rollout_all_modes(eng, dev, mode):
    sc = make_scenario(mode, N=256, M=8, T=40, H=200, W=200, res=0.1, B=12, seed=6, warm_start=True)
    sc["cfg"]["num_vis_state_rollouts"] = 8
    cfg = eng.Config(**sc["cfg"])
    lin, ang = eng.TDM_Numba(cfg), eng.TDM_Numba(cfg)
    lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    pl = eng.MPPI_Numba(cfg)
    pl.setup(sc["params"], lin, ang)
    pl.u_cur_d.copy_to_device(sc["u0"])
    pl.solve()
    got = pl.get_state_rollout()
    m = dict(tdm=MR.MODE_STOCHASTIC, det=MR.MODE_DET_DYN, spd=MR.MODE_SPEED_MAP)[mode]
    want = MR.state_rollouts(m, got.shape[0], lin.sample_grid_batch_d.copy_to_host(), ang.sample_grid_batch_d.copy_to_host(),
                             [0.0, 1.0], [0.0, 1.0], np.float32(lin.res), lin.padded_xlimits.astype(F32),
                             lin.padded_ylimits.astype(F32), sc["params"]["x0"], 0.1, pl.u_cur_d.copy_to_host(),
                             pl.u_prev_d.copy_to_host(), pl.noise_samples_d.copy_to_host(), sc["params"]["vrange"],
                             sc["params"]["wrange"], arith=dev, wrap_clamp=True)
    assert_all_equal(got, want, "state rollout, %s" % mode)


def test_state_rollout_flushes_a_subnormal_heading(eng, dev):
    """theta0 = 1e-40 (subnormal) and zero angular commands: the device's cvt.ftz.f64.f32 flushes theta to 0 at the first
    step, which the ftz oracle predicts and the non-ftz one does not."""
    sc = make_scenario("det", N=128, M=1, T=16, H=100, W=100, res=0.1, B=12, seed=7)
    sc["params"]["x0"] = np.array([5.03, 4.97, 1e-40])
    cfg = eng.Config(**sc["cfg"])
    lin, ang = eng.TDM_Numba(cfg), eng.TDM_Numba(cfg)
    lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    pl = eng.MPPI_Numba(cfg)
    pl.setup(sc["params"], lin, ang)
    pl.solve()
    u = np.zeros((16, 2), F32)
    u[:, 0] = 1.0
    pl.u_cur_d.copy_to_device(u)
    got = pl.get_state_rollout()
    args = (MR.MODE_DET_DYN, got.shape[0], lin.sample_grid_batch_d.copy_to_host(), ang.sample_grid_batch_d.copy_to_host(),
            [0.0, 1.0], [0.0, 1.0], np.float32(lin.res), lin.padded_xlimits.astype(F32), lin.padded_ylimits.astype(F32),
            sc["params"]["x0"], 0.1, pl.u_cur_d.copy_to_host(), pl.u_prev_d.copy_to_host(),
            pl.noise_samples_d.copy_to_host(), sc["params"]["vrange"], sc["params"]["wrange"])
    want = MR.state_rollouts(*args, arith=dev, wrap_clamp=True)
    assert_all_equal(got, want, "state rollout, subnormal heading")
    assert got[0, 0, 2] == F32(1e-40) and (got[0, 1:, 2] == 0).all()
    no_ftz = MR.state_rollouts(*args, arith=AR.Exact(AR.DeviceProvider(eng._lib), ftz=False), wrap_clamp=True)
    assert (no_ftz[0, 1:, 2] == F32(1e-40)).all()


def test_barebone_kernel(eng, dev):
    from mppi_numba_b200 import barebone as BB
    cfg = BB.Config(T=6.4, dt=0.1, num_control_rollouts=4096, num_vis_state_rollouts=4, seed=3)
    pl = BB.MPPI_Numba(cfg)
    p = dict(dt=0.1, x0=np.array([0.3, 0.2, 0.4]), xgoal=np.array([5.0, 4.0]), goal_tolerance=0.3, lambda_weight=1.0,
             num_opt=1, u_std=np.array([2.0, 3.0]), vrange=np.array([0.0, 3.0]), wrange=np.array([-np.pi, np.pi]),
             obs_penalty=1e3, dist_weight=1.0, obstacle_positions=np.array([[2.0, 2.0], [3.5, 2.5], [1.0, 2.8]]),
             obstacle_radius=np.array([0.6, 0.4, 0.5]))
    pl.setup(p)
    rng = np.random.default_rng(2)
    u0 = np.stack([rng.uniform(0, 2, cfg.num_steps), rng.uniform(-1, 1, cfg.num_steps)], 1).astype(F32)
    pl.u_cur_d.copy_to_device(u0)
    pl.solve()
    want = MR.rollout_costs_barebone(p["obstacle_positions"], p["obstacle_radius"], p["vrange"], p["wrange"], p["xgoal"],
                                     p["obs_penalty"], p["goal_tolerance"], 1.0, p["u_std"], p["x0"], 0.1, 1.0,
                                     pl.noise_samples_d.copy_to_host(), u0, arith=dev)
    assert_all_equal(pl.costs_d.copy_to_host(), want, "barebone kernel")


def test_config5_full_launch_on_a_subset_of_maps(eng, dev):
    """Config 5 (N 8192, M 256, T 128, 1024 x 1024 cells at 0.1 m): the kernel runs whole, the oracle checks 8 maps x all
    8192 control sequences."""
    sc = make_scenario("tdm", N=8192, M=256, T=128, H=1024, W=1024, res=0.1, B=12, seed=1, warm_start=True)
    pl, lin, ang = _planner_rollout(eng, sc)
    got = pl.costs_nm_d.copy_to_host()
    maps = np.array([0, 1, 37, 100, 128, 199, 254, 255])
    gl, ga = lin.sample_grid_batch_d.copy_to_host()[maps], ang.sample_grid_batch_d.copy_to_host()[maps]
    want = oracle_rollout_costs(sc, lin, ang, pl.noise_samples_d.copy_to_host(), pl.u_cur_d.copy_to_host(), grids=(gl, ga),
                                arith=dev, ctrl_order="presummed", wrap_clamp=True)
    assert_all_equal(got[:, maps], want, "config 5, 8 maps")


def test_config5_noise_draw_equals_oracle(eng, dev):
    """A whole config-5 noise draw (8192 x 128 x 2): every element equals the oracle's Box-Muller with the device's
    logf / cosf / sqrt.approx."""
    from tests.test_gpu_parity import RawPlanner
    N, T = 8192, 128
    rp = RawPlanner(eng, 1, N, 1, T, 8, 8, seed=5)
    try:
        rp.set_params(u_std=[2.0, 3.0])
        rp.call("sample_noise")
        got = rp.copy_out(eng._lib.BUF_NOISE, (N, T, 2))
    finally:
        rp.close()
    want = MR.sample_noise(X.create_states(N * T, 5), [2.0, 3.0], N, T, arith=dev)
    assert_all_equal(got, want, "config 5 noise")


def run_directed(eng, s, mode):
    """A directed case (tests/directed_cases.py) through the C-ABI planner: uniform grids set directly, its bounds."""
    from tests.test_gpu_parity import RawPlanner
    N, T, R, Cc = s["N"], s["T"], s["R"], s["Cc"]
    rp = RawPlanner(eng, mode, N, s["M"], T, R, Cc)
    try:
        lim = np.array([s["xlo"], s["xlo"] + Cc * s["res"]], F32)
        dummy = np.zeros((2, R, Cc), np.int8)
        dummy[1] = 100
        rp.set_map("lin", dummy, [0.0, 1.0], s["lb"], s["res"], lim, lim, s["obs"], s["unk"], s["risk"] if mode == 2 else None)
        rp.set_map("ang", dummy, [0.0, 1.0], s["ab"], s["res"], lim, lim, s["obs"], s["unk"], None)
        rp.set_grids("lin", s["lin"][:rp.M])
        rp.set_grids("ang", s["ang"][:rp.M])
        rp.copy_in(eng._lib.BUF_NOISE, s["noise"])
        rp.copy_in(eng._lib.BUF_U_CUR, s["u_cur"])
        rp.set_params(x0=list(s["x0"]), xgoal=list(s["goal"]), goal_tolerance=s["tol"])
        rp.call("rollout")
        return rp.copy_out(eng._lib.BUF_COSTS_NM, (N, rp.M)) if mode == 0 else rp.copy_out(eng._lib.BUF_COSTS, (N,))[:, None]
    finally:
        rp.close()


def directed_oracle(s, mode, arith):
    lim = [s["xlo"], s["xlo"] + s["Cc"] * s["res"]]
    return MR.rollout_costs(mode, s["lin"] if mode == 0 else s["lin"][:1], s["ang"] if mode == 0 else s["ang"][:1],
                            s["lb"], s["ab"], s["obs"], s["unk"], s["res"], lim, lim, [0, 3], [-np.pi, np.pi], s["goal"],
                            0.01, 1e5, 1e2, s["tol"], 1.0, [2, 3], s["x0"], 0.1, 1.0, s["noise"], s["u_cur"],
                            risk_map=s["risk"][None], arith=arith, ctrl_order="presummed" if mode == 0 else "sequential",
                            wrap_clamp=True)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("kind", ["state", "traction"])
def test_float64_contractions_on_a_float32_rounding_boundary(eng, dev, kind, mode):
    """Inputs built (with this GPU's cos.approx) so that rounding the traction product or the state product before the
    add moves the first step's float32 x by one ulp and flips the goal flag: every kernel equals the exact oracle, which
    fuses both, so a kernel that split either contraction would differ."""
    from tests.directed_cases import directed_scenario, fma_boundary_case
    case = fma_boundary_case(dev, kind)
    assert case["x1_exact"] != case["x1_other"]
    s = directed_scenario(case, N=40)
    assert_all_equal(run_directed(eng, s, mode), directed_oracle(s, mode, dev), "%s boundary, mode %d" % (kind, mode))
