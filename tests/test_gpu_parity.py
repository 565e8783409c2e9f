"""GPU parity tests proper (run with ``-m gpu`` on an H100): the CUDA engine, called through the
C-ABI / the drop-in Python API, against (1) the committed golden vectors produced by the reference's
own kernels and (2) the oracle on identical seeded inputs, plus size-independent properties.

Against the reference's goldens: per-rollout costs and u_seq within 1e-4 relative fp32 on the same inputs (the
goldens come from the simulator, whose sin / cos / sqrt are exact math); integer work (RNG streams, sampled maps, PMF
preprocessing) bit-exact.  Against the oracle on the engine's own inputs: the exact oracle (oracle/arith.py) with the
device provider -- the GPU's own approximate operations -- predicts every per-(n, m) cost and noise value, so those
comparisons are equalities (tests/test_gpu_exact_oracle.py has more).
"""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import mppi_ref as MR          # noqa: E402
from oracle import terrain_ref as TR       # noqa: E402
from oracle import xoroshiro as X          # noqa: E402
from tests import reduce_bounds as RB      # noqa: E402
from tests.gpu_harness import (RawPlanner, assert_all_equal, assert_same, dev, eng,  # noqa: E402,F401
                               staged_rollout, tdm_pair, tdm_planner)
from tests.scenarios import make_scenario, oracle_rollout_costs   # noqa: E402


def load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name), allow_pickle=False)


def rel_err(a, b):
    return np.abs(a - b) / np.maximum(np.abs(b), 1e-6)


# ----------------------------------------------------------------------------- 1. noise
def test_noise_vs_reference_golden(eng, golden_dir):
    g = load(golden_dir, "ref_noise.npz")
    N, T = int(g["N"]), int(g["T"])
    rp = RawPlanner(eng, 1, N, 1, T, 8, 8, seed=int(g["seed"]))
    try:
        st0 = rp.copy_out(eng._lib.BUF_RNG, (N * T, 2), np.uint64)
        assert (st0 == g["states0"]).all()                       # host jump chain == numba's
        rp.set_params(u_std=list(g["u_std"]))
        rp.call("sample_noise")
        n1 = rp.copy_out(eng._lib.BUF_NOISE, (N, T, 2))
        rp.call("sample_noise")
        n2 = rp.copy_out(eng._lib.BUF_NOISE, (N, T, 2))
        st2 = rp.copy_out(eng._lib.BUF_RNG, (N * T, 2), np.uint64)
        assert (st2 == g["states2"]).all()                       # integer stream bit exact
        # Box-Muller: libdevice logf/cosf + sqrt.approx vs numpy exact math: a few ulp
        np.testing.assert_allclose(n1, g["noise1"], rtol=3e-6, atol=2e-6)
        np.testing.assert_allclose(n2, g["noise2"], rtol=3e-6, atol=2e-6)
    finally:
        rp.close()


def test_noise_statistics_large(eng, dev):
    rp = RawPlanner(eng, 1, 4096, 1, 128, 8, 8, seed=5)
    try:
        rp.set_params(u_std=[2.0, 3.0])
        rp.call("sample_noise")
        n = rp.copy_out(eng._lib.BUF_NOISE, (4096, 128, 2)).astype(np.float64)
        assert np.isfinite(n).all()
        assert abs(n[..., 0].mean()) < 0.02 and abs(n[..., 1].mean()) < 0.03
        assert abs(n[..., 0].std() - 2.0) < 0.02 and abs(n[..., 1].std() - 3.0) < 0.03
        # vs the exact oracle stream, every element (bit-exact integers, the device's logf / cosf / sqrt.approx)
        st = X.create_states(4096 * 128, 5)
        want = MR.sample_noise(st, [2.0, 3.0], 4096, 128, arith=dev)
        assert_all_equal(n.astype(np.float32), want, "noise 4096 x 128")
    finally:
        rp.close()


# ----------------------------------------------------------------------------- 2. PMF setters + sampling
@pytest.mark.parametrize("mode", ["tdm", "det", "spd"])
@pytest.mark.parametrize("alpha", [0.3, 1.0])
def test_setter_and_sampling_vs_reference_golden(eng, golden_dir, mode, alpha):
    g = load(golden_dir, "ref_terrain.npz")
    key = "%s_a%02d" % (mode, int(alpha * 10))
    flags = dict(tdm=dict(use_tdm=True), det=dict(use_det_dynamics=True),
                 spd=dict(use_nom_dynamics_with_speed_map=True))[mode]
    cfg = eng.Config(T=1.0, dt=0.1, num_grid_samples=int(g["M"]), num_control_rollouts=100, seed=int(g["seed"]),
                     max_map_dim=tuple(int(v) for v in g["max_map_dim"]),
                     tdm_sample_thread_dim=tuple(int(v) for v in g["thread_dim"]),
                     max_speed_padding=float(g["max_speed_padding"]), **flags)
    tdm = eng.TDM_Numba(cfg)
    d = dict(res=float(g["res"]), xlimits=g["xlimits"], ylimits=g["ylimits"], bin_values=g["bin_values"],
             bin_values_bounds=np.asarray(g["bounds"]), det_dynamics_cvar_alpha=alpha)
    tdm.set_TDM_from_PMF_grid(g["pmf_lin"], d, g["obstacle"], g["unknown"])
    assert (tdm.pmf_grid_d.copy_to_host() == g[key + "_pmf_padded"]).all()
    np.testing.assert_allclose(tdm.padded_xlimits, g[key + "_pxl"])
    np.testing.assert_allclose(tdm.padded_ylimits, g[key + "_pyl"])
    assert tdm.pad_cells == int(g[key + "_pad"])
    assert (tdm.obstacle_map_d.copy_to_host() == g[key + "_obs_padded"]).all()
    assert (tdm.unknown_map_d.copy_to_host() == g[key + "_unk_padded"]).all()
    if mode == "spd":
        assert (tdm.risk_traction_map_d.copy_to_host() == g[key + "_risk"]).all()
    assert (tdm.rng_states_d.copy_to_host() == g[key + "_states0"]).all()
    g1 = tdm.sample_grids(1.0).copy_to_host()
    assert (g1 == g[key + "_grid1"]).all()
    g2 = tdm.sample_grids(0.6).copy_to_host()
    assert (g2 == g[key + "_grid2"]).all()
    assert (tdm.rng_states_d.copy_to_host() == g[key + "_states2"]).all()


def test_semantic_grid_setter_vs_reference_golden(eng, golden_dir):
    """set_TDM_from_semantic_grid (terrain.py:183-342) for the three modes: padded PMF, cropped semantic grid,
    risk map and the sampled maps (float64 bin values are uploaded uncast on this path: 0.2 -> 20, 0.6 -> 60)."""
    from oracle.make_golden import semantic_inputs, _T
    g = load(golden_dir, "ref_semantic.npz")
    sg, bin_values, names, pmfs, obstacle, unknown = semantic_inputs()
    assert (sg == g["sg"]).all()
    terr = {n: _T(n) for n in names.values()}
    t2p = {terr[n]: (bin_values, pmfs[n]) for n in terr}
    for mode, flags, alphas in (("tdm", dict(use_tdm=True), (None,)), ("det", dict(use_det_dynamics=True), (0.3, 1.0)),
                                ("spd", dict(use_nom_dynamics_with_speed_map=True), (0.3, 1.0))):
        for alpha in alphas:
            cfg = eng.Config(T=1.0, dt=0.1, num_grid_samples=2, num_control_rollouts=100, seed=1, max_map_dim=(14, 12),
                             tdm_sample_thread_dim=(3, 2), max_speed_padding=5.0, **flags)
            tdm = eng.TDM_Numba(cfg)
            tdm.set_TDM_from_semantic_grid(sg, 0.5, len(bin_values), bin_values, np.array([0.0, 1.0]),
                                           np.array([0.0, 3.5]), np.array([0.0, 4.5]), names, terr, t2p,
                                           det_dynamics_cvar_alpha=alpha, obstacle_map=obstacle, unknown_map=unknown)
            key = "%s_%s" % (mode, "none" if alpha is None else "a%02d" % int(alpha * 10))
            assert (tdm.pmf_grid_d.copy_to_host() == g[key + "_pmf_padded"]).all(), key
            assert (np.asarray(tdm.semantic_grid) == g[key + "_semantic_cropped"]).all(), key
            if mode == "spd":
                assert (tdm.risk_traction_map_d.copy_to_host() == g[key + "_risk"]).all(), key
            assert (tdm.sample_grids(0.9).copy_to_host() == g[key + "_grid1"]).all(), key


def test_sampling_generic_path_ill_formed_pmf_and_large_alpha(eng):
    """PMF columns that do not reach 100 and alpha_dyn > 1 (thresholds above every cumulative sum, int8 wrap
    above 127) take the generic kernel: cells whose column never reaches the threshold KEEP their previous
    content, like the reference (terrain.py:683-694, SURVEY.md 9-N4).  Bit-exact against the oracle."""
    rng = np.random.default_rng(31)
    B, H, W = 6, 30, 26
    pmf = rng.integers(0, 18, (B, H, W)).astype(np.int8)            # column sums 0..102, mostly < 100
    cfg = eng.Config(T=1.0, dt=0.1, num_grid_samples=5, num_control_rollouts=100, seed=3, max_map_dim=(36, 34),
                     tdm_sample_thread_dim=(4, 5), max_speed_padding=5.0, use_tdm=True)
    tdm = eng.TDM_Numba(cfg)
    d = dict(res=0.5, xlimits=np.array([0.0, W * 0.5]), ylimits=np.array([0.0, H * 0.5]),
             bin_values=np.array([0.0, 0.2, 0.4, 0.6, 0.8, 1.0]), bin_values_bounds=np.array([0.0, 1.0]),
             det_dynamics_cvar_alpha=1.0)
    tdm.set_TDM_from_PMF_grid(pmf, d)
    padded = tdm.pmf_grid_d.copy_to_host()
    st = TR.sample_rng_states(cfg.seed, 5, cfg.tdm_sample_thread_dim, False)
    want = np.zeros(tdm.sample_grid_batch_d.shape, dtype=np.int8)
    for alpha in (1.0, 1.5, 0.3):
        got = tdm.sample_grids(alpha).copy_to_host()
        TR.sample_grids(want, padded, st, tdm.bin_values, tdm.bin_values_bounds, alpha, cfg.tdm_sample_thread_dim, 5)
        assert (got == want).all(), alpha
        assert (tdm.rng_states_d.copy_to_host() == st).all(), alpha


def test_long_horizon_uses_smaller_window(eng, dev):
    """T = 800 steps (> 700): the windowed kernel switches to its 224-row variant; every cost equals the exact oracle."""
    sc = make_scenario("tdm", N=128, M=4, T=800, H=200, W=200, res=0.2, B=5, seed=14, warm_start=True)
    pl = staged_rollout(eng, sc)
    assert pl.cfg.num_steps == 800
    want = oracle_rollout_costs(sc, pl.lin_tdm, pl.ang_tdm, pl.noise_samples_d.copy_to_host(), pl.u_cur_d.copy_to_host(), arith=dev,
                                ctrl_order="presummed", wrap_clamp=True)
    assert_all_equal(pl.costs_nm_d.copy_to_host(), want, "T 800")
    assert pl.solve().shape == (800, 2)


def test_sampling_bit_exact_vs_oracle_config3_shape(eng):
    """512x512 map, 12 bins with non-representable bin values (compiled float64 truncation), M=64,
    16x16 thread tiles: bit-exact against the oracle's restatement of sample_grids_numba."""
    sc = make_scenario("tdm", N=128, M=64, T=8, H=512, W=512, res=0.1, B=12, seed=2)
    cfg = eng.Config(**sc["cfg"])
    tdm = eng.TDM_Numba(cfg)
    tdm.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    got = tdm.sample_grids(0.8).copy_to_host()
    padded = tdm.pmf_grid_d.copy_to_host()
    st = TR.sample_rng_states(cfg.seed, cfg.num_grid_samples, cfg.tdm_sample_thread_dim, False)
    want = np.zeros_like(got)
    TR.sample_grids(want, padded, st, tdm.bin_values, tdm.bin_values_bounds, 0.8, cfg.tdm_sample_thread_dim, 64)
    assert (got == want).all()
    assert (tdm.rng_states_d.copy_to_host() == st).all()
    # distribution property: the sampled bin frequencies follow the PMF (chi-square-ish bound)
    inner = got[:, 5:-5, 5:-5].astype(np.int64)
    assert 30 < inner.mean() < 70


# ----------------------------------------------------------------------------- 3. rollouts
def _golden_rollout_planner(eng, g, mode, goal, M):
    R, Cc = g["lin"].shape[1:]
    Hp, Wp = g["obs"].shape
    N, T = g["noise"].shape[:2]
    rp = RawPlanner(eng, mode, N, M, T, R, Cc)
    dummy = np.zeros((2, Hp, Wp), dtype=np.int8)
    dummy[1] = 100
    for which in ("lin", "ang"):
        rp.set_map(which, dummy, [0.0, 1.0], g[which + "_bounds"], g["res"], g["xlim"], g["ylim"],
                   g["obs"], g["unk"], g["risk"][0] if mode == 2 else None)
    rp.set_grids("lin", g["lin"][:rp.M])
    rp.set_grids("ang", g["ang"][:rp.M])
    rp.copy_in(eng._lib.BUF_NOISE, g["noise"])
    rp.copy_in(eng._lib.BUF_U_CUR, g["u_cur"])
    return rp


@pytest.mark.parametrize("gname", ["near", "far"])
def test_rollouts_vs_reference_golden(eng, golden_dir, gname):
    g = load(golden_dir, "ref_rollout.npz")
    goal = g["xgoal_" + gname]
    common = dict(x0=list(g["x0"]), xgoal=list(goal), dt=float(g["dt"]))
    M = g["lin"].shape[0]
    N = g["noise"].shape[0]
    for alpha in (0.5, 0.9, 1.0):
        rp = _golden_rollout_planner(eng, g, 0, goal, M)
        try:
            rp.set_params(cvar_alpha=alpha, **common)
            rp.call("rollout")
            cnm = rp.copy_out(eng._lib.BUF_COSTS_NM, (N, M))
            assert rel_err(cnm, g["sto_cnm_" + gname]).max() < 1e-4
            cv = rp.copy_out(eng._lib.BUF_COSTS, (N,))
            assert rel_err(cv, g["sto_cvar%02d_%s" % (int(alpha * 10), gname)]).max() < 1e-4
        finally:
            rp.close()
    for mode, key in ((1, "det_"), (2, "spd_")):
        rp = _golden_rollout_planner(eng, g, mode, goal, 1)
        try:
            rp.set_params(**common)
            rp.call("rollout")
            c = rp.copy_out(eng._lib.BUF_COSTS, (N,))
            assert rel_err(c, g[key + gname]).max() < 1e-4
        finally:
            rp.close()


@pytest.mark.parametrize("mode,N,M,T,H,res,B,near,warm", [
    ("det", 1024, 1, 64, 256, 0.2, 2, False, False),       # BASELINE config 2
    ("tdm", 1024, 64, 64, 512, 0.1, 12, False, True),      # BASELINE config 3
    ("tdm", 512, 32, 48, 200, 0.1, 12, True, True),        # goal within reach: early exits
    ("det", 4096, 1, 128, 512, 0.2, 32, False, True),      # BASELINE config 4 (CVaR-dynamics alpha 0.3)
    ("spd", 1024, 1, 64, 256, 0.2, 12, True, True),        # speed-map mode
    ("tdm", 512, 16, 128, 900, 0.05, 12, False, True),     # fine grid: rollouts LEAVE the staged window
    ("tdm", 256, 1100, 32, 128, 0.1, 12, False, True),     # M > 1024: the reference's "oversized" dispatch
])
def test_rollout_costs_vs_oracle(eng, dev, mode, N, M, T, H, res, B, near, warm):
    sc = make_scenario(mode, N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=4, near_goal=near, warm_start=warm,
                       det_alpha=0.3 if B == 32 else 1.0)
    pl = staged_rollout(eng, sc)                          # warm-started from sc["u0"] exactly when `warm`
    assert pl.cfg.num_steps == T
    noise = pl.noise_samples_d.copy_to_host()
    u_cur = pl.u_cur_d.copy_to_host()
    # the windowed kernel (stochastic mode) adds the pre-summed control cost, the deterministic kernels add the terms
    # one by one: the exact oracle in each kernel's order, every (n, m) equal
    want = oracle_rollout_costs(sc, pl.lin_tdm, pl.ang_tdm, noise, u_cur, arith=dev, wrap_clamp=True,
                                ctrl_order="presummed" if mode == "tdm" else "sequential")
    if mode == "tdm":
        got = pl.costs_nm_d.copy_to_host()
    else:
        got = pl.costs_d.copy_to_host()[:, None]
    assert_all_equal(got, want, "%s N%d M%d T%d" % (mode, N, M, T))
    if mode == "tdm":
        cv = pl.costs_d.copy_to_host()
        # CVaR of the engine's own per-(n,m) costs: the exact mean of the numel largest, within the kernel's bound
        RB.check_cvar(cv, got, sc["params"]["cvar_alpha"], label="%s N%d M%d" % (mode, N, M))
    if near:
        assert (got < 0.5 * np.median(got)).any(), "near-goal case should contain early exits"


@pytest.mark.parametrize("maskmax", [1, 3])
def test_window_kernel_equals_generic_kernel(eng, monkeypatch, maskmax):
    """The TMA-window kernel and the generic global-memory kernel walk identical trajectories: per-(n,m)
    costs agree to the rounding of the pre-summed control cost (~1 ulp), including rollouts that leave
    the window (res 0.05 m, T = 128).  maskmax = 1: masks of 0 / 1 (the windowed kernel's MASK01 variant);
    3: obstacle bytes 0 .. 3 (its general penalty arithmetic)."""
    sc = make_scenario("tdm", N=512, M=16, T=128, H=900, W=900, res=0.05, B=12, seed=8, warm_start=True)
    if maskmax > 1:
        rng = np.random.default_rng(3)
        sc["obstacle"] = (sc["obstacle"].astype(np.int64) * rng.integers(1, maskmax + 1, sc["obstacle"].shape)).astype(sc["obstacle"].dtype)
        assert sc["obstacle"].max() > 1
    outs = []
    for no_win in (False, True):
        if no_win:
            monkeypatch.setenv("B200MPPI_NO_WINDOW", "1")
        pl = staged_rollout(eng, sc)
        outs.append(pl.costs_nm_d.copy_to_host())
    monkeypatch.delenv("B200MPPI_NO_WINDOW")
    r = rel_err(outs[0], outs[1])
    assert r.max() < 2e-6, r.max()


CVAR_SHAPES = [1, 31, 32, 33, 63, 64, 65, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 4097, 16384]


def _cvar_alpha(M, numel):
    if numel >= M:
        return 1.0
    a = (numel - 0.5) / M
    assert RB.cvar_numel(M, a) == numel
    return a


def test_cvar_selection_properties(eng):
    """CVaR kernel alone on adversarial inputs: ties (also at the threshold), signed zeros, +inf, negatives, magnitudes
    1e-30 .. 1e30, M around every PER step and the CTA kernel, numel in {1, 2, M-1, M} and the alpha edge cases; the
    exact mean of the numel largest values within the kernel's bound (tests/reduce_bounds.py)."""
    L = eng._lib
    rng = np.random.default_rng(0)
    cases = [(6, 0.5), (33, 0.1), (100, 0.999), (256, 0.5), (1000, 0.25), (1024, 1.0), (7, 0.01), (1, 0.5),
             (1025, 0.5), (3000, 0.1), (2048, 1.0), (15000, 0.999), (4097, 0.0001),     # CTA kernel (M > 1024)
             (1000, 0.1)]                 # float32(0.1) * 1000: ceil 101 in float64, 100 in float32
    cases = list(dict.fromkeys(cases + sorted({(M, _cvar_alpha(M, k)) for M in CVAR_SHAPES for k in (1, 2, M - 1, M)
                                               if 1 <= k <= M})))
    worst = 0.0
    for M, alpha in cases:
        N = 130
        rp = RawPlanner(eng, 0, N, M, 4, 8, 8)
        try:
            c = rng.normal(0, 100, (N, M)).astype(np.float32)
            c[:, ::3] = np.round(c[:, ::3])            # many exact ties
            c[5] = 7.0                                  # all equal
            c[6] = -np.abs(c[6])                        # all negative
            extra = RB.cvar_rows(M, RB.cvar_numel(M, alpha), M)
            c[10:10 + len(extra)] = extra
            rp.copy_in(L.BUF_COSTS_NM, c)
            rp.set_params(cvar_alpha=alpha)
            rp.call("cvar")
            got = rp.copy_out(L.BUF_COSTS, (N,))
            worst = max(worst, RB.check_cvar(got, c, alpha, label="M=%d alpha=%r" % (M, alpha)))
        finally:
            rp.close()
    print("\n[cvar] largest |error| / bound %.3g" % worst)


# ----------------------------------------------------------------------------- 4. update
@pytest.mark.parametrize("lam", [1.0, 0.3])
def test_update_vs_reference_golden(eng, golden_dir, lam):
    g = load(golden_dir, "ref_update.npz")
    N, T = g["noise"].shape[:2]
    rp = RawPlanner(eng, 1, N, 1, T, 8, 8)
    try:
        rp.set_params(lambda_weight=lam, vrange=list(g["vrange"]), wrange=list(g["wrange"]))
        rp.copy_in(eng._lib.BUF_NOISE, g["noise"])
        rp.copy_in(eng._lib.BUF_U_CUR, g["u0"])
        c = np.ascontiguousarray(g["costs"])
        rp.call("update", eng._lib.ptr(c))
        u = rp.copy_out(eng._lib.BUF_U_CUR, (T, 2))
        w = rp.copy_out(eng._lib.BUF_WEIGHTS, (N,))
        np.testing.assert_allclose(w, g["w_lam%02d" % int(lam * 10)], rtol=1e-4, atol=1e-9)
        np.testing.assert_allclose(u, g["u_lam%02d" % int(lam * 10)], rtol=1e-4, atol=1e-5)
        RB.check_update(u, w, g["costs"], g["noise"], g["u0"], lam, g["vrange"], g["wrange"], label="golden")
        assert (rp.copy_out(eng._lib.BUF_COSTS, (N,)) == g["costs"]).all()     # costs_d is not clobbered
    finally:
        rp.close()


VR32, WR32 = np.array([0, 3], np.float32), np.array([-np.pi, np.pi], np.float32)
UPD_SHAPES = [(8192, 128), (1000, 50), (100, 1024), (37, 3),
              (1, 1024), (2, 513), (31, 512), (32, 511), (33, 257), (9472, 256), (9473, 255), (16384, 1), (15000, 64),
              (16384, 1024)]
UPD_VALUES = [(k, lam) for k in ("mild", "underflow", "far", "signed", "inf", "clip", "cancel")
              for lam in (1e-3, 0.3, 1.0, 1e3)]


def _gpu_update(eng, costs, noise, u0, lam):
    N, T = noise.shape[:2]
    rp = RawPlanner(eng, 1, N, 1, T, 8, 8)
    try:
        rp.set_params(lambda_weight=lam)
        rp.copy_in(eng._lib.BUF_NOISE, noise)
        rp.copy_in(eng._lib.BUF_U_CUR, u0)
        c = np.ascontiguousarray(costs)
        rp.call("update", eng._lib.ptr(c))
        return rp.copy_out(eng._lib.BUF_U_CUR, (T, 2)), rp.copy_out(eng._lib.BUF_WEIGHTS, (N,))
    finally:
        rp.close()


@pytest.mark.parametrize("N,T,kind,lam", [pytest.param(N, T, "base", 1.0, id="%d-%d" % (N, T)) for N, T in UPD_SHAPES] +
                         [(N, T, k, lam) for N, T in ((1000, 50), (9473, 33)) for k, lam in UPD_VALUES])
def test_update_vs_oracle_large(eng, N, T, kind, lam):
    """The one-launch update against the float64 reference within the bound of tests/reduce_bounds.py, across the
    row batches, the four column chunks and the value cases (underflowing CTAs, costs near 1e6, signed costs,
    scattered +inf, u0 on the clip bounds, cancelling noise, lambda 1e-3 .. 1e3)."""
    if kind == "base":
        rng = np.random.default_rng(N)
        costs = rng.uniform(4000, 4020, N).astype(np.float32)
        noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(np.float32)
        u0 = np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(np.float32)
    else:
        costs, noise, u0 = RB.update_inputs(kind, N, T, seed=N + T, lam=lam)
    u, w = _gpu_update(eng, costs, noise, u0, lam)
    ru, rw = RB.check_update(u, w, costs, noise, u0, lam, VR32, WR32, label="N%d T%d %s lam %g" % (N, T, kind, lam))
    print("\n[update N%d T%d %s lam %g] |error| / bound: u %.3g, weights %.3g" % (N, T, kind, lam, ru, rw))
    assert abs(float(w.sum(dtype=np.float64)) - 1.0) < 1e-5


@pytest.mark.parametrize("N", [1000, 9473])
def test_update_with_an_all_inf_cta_slab(eng, N):
    """One CTA slab of +inf costs (its baseline is +inf, c - beta = inf - inf): the slab's rollouts get weight exactly
    0, no weight is NaN and u equals the float64 reference (whose beta is the global minimum) within the bound --
    before, the slab's NaN partial made u the clip bounds' upper ends."""
    T = 4 if N == 1000 else 64
    costs = RB.inf_slab_costs(N)
    rng = np.random.default_rng(N)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(np.float32)
    u0 = np.stack([rng.uniform(0, 2.9, T), rng.uniform(-3, 3, T)], 1).astype(np.float32)
    u, w = _gpu_update(eng, costs, noise, u0, 1.0)
    RB.check_update(u, w, costs, noise, u0, 1.0, VR32, WR32, label="all-inf slab, N %d" % N)


def test_update_sharded_equals_single(eng):
    """N sharded over 4 'ranks' (4 planners on one GPU), partials gathered by hand -> same u as 1 rank, each within the
    bound of the float64 reference (host combine and device combine)."""
    _sharded_update(eng, "mild")


def test_update_sharded_with_an_all_inf_rank(eng):
    """One rank's rollouts all cost +inf: that rank's partial (beta +inf, S 0, V 0) must not poison the others' u, in
    the host combine and in every rank's device combine; its rollouts get weight exactly 0."""
    _sharded_update(eng, "inf_rank")


def _sharded_update(eng, kind):
    L = eng._lib
    N, T, ws = 2048, 64, 4
    rng = np.random.default_rng(3)
    costs = rng.uniform(900, 930, N).astype(np.float32)
    if kind == "inf_rank":
        costs[N // ws: 2 * N // ws] = np.inf
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(np.float32)
    u0 = rng.uniform(0, 1, (T, 2)).astype(np.float32)
    single = RawPlanner(eng, 1, N, 1, T, 8, 8)
    ranks = [RawPlanner(eng, 1, N, 1, T, 8, 8, rank=r, world=ws) for r in range(ws)]
    try:
        single.set_params()
        single.copy_in(L.BUF_NOISE, noise)
        single.copy_in(L.BUF_U_CUR, u0)
        single.call("update", L.ptr(costs))
        u1 = single.copy_out(L.BUF_U_CUR, (T, 2))
        w1 = single.copy_out(L.BUF_WEIGHTS, (N,))
        RB.check_update(u1, w1, costs, noise, u0, 1.0, VR32, WR32, label="one rank " + kind)
        parts = []
        for r, rp in enumerate(ranks):
            sl = slice(N * r // ws, N * (r + 1) // ws)
            rp.set_params()
            rp.copy_in(L.BUF_NOISE, noise[sl])
            rp.copy_in(L.BUF_U_CUR, u0)
            c = np.ascontiguousarray(costs[sl])
            rp.call("update", L.ptr(c))                       # world > 1: stops after the rank partial
            parts.append(rp.copy_out(L.BUF_PARTIAL, (2 * T + 2,)))
        gathered = np.ascontiguousarray(np.stack(parts))
        # host combine (the library's reference implementation of the exchange math)
        out = np.empty((T, 2), np.float32)
        L.check(L.lib.b200mppi_combine_partials_host(L.ptr(gathered), ws, T, np.float32(1.0), L.ptr(u0), L.ptr(VR32),
                                                     L.ptr(WR32), L.ptr(out)))
        RB.check_update(out, None, costs, noise, u0, 1.0, VR32, WR32, N=N // ws, merges=ws, label="host combine " + kind)
        # device combine on every rank from a device copy of the gathered partials
        import torch
        gd = torch.from_numpy(gathered).cuda()
        ws_w, us = [], []
        for r, rp in enumerate(ranks):
            rp.call("solve_finish", C.c_void_p(gd.data_ptr()), None)
            rp.call("synchronize")
            us.append(rp.copy_out(L.BUF_U_CUR, (T, 2)))
            ws_w.append(rp.copy_out(L.BUF_WEIGHTS, (rp.n_local,)))
        assert all((x == us[0]).all() for x in us)
        RB.check_update(us[0], np.concatenate(ws_w), costs, noise, u0, 1.0, VR32, WR32, N=N // ws, merges=ws,
                        label="device combine " + kind)
    finally:
        single.close()
        for rp in ranks:
            rp.close()


def _rank_planner(eng, sc, rank, world):
    """(planner, lin, ang) of scenario sc as rank `rank` of `world`, its params on the device."""
    pl = tdm_planner(eng, sc, rank=rank, world_size=world)
    pl.move_mppi_task_vars_to_device()
    return pl, pl.lin_tdm, pl.ang_tdm


def test_map_sharded_solve_equals_single_rank(eng):
    """MODE_TDM on 2 'ranks' (both on this GPU, the all-to-all / all-gather done by hand): each rank's
    sampled maps are bit-identical to its slice of the single-rank maps, its CVaR costs are bit-identical
    to the single-rank costs of its control sequences, and every rank ends with the single-rank u."""
    import torch
    L = eng._lib
    ws = 2
    sc = make_scenario("tdm", N=256, M=16, T=32, H=120, W=120, res=0.2, B=8, seed=10, warm_start=True)
    single, slin, sang = _rank_planner(eng, sc, 0, 1)
    u_single = single.solve()
    maps_single = slin.sample_grid_batch_d.copy_to_host()
    costs_single = single.costs_d.copy_to_host()
    ranks = [_rank_planner(eng, sc, r, ws) for r in range(ws)]
    N, M = sc["N"], sc["M"]
    sends = []
    for r, (pl, lin, ang) in enumerate(ranks):
        assert lin.sample_grid_batch_d.shape[0] == M // ws and pl.costs_nm_d.shape == (N, M // ws)
        L.check(L.lib.b200mppi_planner_solve_local(pl._handle, 1))
        L.check(L.lib.b200mppi_planner_synchronize(pl._handle))
        assert (lin.sample_grid_batch_d.copy_to_host() == maps_single[r * M // ws:(r + 1) * M // ws]).all()
        assert (pl.noise_samples_d.copy_to_host() == single.noise_samples_d.copy_to_host()).all()
        sends.append(pl.costs_nm_d.copy_to_host())
    parts, keep = [], []
    for d, (pl, lin, ang) in enumerate(ranks):
        # what the all-to-all delivers: block g = rank g's maps x this rank's control sequences, map-major
        recv = np.ascontiguousarray(np.stack([sends[g][d * N // ws:(d + 1) * N // ws].T for g in range(ws)]))
        t = torch.from_numpy(recv).cuda()
        keep.append(t)
        L.check(L.lib.b200mppi_planner_solve_reduce(pl._handle, C.c_void_p(t.data_ptr())))
        L.check(L.lib.b200mppi_planner_synchronize(pl._handle))
        assert (pl.costs_d.copy_to_host() == costs_single[d * N // ws:(d + 1) * N // ws]).all()
        parts.append(pl.partial_d.copy_to_host())
    gathered = torch.from_numpy(np.ascontiguousarray(np.stack(parts))).cuda()
    for pl, lin, ang in ranks:
        u = np.empty_like(u_single)
        L.check(L.lib.b200mppi_planner_solve_finish(pl._handle, C.c_void_p(gathered.data_ptr()), L.ptr(u)))
        np.testing.assert_allclose(u, u_single, rtol=1e-5, atol=2e-6)


def _connect_local(L, planners):
    hs = [pl._handle.value if hasattr(pl._handle, "value") else pl._handle for pl in planners]
    arr = (C.c_void_p * len(hs))(*hs)
    for pl in planners:
        L.check(L.lib.b200mppi_planner_p2p_connect_local(pl._handle, arr, len(hs)))


@pytest.mark.parametrize("mode,ws", [("tdm", 2), ("tdm", 4), ("det", 4)])
def test_p2p_exchange_equals_single_rank(eng, mode, ws):
    """The peer-memory exchange (p2p.cu): ws 'ranks' living in this process on this GPU, connected with
    p2p_connect_local, run the phase calls of solve_p2p interleaved (local / push / reduce / finish) without
    host synchronisation in between; three consecutive solves (epoch flags, double-buffered gather) give
    the single-rank u on every rank, and the CVaR costs of each rank's slice are bit-identical."""
    L = eng._lib
    sc = make_scenario(mode, N=512, M=16 if mode == "tdm" else 1, T=32, H=120, W=120, res=0.2, B=8, seed=14,
                       warm_start=True)
    single = _rank_planner(eng, sc, 0, 1)
    ranks = [_rank_planner(eng, sc, r, ws) for r in range(ws)]
    pls = [r[0] for r in ranks]
    _connect_local(L, pls)
    N = sc["N"]
    for it in range(3):
        u_single = single[0].solve()
        costs_single = single[0].costs_d.copy_to_host()
        for pl in pls:
            L.check(L.lib.b200mppi_planner_solve_local(pl._handle, 1))
        if mode == "tdm":
            for pl in pls:
                L.check(L.lib.b200mppi_planner_p2p_push(pl._handle))
        for pl in pls:
            L.check(L.lib.b200mppi_planner_p2p_reduce(pl._handle))
        us = []
        for pl in pls:
            u = np.empty_like(u_single)
            L.check(L.lib.b200mppi_planner_p2p_finish(pl._handle, L.ptr(u)))
            us.append(u)
        for d, pl in enumerate(pls):
            assert (pl.costs_d.copy_to_host() == costs_single[d * N // ws:(d + 1) * N // ws]).all(), (it, d)
            np.testing.assert_allclose(us[d], u_single, rtol=1e-5, atol=2e-6, err_msg="solve %d rank %d" % (it, d))
            assert (us[d] == us[0]).all()                      # every rank combines the same partials
            pl.u_cur_d.copy_to_device(u_single)                # (u differs from 1 rank by summation order only;
                                                               #  re-align so the next solve's costs compare bitwise)


def test_p2p_wait_times_out_instead_of_hanging(eng, monkeypatch):
    """A rank that never arrives: the wait kernel gives up after B200MPPI_P2P_TIMEOUT_MS and the call
    reports which rank was missing (no hung GPU)."""
    L = eng._lib
    monkeypatch.setenv("B200MPPI_P2P_TIMEOUT_MS", "50")
    sc = make_scenario("det", N=256, M=1, T=16, H=60, W=60, res=0.2, B=4, seed=15)
    pls = [_rank_planner(eng, sc, r, 2) for r in range(2)]
    _connect_local(L, [p[0] for p in pls])
    pl = pls[0][0]
    L.check(L.lib.b200mppi_planner_solve_local(pl._handle, 1))
    L.check(L.lib.b200mppi_planner_p2p_reduce(pl._handle))
    u = np.empty((16, 2), np.float32)
    rc = L.lib.b200mppi_planner_p2p_finish(pl._handle, L.ptr(u))          # rank 1 never posts its partial
    assert rc != 0
    assert "rank 1" in L.lib.b200mppi_last_error().decode()


# ----------------------------------------------------------------------------- 5. whole solve through the public API
def _golden_solve_planner(eng, g, mode, **cfg_kw):
    """(planner, lin, ang) of the ref_solve.npz scenario in `mode`, set up as the reference's public calls set it up."""
    flags = dict(tdm=dict(use_tdm=True), det=dict(use_det_dynamics=True),
                 spd=dict(use_nom_dynamics_with_speed_map=True))[mode]
    cfg = eng.Config(T=float(g["T_s"]), dt=float(g["dt"]), num_grid_samples=int(g["M"]),
                     num_control_rollouts=int(g["N"]), seed=int(g["seed"]),
                     max_map_dim=tuple(int(v) for v in g["max_map_dim"]),
                     tdm_sample_thread_dim=tuple(int(v) for v in g["thread_dim"]),
                     max_speed_padding=float(g["max_speed_padding"]), **cfg_kw, **flags)
    H, W = g["obstacle"].shape
    res = float(g["res"])
    d = dict(res=res, xlimits=np.array([0.0, W * res]), ylimits=np.array([0.0, H * res]),
             bin_values=g["bin_values"], bin_values_bounds=np.array([0.0, 1.0]), det_dynamics_cvar_alpha=0.4)
    lin, ang = tdm_pair(eng, cfg, g["pmf_lin"], g["pmf_ang"], d, g["obstacle"], g["unknown"])
    pl = eng.MPPI_Numba(cfg)
    p = dict(dt=0.1, x0=np.array([2.3, 3.1, 0.3]), xgoal=np.array([5.0, 4.5]), goal_tolerance=0.5,
             v_post_rollout=0.01, cvar_alpha=0.5, alpha_dyn=1.0, dist_weight=1.0, lambda_weight=1.0, num_opt=1,
             u_std=np.array([2.0, 3.0]), vrange=np.array([0.0, 3.0]), wrange=np.array([-np.pi, np.pi]),
             obs_penalty=1e5, unknown_penalty=1e2)
    pl.setup(p, lin, ang)
    return pl, lin, ang


@pytest.mark.parametrize("mode", ["tdm", "det", "spd"])
def test_solve_vs_reference_golden(eng, golden_dir, mode):
    """Config -> TDM setters -> setup -> solve -> shift_and_update -> solve, the reference's public call
    sequence, against what the reference itself returned for the same seed (ref_solve.npz)."""
    g = load(golden_dir, "ref_solve.npz")
    pl, lin, ang = _golden_solve_planner(eng, g, mode)
    u1 = pl.solve()
    assert (lin.sample_grid_batch_d.copy_to_host() == g[mode + "_lin_grid1"]).all()
    assert (ang.sample_grid_batch_d.copy_to_host() == g[mode + "_ang_grid1"]).all()
    np.testing.assert_allclose(pl.noise_samples_d.copy_to_host(), g[mode + "_noise1"], rtol=3e-6, atol=2e-6)
    np.testing.assert_allclose(u1, g[mode + "_u1"], rtol=1e-3, atol=2e-4)
    pl.shift_and_update(np.array([2.4, 3.15, 0.35]), g[mode + "_u1"], num_shifts=1)
    u2 = pl.solve()
    np.testing.assert_allclose(u2, g[mode + "_u2"], rtol=2e-3, atol=5e-4)
    w = pl.weights_d.copy_to_host()
    assert abs(float(w.sum()) - 1.0) < 1e-5


@pytest.mark.parametrize("mode", ["tdm", "det", "spd"])
def test_state_rollout_vs_reference_golden(eng, dev, golden_dir, mode):
    """get_state_rollout() after the first solve() of the ref_solve.npz scenario against what the reference's
    own kernels (mppi.py:1194-1351) returned (ref_state_rollout.npz), and against the oracle on the engine's
    own buffers."""
    g = load(golden_dir, "ref_solve.npz")
    s = load(golden_dir, "ref_state_rollout.npz")
    pl, lin, ang = _golden_solve_planner(eng, g, mode, num_vis_state_rollouts=5)
    res, p = float(g["res"]), pl.params
    pl.solve()
    got = pl.get_state_rollout()
    assert got.shape == s[mode + "_states"].shape
    m = dict(tdm=MR.MODE_STOCHASTIC, det=MR.MODE_DET_DYN, spd=MR.MODE_SPEED_MAP)[mode]
    want = MR.state_rollouts(m, got.shape[0], lin.sample_grid_batch_d.copy_to_host(),
                             ang.sample_grid_batch_d.copy_to_host(), [0.0, 1.0], [0.0, 1.0], res, lin.padded_xlimits,
                             lin.padded_ylimits, p["x0"], 0.1, pl.u_cur_d.copy_to_host(), pl.u_prev_d.copy_to_host(),
                             pl.noise_samples_d.copy_to_host(), p["vrange"], p["wrange"], arith=dev, wrap_clamp=True)
    assert_all_equal(got, want, "state rollout, %s" % mode)                  # same inputs: engine vs exact oracle
    np.testing.assert_allclose(got, s[mode + "_states"], rtol=2e-3, atol=2e-3)   # vs the reference's run (its u1
                                                                                 # differs from ours by ~1e-4)


def test_solve_preconditions_and_api_surface(eng, capsys):
    sc = make_scenario("det", N=128, M=1, T=16, H=40, W=40, res=0.5, B=5, seed=9)
    cfg = eng.Config(**sc["cfg"])
    pl = eng.MPPI_Numba(cfg)
    assert pl.solve() is None                                    # print + None, like the reference
    assert "not set" in capsys.readouterr().out
    lin, ang = eng.TDM_Numba(cfg), eng.TDM_Numba(cfg)
    pl.set_tdm(lin, ang)
    lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    bad = dict(sc["params"])
    bad["x0"] = np.array([1e3, 0.0, 0.0])
    with pytest.raises(AssertionError):
        pl.set_params(bad)
    pl.set_params(sc["params"])
    assert pl.solve() is None                                    # angular PMF missing
    ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    u = pl.solve()
    assert u.shape == (16, 2) and u.dtype == np.float32
    assert (u[:, 0] >= 0).all() and (u[:, 0] <= 3).all() and (np.abs(u[:, 1]) <= np.pi + 1e-6).all()
    for name, shape in (("noise_samples_d", (128, 16, 2)), ("u_cur_d", (16, 2)), ("costs_d", (128,)),
                        ("weights_d", (128,)), ("rng_states_d", (128 * 16, 2))):
        a = getattr(pl, name)
        assert a.shape == shape and a.copy_to_host().shape == shape
    assert (pl.u_cur_d.copy_to_host() == u).all()
    assert (pl.u_prev_d.copy_to_host() == u).all()               # det modes: u_prev aliases u_cur (9-Q2)
    sr = pl.get_state_rollout()
    assert sr.shape == (cfg.num_vis_state_rollouts, 17, 3)
    np.testing.assert_allclose(sr[:, 0, :], np.tile(sc["params"]["x0"].astype(np.float32), (sr.shape[0], 1)))
    # shift keeps the tail
    pl.shift_and_update(sc["params"]["x0"], u, num_shifts=2)
    s = pl.u_cur_d.copy_to_host()
    assert (s[:-2] == u[2:]).all() and (s[-2:] == u[-2:]).all()
    # zero-copy view
    import torch
    t = torch.as_tensor(pl.u_cur_d, device="cuda")
    assert (t.cpu().numpy() == s).all()


def test_barebone_variant_vs_reference_notebook_golden(eng, golden_dir):
    """The map-free MPPI of barebone_mppi_numba.ipynb: kernel-level costs on injected noise, then the notebook's
    public call sequence (setup / solve / get_state_rollout / shift_and_update / solve) against what the
    notebook's own classes returned for the same seed."""
    from mppi_numba_b200 import barebone as BB
    g = load(golden_dir, "ref_barebone.npz")
    L = eng._lib
    N, T = g["noise"].shape[:2]
    for gname in ("near", "far"):
        rp_pod = L.ConfigPOD(num_steps=T, num_control_rollouts=N, num_grid_samples=1, max_map_rows=1, max_map_cols=1,
                             tdm_thread_x=1, tdm_thread_y=1, num_vis_state_rollouts=1, mode=L.MODE_BAREBONE, device=0,
                             rank=0, world_size=1, seed=1)
        h = C.c_void_p()
        L.check(L.lib.b200mppi_planner_create(C.byref(rp_pod), C.byref(h)))
        try:
            p = L.ParamsPOD()
            p.dt = 0.1
            p.x0 = L.c_floats(g["x0"], 3)
            p.xgoal = L.c_floats(g["goal_" + gname], 2)
            p.goal_tolerance, p.lambda_weight, p.cvar_alpha, p.num_opt, p.alpha_dyn = 0.5, 1.0, 1.0, 1, 1.0
            p.u_std = L.c_floats([1.0, 1.0], 2)
            p.vrange = L.c_floats([0.0, 2.0], 2)
            p.wrange = L.c_floats(np.array([-np.pi, np.pi], np.float32), 2)
            p.obs_penalty, p.dist_weight = 1e6, 10.0
            L.check(L.lib.b200mppi_planner_set_params(h, C.byref(p)))
            pos, rad = np.ascontiguousarray(g["obs_pos"]), np.ascontiguousarray(g["obs_r"])
            L.check(L.lib.b200mppi_planner_set_obstacles(h, L.ptr(pos), L.ptr(rad), len(rad)))
            noise, u_cur = np.ascontiguousarray(g["noise"]), np.ascontiguousarray(g["u_cur"])
            L.check(L.lib.b200mppi_planner_copy_in(h, L.BUF_NOISE, L.ptr(noise), noise.nbytes))
            L.check(L.lib.b200mppi_planner_copy_in(h, L.BUF_U_CUR, L.ptr(u_cur), u_cur.nbytes))
            L.check(L.lib.b200mppi_planner_rollout(h))
            c = np.empty(N, np.float32)
            L.check(L.lib.b200mppi_planner_copy_out(h, L.BUF_COSTS, L.ptr(c), c.nbytes))
            assert rel_err(c, g["costs_" + gname]).max() < 1e-4
        finally:
            L.lib.b200mppi_planner_destroy(h)
    cfg = BB.Config(T=1.0, dt=0.1, num_control_rollouts=100, num_vis_state_rollouts=5, seed=1)
    pl = BB.MPPI_Numba(cfg)
    params = dict(dt=0.1, x0=np.array([0.0, 0.0, np.pi / 4]), xgoal=np.array([7.0, 5.0]), goal_tolerance=0.5,
                  dist_weight=10, lambda_weight=1.0, num_opt=1, u_std=np.array([1.0, 1.0]),
                  vrange=np.array([0.0, 2.0]), wrange=np.array([-np.pi, np.pi]),
                  obstacle_positions=np.array([[5, 4.5], [2, 1]]), obstacle_radius=np.array([1.5, 1.0]), obs_penalty=1e6)
    assert pl.solve() is None
    pl.setup(params)
    u1 = pl.solve()
    np.testing.assert_allclose(pl.noise_samples_d.copy_to_host(), g["solve_noise1"], rtol=3e-6, atol=2e-6)
    np.testing.assert_allclose(u1, g["solve_u1"], rtol=1e-3, atol=2e-4)
    np.testing.assert_allclose(pl.get_state_rollout(), g["solve_states1"], rtol=1e-3, atol=1e-3)
    pl.shift_and_update(np.array([0.05, 0.06, 0.8]), g["solve_u1"], num_shifts=1)
    np.testing.assert_allclose(pl.solve(), g["solve_u2"], rtol=2e-3, atol=5e-4)


def test_full_size_config5_properties(eng, dev):
    """BASELINE config 5 at FULL size (N 8192, M 256, T 128, 1034x1034 maps) through size-independent
    properties: run-to-run determinism, CVaR == host selection on the engine's own per-(n,m) costs,
    sampled values drawn from the quantised bin set with the right marginal, normalised weights, clipped u,
    and equality with the exact oracle on a slice (256 control sequences x 8 maps x 128 steps)."""
    from bench import build_scenario
    sc = build_scenario("c5")
    L = eng._lib
    a = tdm_planner(eng, sc)
    alin = a.lin_tdm
    u1 = a.solve()
    u2 = a.solve()
    cnm = a.costs_nm_d.copy_to_host()
    cv = a.costs_d.copy_to_host()
    N, M = cnm.shape
    assert (N, M) == (8192, 256)
    k = MR.cvar_count(M, sc["params"]["cvar_alpha"])
    top = np.sort(cnm, axis=1)[:, M - k:]                       # the k largest per control sequence
    np.testing.assert_allclose(cv, top.astype(np.float64).mean(axis=1), rtol=3e-6)
    w = a.weights_d.copy_to_host()
    assert abs(float(w.sum(dtype=np.float64)) - 1.0) < 1e-5 and (w >= 0).all()
    for u in (u1, u2):
        assert np.isfinite(u).all() and (u[:, 0] >= 0).all() and (u[:, 0] <= 3).all()
        assert (np.abs(u[:, 1]) <= np.float32(np.pi)).all()
    # sampled maps: every value is one of the quantised bin values; marginal frequency of the top bin
    g = alin.sample_grid_batch_d.copy_to_host()
    q = TR.quantise_bin_values(alin.bin_values, alin.bin_values_bounds)
    assert np.isin(g[:, 5:-5, 5:-5], q).all()
    pad = alin.pad_cells
    exp_top = sc["pmf_lin"][-1].astype(np.float64).mean() / 100.0
    got_top = float((g[:8, pad:-pad, pad:-pad] == q[-1]).mean())
    assert abs(got_top - exp_top) < 2e-3
    # determinism: a second engine with the same seed reproduces both solves bit for bit
    b = tdm_planner(eng, sc)
    blin, bang = b.lin_tdm, b.ang_tdm
    assert (b.solve() == u1).all() and (b.solve() == u2).all()
    # oracle parity on a slice of the second solve's inputs
    noise = b.noise_samples_d.copy_to_host()[:256]
    gl, ga = blin.sample_grid_batch_d.copy_to_host()[:8], bang.sample_grid_batch_d.copy_to_host()[:8]
    want = oracle_rollout_costs(sc, blin, bang, noise, u1, grids=(gl, ga), arith=dev, ctrl_order="presummed",
                                wrap_clamp=True)                              # u1 was the warm start of solve 2
    assert_all_equal(b.costs_nm_d.copy_to_host()[:256, :8], want, "config 5 slice")


def test_determinism_and_checkpoint_resume(eng):
    sc = make_scenario("tdm", N=256, M=16, T=32, H=100, W=100, res=0.2, B=8, seed=6)
    a = tdm_planner(eng, sc)
    b = tdm_planner(eng, sc)
    ua = [a.solve() for _ in range(3)]
    ub = [b.solve() for _ in range(2)]
    assert (ua[0] == ub[0]).all() and (ua[1] == ub[1]).all()     # same seed -> bit-identical, run to run
    st = b.get_state()
    c = tdm_planner(eng, sc)
    c.set_state(st)
    assert (c.solve() == ua[2]).all()                            # resume from checkpoint == uninterrupted
    assert not (ua[0] == ua[1]).all()                            # streams advance between solves


def test_oversized_map_count_solve(eng, capsys):
    """num_grid_samples > 1024: solve() dispatches to solve_stochastic_oversized (mppi.py:199-203) and equals
    the stage-by-stage replay through the C-ABI, whose CVaR stage is checked against the oracle's sort."""
    sc = make_scenario("tdm", N=128, M=1030, T=16, H=40, W=40, res=0.25, B=6, seed=21, cvar_alpha=0.3)
    a = tdm_planner(eng, sc)
    assert "oversized kernel" in capsys.readouterr().out          # Config's warning, like the reference's
    assert a.cfg.num_grid_samples == 1030
    u = a.solve()
    assert u.shape == (16, 2) and np.isfinite(u).all()
    b = staged_rollout(eng, sc)
    L = eng._lib
    nm = b.costs_nm_d.copy_to_host()
    cv = b.costs_d.copy_to_host()
    RB.check_cvar(cv, nm, 0.3, label="oversized")
    c = np.ascontiguousarray(cv)
    L.check(L.lib.b200mppi_planner_update(b._handle, L.ptr(c)))
    assert (b.u_cur_d.copy_to_host() == u).all()


def test_closed_loop_reaches_goal(eng):
    """The reference's test.ipynb scenario in miniature: receding-horizon loop on the mean-traction map
    until the goal tolerance is met (SURVEY.md section 4-iv)."""
    sc = make_scenario("det", N=512, M=1, T=40, H=60, W=60, res=0.25, B=6, seed=12, mask_p=0.0)
    p = dict(sc["params"])
    p["x0"] = np.array([3.0, 3.0, 0.0])
    p["xgoal"] = np.array([10.0, 10.0])
    p["num_opt"] = 2
    pl = tdm_planner(eng, dict(sc, obstacle=None, unknown=None), params=p)     # no masks
    bv = pl.lin_tdm.bin_values
    mean_l = (sc["pmf_lin"].astype(float) * bv[:, None, None]).sum(0) / 100
    mean_a = (sc["pmf_ang"].astype(float) * bv[:, None, None]).sum(0) / 100
    world = eng.TractionGrid(mean_l, mean_a, res=0.25)
    x = p["x0"].copy()
    reached = False
    for _ in range(150):
        u = pl.solve()
        lt, at = world.get(x[0], x[1])
        x = x + 0.1 * np.array([lt * u[0, 0] * np.cos(x[2]), lt * u[0, 0] * np.sin(x[2]), at * u[0, 1]])
        if np.hypot(*(x[:2] - p["xgoal"])) <= 0.5:
            reached = True
            break
        pl.shift_and_update(x, u, 1)
    assert reached, "closed loop did not reach the goal; final state %s" % x


# ----------------------------------------------------------------------------- reach-box map sampling
@pytest.mark.parametrize("N,M,T,H,res,warm,tdim,diverge", [
    # BASELINE config 3
    pytest.param(1024, 64, 64, 512, 0.1, False, (16, 16), False, id="1024-64-64-512-0.1-False-tdim0"),
    # ragged tiles, warm start (longer reach), 40 maps: partial map groups
    pytest.param(512, 40, 64, 420, 0.1, True, (7, 5), False, id="512-40-64-420-0.1-True-tdim1"),
    # the speed-limit box (4.8 m) leaves the 10 m map, the actual reach does not
    pytest.param(256, 16, 16, 200, 0.05, True, (4, 12), False, id="256-16-16-200-0.05-True-tdim2"),
    # lin's stream ahead of ang's: each TDM sampled (and boxed) on its own
    pytest.param(512, 40, 64, 420, 0.1, True, (7, 5), True, id="512-40-64-420-0.1-True-tdim1-diverged"),
])
def test_boxed_solve_identical_to_whole_map_solve(eng, monkeypatch, N, M, T, H, res, warm, tdim, diverge):
    """solve() samples only the cells its rollouts can reach (include/b200mppi.h, b200mppi_planner_sample_box).
    Against whole-map sampling (what the reference does, terrain.py:610-694) over a closed loop with a moving
    robot: u, CVaR costs, per-(n,m) costs, noise and EVERY generator state bit-identical; afterwards the sampled
    maps read through the public handle are the whole maps of that sampling call (completed on demand).
    With `diverge`, one public lin.sample_grids() before the loop leaves the two TDMs in different generator states,
    so the maps are not sampled from one stream but one TDM at a time."""
    sc = make_scenario("tdm", N=N, M=M, T=T, H=H, W=H, res=res, B=12, seed=11, warm_start=warm, thread_dim=tdim)
    runs = {}
    for box in ("off", "static", "dynamic"):
        pl = tdm_planner(eng, sc, box=box, monkeypatch=monkeypatch)
        lin, ang = pl.lin_tdm, pl.ang_tdm
        if diverge:
            lin.sample_grids(sc["params"]["alpha_dyn"])
        x0 = sc["params"]["x0"].copy()
        hist, modes, launches = [], [], []
        for k in range(4):
            l0 = pl.launch_count()
            u = pl.solve()
            launches.append(pl.launch_count() - l0)
            modes.append(pl.sample_box())
            hist.append(dict(u=u.copy(), costs=pl.costs_d.copy_to_host(), costs_nm=pl.costs_nm_d.copy_to_host()))
            x0 = x0 + np.array([0.37, -0.21, 0.05])
            pl.shift_and_update(x0, u, 1)
        runs[box] = dict(hist=hist, modes=modes, launches=launches,
                         state=dict(lin_rng=lin.rng_states_d.copy_to_host(), ang_rng=ang.rng_states_d.copy_to_host(),
                                    rng=pl.rng_states_d.copy_to_host(), noise=pl.noise_samples_d.copy_to_host(),
                                    lin_grid=lin.sample_grid_batch_d.copy_to_host(),
                                    ang_grid=ang.sample_grid_batch_d.copy_to_host()))
    ref = runs["off"]
    assert all(m[0] == 0 for m in ref["modes"])
    # a box that would leave the map is not used (whole maps); the box from the controls is the tighter one.
    # speed-limit box of the FIRST solve (reach_radius, kernels.h): R = dt * max|traction| * T * vmax * 1.0002 plus the
    # float32 rounding of the state and of the cell index
    pad = int(np.ceil(5.0 * 0.1 / res))
    c0 = sc["params"]["x0"][:2].astype(np.float32).astype(np.float64)
    u, pxl = 5.9605e-8, float(np.float32(-pad * res))
    D = (0.1 * 1.0 * T * 3.0 * 1.0002 + T * u * np.abs(c0).sum()) / (1 - T * u)
    R = D + u * (np.abs(c0 - pxl).sum() + 2 * D)
    static_fits = all((c - R + pad * res) / res > 2.0 and (c + R + pad * res) / res < H + 2 * pad - 3.0 for c in c0)
    assert runs["static"]["modes"][0][0] == (1 if static_fits else 0), runs["static"]["modes"]
    assert all(m[0] in (0, 1) for m in runs["static"]["modes"])
    assert all(m[0] == 2 for m in runs["dynamic"]["modes"]), runs["dynamic"]["modes"]
    # launches per solve: noise + controls, rollout, CVaR, update, and the sampler -- one launch for both maps when the
    # TDMs share a stream, one per TDM otherwise -- each followed, when boxed, by its generator-state advance
    samplers = 2 if diverge else 1
    for box in ("off", "static", "dynamic"):
        r = runs[box]
        assert r["launches"] == [4 + samplers * (2 if m[0] else 1) for m in r["modes"]], (box, r["launches"])
    if not diverge:
        assert runs["dynamic"]["launches"] == [6] * 4                 # README: a stochastic solve is 6 launches
    Hp = H + 2 * int(np.ceil(5.0 * 0.1 / res))
    for box in ("static", "dynamic"):
        r = runs[box]
        for k, (h, h0) in enumerate(zip(r["hist"], ref["hist"])):
            assert_same(h, h0, "box %s, solve %d" % (box, k))
        assert_same(r["state"], ref["state"], "box %s" % box)
    # the dynamic box is the smaller one, and a real restriction
    ms, md = runs["static"]["modes"][-1], runs["dynamic"]["modes"][-1]
    area = lambda m: (m[2] - m[1]) * (m[4] - m[3])
    assert area(md) < Hp * Hp
    if ms[0]:
        assert area(md) <= area(ms) < Hp * Hp


def test_boxed_solve_falls_back_near_the_map_edge_and_for_several_iterations(eng, monkeypatch):
    """The reach box must lie strictly inside the map (out-of-map indices wrap); num_opt > 1 cannot use this
    solve's controls (the maps are sampled once for several noise draws) and takes the static bound."""
    sc = make_scenario("tdm", N=256, M=16, T=32, H=200, W=200, res=0.1, B=12, seed=5, thread_dim=(4, 4))
    sc["params"]["x0"] = np.array([1.0, 10.0, 0.3])                 # 10 cells from the left edge: reach > 10 cells
    pl = tdm_planner(eng, sc, box="dynamic", monkeypatch=monkeypatch)
    assert pl.solve() is not None
    assert pl.sample_box()[0] == 0
    sc["params"]["x0"] = np.array([10.0, 10.0, 0.3])
    sc["params"]["num_opt"] = 2
    sc["params"]["vrange"] = np.array([0.0, 1.0])                   # static reach 3.2 m = 32 cells: inside the 20 m map
    pl = tdm_planner(eng, sc, box="dynamic", monkeypatch=monkeypatch)
    u = pl.solve()
    assert pl.sample_box()[0] == 1
    pl2 = tdm_planner(eng, sc, box="off", monkeypatch=monkeypatch)
    u2 = pl2.solve()
    lin, lin2 = pl.lin_tdm, pl2.lin_tdm
    assert_same(dict(u=u2, lin_map=lin2.sample_grid_batch_d.copy_to_host(), lin_rng=lin2.rng_states_d.copy_to_host()),
                dict(u=u, lin_map=lin.sample_grid_batch_d.copy_to_host(), lin_rng=lin.rng_states_d.copy_to_host()),
                "whole maps against the static box")


def test_state_rollout_and_public_sampling_after_boxed_solve(eng, monkeypatch):
    """Everything that reads the sampled maps outside solve() sees whole maps: get_state_rollout(), a following
    public sample_grids() (fresh whole maps, streams continue), the stage-level rollout entry point."""
    sc = make_scenario("tdm", N=256, M=16, T=48, H=240, W=240, res=0.1, B=12, seed=9, thread_dim=(5, 6))
    out = {}
    for box in ("off", "dynamic"):
        pl = tdm_planner(eng, sc, box=box, monkeypatch=monkeypatch)
        lin, ang = pl.lin_tdm, pl.ang_tdm
        pl.solve()
        if box == "dynamic":
            assert pl.sample_box()[0] == 2
        st = pl.get_state_rollout()
        from mppi_numba_b200._lib import lib, check
        check(lib.b200mppi_planner_rollout(pl._handle))                # re-rolls the same noise on the same maps
        cnm = pl.costs_nm_d.copy_to_host()
        pl.solve()                                                      # boxed again
        g2 = lin.sample_grids(1.0).copy_to_host()                       # public call: whole fresh maps
        out[box] = dict(state_rollout=st, costs_nm=cnm, lin_map=g2, ang_rng=ang.rng_states_d.copy_to_host(),
                        lin_rng=lin.rng_states_d.copy_to_host())
    assert_same(out["off"], out["dynamic"], "after a boxed solve")


def test_sampler_wide_thread_tiles(eng):
    """tdm_sample_thread_dim with more than 32 tile columns (Config only bounds the product): the staged sampler
    runs fewer maps per CTA instead of exceeding its launch bound (ADVICE r1), up to 256 columns; wider tiles use
    the generic kernel.  Bit-exact against the oracle either way, streams included."""
    for tdim, M in (((4, 64), 5), ((1, 40), 9), ((2, 300), 2)):
        H = W = 320
        sc = make_scenario("tdm", N=128, M=M, T=8, H=H, W=W, res=0.5, B=12, seed=21, thread_dim=tdim)
        cfg = eng.Config(**sc["cfg"])
        lin = eng.TDM_Numba(cfg)
        lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        got = lin.sample_grids(1.0).copy_to_host()
        want = np.zeros_like(got)
        st = X.create_states(tdim[0] * tdim[1] * M, cfg.seed)
        TR.sample_grids(want, lin.pmf_grid_d.copy_to_host(), st, lin.bin_values, lin.bin_values_bounds, 1.0, tdim, M)
        assert (got == want).all(), tdim
        assert (lin.rng_states_d.copy_to_host() == st).all(), tdim
