"""Pin the oracle (oracle/*.py) against outputs of the reference's own kernels
(tests/golden/ref_*.npz, produced by oracle/make_golden.py under Numba's CUDA simulator)."""
import os

import numpy as np
import pytest

from oracle import xoroshiro as X
from oracle import terrain_ref as TR
from oracle import mppi_ref as MR


def load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name), allow_pickle=False)


# ----------------------------------------------------------------------------- RNG
def test_xoroshiro_known_answers():
    """KATs of numba 0.65.0's generator (SURVEY.md 8c)."""
    st = X.create_states(4, 1)
    exp = [(0x910a2dec89025cc1, 0x910a2dec89025cc1), (0x73c19a5348fc9098, 0x6c96c932f21d71ee),
           (0x0b3d0cd6ddfa7a4c, 0xd3c2c33e9b8e707a), (0x3b80c389fcd31ee7, 0xb43c70624d182bbb)]
    assert [(int(a), int(b)) for a, b in st] == exp
    s = st[:1].copy()
    outs = [int(X.next_u64(s)[0]) for _ in range(4)]
    assert outs == [0x22145bd91204b982, 0x60c88516f644812e, 0x3b056fab69fc74dd, 0x75dde50d5f276a45]
    u = X.uniform_float32(np.array(outs, dtype=np.uint64))
    np.testing.assert_allclose(u, [0.13312314, 0.37805969, 0.23055170, 0.46041709], rtol=1e-7)


def test_create_states_doubling_equals_sequential():
    big = X.create_states(300, 5)
    z = X.splitmix64(5)
    s = (z, z)
    for i in range(300):
        assert (int(big[i, 0]), int(big[i, 1])) == s
        s = X.jump_scalar(*s)


def test_noise_matches_reference(golden_dir):
    g = load(golden_dir, "ref_noise.npz")
    N, T = int(g["N"]), int(g["T"])
    st = X.create_states(N * T, int(g["seed"]))
    assert (st == g["states0"]).all()
    n1 = MR.sample_noise(st, g["u_std"], N, T)
    n2 = MR.sample_noise(st, g["u_std"], N, T)
    assert (st == g["states2"]).all()                    # integer stream: bit exact
    np.testing.assert_allclose(n1, g["noise1"], rtol=2e-6, atol=1e-6)
    np.testing.assert_allclose(n2, g["noise2"], rtol=2e-6, atol=1e-6)
    assert abs(float(n1[0, 0, 0]) - (-2.8941278)) < 1e-5  # SURVEY.md 8c KAT


# ----------------------------------------------------------------------------- terrain
@pytest.mark.parametrize("mode", ["tdm", "det", "spd"])
@pytest.mark.parametrize("alpha", [0.3, 1.0])
def test_pmf_setter_and_sampling_match_reference(golden_dir, mode, alpha):
    g = load(golden_dir, "ref_terrain.npz")
    key = "%s_a%02d" % (mode, int(alpha * 10))
    mmd = tuple(int(v) for v in g["max_map_dim"])
    pmf = g["pmf_lin"]
    if mode == "det":
        pmf_use = TR.collapse_pmf_det_dynamics(pmf, g["bin_values"], alpha)
    elif mode == "spd":
        pmf_use, risk = TR.risk_traction_map(pmf, g["bin_values"], g["bounds"], alpha)
        risk_p = TR.set_padding_2d(risk[0], float(g["max_speed_padding"]), float(g["dt"]), float(g["res"]), mmd)
        assert (risk_p[None] == g[key + "_risk"]).all()
    else:
        pmf_use = pmf.astype(np.int8)
    padded, pxl, pyl, pad = TR.set_padding(pmf_use, float(g["max_speed_padding"]), float(g["dt"]),
                                           float(g["res"]), g["xlimits"], g["ylimits"], mmd)
    assert pad == int(g[key + "_pad"])
    assert (padded == g[key + "_pmf_padded"]).all()
    np.testing.assert_allclose(pxl, g[key + "_pxl"])
    np.testing.assert_allclose(pyl, g[key + "_pyl"])
    obs_p = TR.set_padding_2d(g["obstacle"], float(g["max_speed_padding"]), float(g["dt"]), float(g["res"]), mmd)
    assert (obs_p == g[key + "_obs_padded"]).all()

    # sampling: two consecutive calls (alpha_dyn 1.0 then 0.6), bit exact incl. the RNG stream
    det_dyn = mode != "tdm"
    M = 1 if det_dyn else int(g["M"])
    td = tuple(int(v) for v in g["thread_dim"])
    st = TR.sample_rng_states(int(g["seed"]), int(g["M"]), td, det_dyn)
    assert (st == g[key + "_states0"]).all()
    grid = np.zeros((M,) + mmd, dtype=np.int8)
    TR.sample_grids(grid, padded, st, g["bin_values"], g["bounds"], 1.0, td, M)
    assert (grid == g[key + "_grid1"]).all()
    TR.sample_grids(grid, padded, st, g["bin_values"], g["bounds"], 0.6, td, M)
    assert (grid == g[key + "_grid2"]).all()
    assert (st == g[key + "_states2"]).all()


def test_quantise_compiled_typing():
    """SURVEY.md 9-N4 / 8c-iv: compiled float64 truncation, 0.21f -> 20, 0.7f -> 69, 1/11 -> 9."""
    q = TR.quantise_bin_values([0.0, 0.21, 0.525, 0.7, 1.0], [0.0, 1.0])
    assert q.tolist() == [0, 20, 52, 69, 100]
    q = TR.quantise_bin_values(np.linspace(0, 1, 12), [0.0, 1.0])
    assert q[1] == 9


# ----------------------------------------------------------------------------- rollouts
def _rollout(g, mode, goal, grids_l, grids_a):
    return MR.rollout_costs(mode, grids_l, grids_a, g["lin_bounds"], g["ang_bounds"], g["obs"], g["unk"],
                            g["res"], g["xlim"], g["ylim"], g["vrange"], g["wrange"], goal, g["v_post"],
                            g["obs_cost"], g["unk_cost"], g["goal_tol"], g["lam"], g["u_std"], g["x0"],
                            g["dt"], g["dist_weight"], g["noise"], g["u_cur"], risk_map=g["risk"])


@pytest.mark.parametrize("gname", ["near", "far"])
def test_rollouts_match_reference(golden_dir, gname):
    g = load(golden_dir, "ref_rollout.npz")
    goal = g["xgoal_" + gname]
    cnm = _rollout(g, MR.MODE_STOCHASTIC, goal, g["lin"], g["ang"])
    ref = g["sto_cnm_" + gname]
    rel = np.abs(cnm - ref) / np.maximum(np.abs(ref), 1e-6)
    assert rel.max() < 2e-6, rel.max()
    for alpha in (0.5, 0.9, 1.0):
        cv = MR.cvar_reduce(cnm, alpha)
        refc = g["sto_cvar%02d_%s" % (int(alpha * 10), gname)]
        np.testing.assert_allclose(cv, refc, rtol=2e-6)
    det = _rollout(g, MR.MODE_DET_DYN, goal, g["lin"][:1], g["ang"][:1])[:, 0]
    np.testing.assert_allclose(det, g["det_" + gname], rtol=2e-6)
    spd = _rollout(g, MR.MODE_SPEED_MAP, goal, g["lin"][:1], g["ang"][:1])[:, 0]
    np.testing.assert_allclose(spd, g["spd_" + gname], rtol=2e-6)


@pytest.mark.parametrize("gname", ["near", "far"])
def test_oversized_kernel_mean_matches_reference(golden_dir, gname):
    """rollout_oversized_numba (mppi.py:760-913; num_grid_samples > threads per block, several maps per thread)
    at cvar_alpha = 1, its only meaningful setting (SURVEY.md 9-B1: for alpha < 1 it swaps unconditionally and
    indexes shared memory out of bounds): the oracle's mean over the M per-map costs is what it returns."""
    g = load(golden_dir, "ref_rollout.npz")
    o = load(golden_dir, "ref_oversized.npz")
    cnm = _rollout(g, MR.MODE_STOCHASTIC, g["xgoal_" + gname], g["lin"], g["ang"])
    np.testing.assert_allclose(MR.cvar_reduce(cnm, 1.0), o["over_a10_" + gname], rtol=2e-6)


@pytest.mark.parametrize("mode", ["tdm", "det", "spd"])
def test_state_rollouts_match_reference(golden_dir, mode):
    """get_state_rollout (mppi.py:545-608, kernels :1194-1351) after a solve of the reference, three modes."""
    g = load(golden_dir, "ref_state_rollout.npz")
    m = dict(tdm=MR.MODE_STOCHASTIC, det=MR.MODE_DET_DYN, spd=MR.MODE_SPEED_MAP)[mode]
    got = MR.state_rollouts(m, int(g[mode + "_V"]), g[mode + "_lin_grid"], g[mode + "_ang_grid"], g["bounds"],
                            g["bounds"], g["res"], g[mode + "_pxl"], g[mode + "_pyl"], g["x0"], g["dt"],
                            g[mode + "_u_cur"], g[mode + "_u_prev"], g[mode + "_noise"], g["vrange"], g["wrange"])
    ref = g[mode + "_states"]
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, rtol=2e-6, atol=2e-6)
    if mode != "tdm":
        assert not np.allclose(ref[0], ref[1])          # block 0 = optimal sequence, the others are noisy samples


def test_near_goal_case_exercises_early_exit(golden_dir):
    g = load(golden_dir, "ref_rollout.npz")
    # a reached rollout has no terminal cost: far smaller than dist/v_post of the others
    assert (g["sto_cnm_near"] < 50).any() and (g["sto_cnm_near"] > 50).any()


def test_cvar_count_float32_alpha():
    assert MR.cvar_count(10, 0.1) == 2          # SURVEY.md 9-N3
    assert MR.cvar_count(256, 0.5) == 128
    assert MR.cvar_count(6, 1.0) == 6


# ----------------------------------------------------------------------------- update
@pytest.mark.parametrize("lam", [1.0, 0.3])
def test_update_matches_reference(golden_dir, lam):
    g = load(golden_dir, "ref_update.npz")
    u, w = MR.update_useq(lam, g["costs"], g["noise"], g["vrange"], g["wrange"], g["u0"])
    np.testing.assert_allclose(w, g["w_lam%02d" % int(lam * 10)], rtol=2e-5, atol=1e-9)
    np.testing.assert_allclose(u, g["u_lam%02d" % int(lam * 10)], rtol=1e-5, atol=2e-6)


def test_shift_keeps_tail():
    u = np.arange(10, dtype=np.float32).reshape(5, 2)
    s = MR.shift_useq(u, 2)
    assert (s[:3] == u[2:]).all() and (s[3:] == u[3:]).all()


# ----------------------------------------------------------------------------- barebone (map-free) variant
@pytest.mark.parametrize("gname", ["near", "far"])
def test_barebone_rollout_matches_reference_notebook(golden_dir, gname):
    g = load(golden_dir, "ref_barebone.npz")
    c = MR.rollout_costs_barebone(g["obs_pos"], g["obs_r"], g["vrange"], g["wrange"], g["goal_" + gname], g["obs_cost"],
                                  g["goal_tol"], g["lam"], g["u_std"], g["x0"], g["dt"], g["dist_weight"], g["noise"],
                                  g["u_cur"])
    np.testing.assert_allclose(c, g["costs_" + gname], rtol=3e-6)
    if gname == "near":
        assert (g["costs_near"] < 0.1 * np.median(g["costs_far"])).any()      # early exits exercised


def test_barebone_state_rollouts_match_reference_notebook(golden_dir):
    """The notebook's get_state_rollout after its first solve (cfg T 1.0, dt 0.1, N 100, V 5; x0 (0, 0, pi/4)).  Its
    solve aliases u_prev_d to u_cur_d, so both are the solve's result solve_u1; the noise is that solve's draw."""
    g = load(golden_dir, "ref_barebone.npz")
    ref = g["solve_states1"]
    u1 = g["solve_u1"]
    got = MR.state_rollouts_barebone(ref.shape[0], [0.0, 0.0, np.pi / 4], 0.1, u1, u1, g["solve_noise1"], [0.0, 2.0],
                                     [-np.pi, np.pi])
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, rtol=2e-6, atol=2e-6)
    assert not np.allclose(ref[0], ref[1])              # row 0 = the optimal sequence, the others noisy samples
    # the noisy rows are clipped: without the clip (or without the noise) they differ from the notebook's
    raw = MR.state_rollouts_barebone(ref.shape[0], [0.0, 0.0, np.pi / 4], 0.1, u1, u1, g["solve_noise1"], [-1e9, 1e9],
                                     [-1e9, 1e9])
    assert not np.allclose(raw[1:], ref[1:], rtol=2e-6, atol=2e-6)
