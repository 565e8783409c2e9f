"""The generic rollout kernels' and the visualisation kernel's real source, executed on the host by
tests/emu_rollout.py, against what the REFERENCE's own kernels returned for the same inputs (tests/golden, produced
by the unmodified reference under Numba's simulator): per-(n,m) costs of the stochastic kernel, costs of the
deterministic and speed-map kernels (near goal = early exits, far goal), the barebone notebook kernel, and the
state sequences of get_state_rollout for the three modes."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.emu_rollout import build

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F32 = np.float32


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build(str(tmp_path_factory.mktemp("emu_rollout")))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def _fparams(res, xlo, ylo, dt, x0, goal, tol, v_post, lam, u_std, vr, wr, obs_c, unk_c, dist_w, lin_lo, ang_lo):
    return _c([res, xlo, ylo, dt, x0[0], x0[1], x0[2], goal[0], goal[1], tol, v_post, lam, u_std[0], u_std[1], vr[0], vr[1],
               wr[0], wr[1], obs_c, unk_c, dist_w, lin_lo, ang_lo], F32)


def _ratios(lb, ab):
    return _c([0.01 * np.float64(F32(F32(lb[1]) - F32(lb[0]))), 0.01 * np.float64(F32(F32(ab[1]) - F32(ab[0])))], np.float64)


@pytest.mark.parametrize("gname", ["near", "far"])
def test_rollout_kernels_match_reference(emu, gname):
    g = np.load(os.path.join(GOLDEN, "ref_rollout.npz"))
    lin, ang = _c(g["lin"], np.int8), _c(g["ang"], np.int8)
    obs, unk, risk = _c(g["obs"], np.int8), _c(g["unk"], np.int8), _c(g["risk"][0], np.int8)
    noise, u_cur = _c(g["noise"], F32), _c(g["u_cur"], F32)
    M, R, Cc = lin.shape
    Hp, Wp = obs.shape
    N, T = noise.shape[:2]
    goal = g["xgoal_" + gname]
    f = _fparams(g["res"], g["xlim"][0], g["ylim"][0], g["dt"], g["x0"], goal, g["goal_tol"], g["v_post"], g["lam"],
                 g["u_std"], g["vrange"], g["wrange"], g["obs_cost"], g["unk_cost"], g["dist_weight"],
                 g["lin_bounds"][0], g["ang_bounds"][0])
    ratios = _ratios(g["lin_bounds"], g["ang_bounds"])

    def launch(mode, Mk):
        geo = _c([Hp, Wp, R, Cc, Cc, Wp, T, N, Mk], np.int32)
        cnm, costs = np.zeros((N, Mk), F32), np.zeros(N, F32)
        emu.emu_rollout(mode, _p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), _p(risk), _p(noise),
                        _p(u_cur), _p(cnm), _p(costs), None, 0)
        return cnm, costs
    cnm, _ = launch(0, M)
    ref = g["sto_cnm_" + gname]
    assert (np.abs(cnm - ref) / np.maximum(np.abs(ref), 1e-6)).max() < 3e-6
    _, det = launch(1, 1)
    np.testing.assert_allclose(det, g["det_" + gname], rtol=3e-6)
    _, spd = launch(2, 1)
    np.testing.assert_allclose(spd, g["spd_" + gname], rtol=3e-6)
    # and every cost equals the exact oracle (libm provider: what the emulation substitutes for the MUFU operations)
    from oracle import mppi_ref as MR
    from tests.test_exact_oracle_cpu import EXACT, assert_equal
    for mode, got in ((MR.MODE_STOCHASTIC, cnm), (MR.MODE_DET_DYN, det[:, None]), (MR.MODE_SPEED_MAP, spd[:, None])):
        want = MR.rollout_costs(mode, lin, ang, g["lin_bounds"], g["ang_bounds"], obs, unk, F32(g["res"]), g["xlim"],
                                g["ylim"], g["vrange"], g["wrange"], goal, g["v_post"], g["obs_cost"], g["unk_cost"],
                                g["goal_tol"], g["lam"], g["u_std"], g["x0"], g["dt"], g["dist_weight"], noise, u_cur,
                                risk_map=risk[None], arith=EXACT)
        assert_equal(got, want, "mode %d" % mode)
    if gname == "near":
        assert (cnm < 50).any() and (cnm > 50).any()        # the early-exit branch is exercised


@pytest.mark.parametrize("gname", ["near", "far"])
def test_barebone_kernel_matches_reference_notebook(emu, gname):
    g = np.load(os.path.join(GOLDEN, "ref_barebone.npz"))
    noise, u_cur = _c(g["noise"], F32), _c(g["u_cur"], F32)
    N, T = noise.shape[:2]
    f = _fparams(1.0, 0.0, 0.0, g["dt"], g["x0"], g["goal_" + gname], g["goal_tol"], 0.0, g["lam"], g["u_std"], g["vrange"],
                 g["wrange"], g["obs_cost"], 0.0, g["dist_weight"], 0.0, 0.0)
    geo = _c([1, 1, 1, 1, 1, 1, T, N, 1], np.int32)
    ob = _c(np.concatenate([np.asarray(g["obs_pos"]).reshape(-1, 2), np.asarray(g["obs_r"]).reshape(-1, 1)], axis=1), F32)
    costs = np.zeros(N, F32)
    emu.emu_rollout(3, _p(f), _p(geo), _p(_c([0.01, 0.01], np.float64)), None, None, None, None, None, _p(noise), _p(u_cur),
                    None, _p(costs), _p(ob), ob.shape[0])
    np.testing.assert_allclose(costs, g["costs_" + gname], rtol=3e-6)
    from oracle import mppi_ref as MR
    from tests.test_exact_oracle_cpu import EXACT
    want = MR.rollout_costs_barebone(g["obs_pos"], g["obs_r"], g["vrange"], g["wrange"], g["goal_" + gname], g["obs_cost"],
                                     g["goal_tol"], g["lam"], g["u_std"], g["x0"], g["dt"], g["dist_weight"], noise, u_cur,
                                     arith=EXACT)
    assert (costs.view(np.uint32) == want.view(np.uint32)).all(), int((costs != want).sum())


@pytest.mark.parametrize("mode", ["tdm", "det", "spd"])
def test_state_rollout_kernel_matches_reference(emu, mode):
    g = np.load(os.path.join(GOLDEN, "ref_state_rollout.npz"))
    lin, ang = _c(g[mode + "_lin_grid"], np.int8), _c(g[mode + "_ang_grid"], np.int8)
    noise, u_cur, u_prev = _c(g[mode + "_noise"], F32), _c(g[mode + "_u_cur"], F32), _c(g[mode + "_u_prev"], F32)
    V = int(g[mode + "_V"])
    T = u_cur.shape[0]
    Mm, R, Cc = lin.shape
    b = g["bounds"]
    f = _fparams(g["res"], F32(g[mode + "_pxl"][0]), F32(g[mode + "_pyl"][0]), g["dt"], g["x0"], [0, 0], 0.0, 1.0, 1.0,
                 [1, 1], g["vrange"], g["wrange"], 0.0, 0.0, 1.0, b[0], b[0])
    geo = _c([R, Cc, R, Cc, Cc, Cc, T, noise.shape[0], Mm], np.int32)
    out = np.zeros((V, T + 1, 3), F32)
    emu.emu_state_rollout(0 if mode == "tdm" else 1, V, _p(f), _p(geo), _p(_ratios(b, b)), _p(lin), _p(ang), _p(noise),
                          _p(u_cur), _p(u_prev), _p(out))
    np.testing.assert_allclose(out, g[mode + "_states"], rtol=3e-6, atol=3e-6)
    from oracle import mppi_ref as MR
    from tests.test_exact_oracle_cpu import EXACT
    want = MR.state_rollouts(dict(tdm=MR.MODE_STOCHASTIC, det=MR.MODE_DET_DYN, spd=MR.MODE_SPEED_MAP)[mode], V, lin, ang, b, b,
                             g["res"], [F32(g[mode + "_pxl"][0]), 0], [F32(g[mode + "_pyl"][0]), 0], g["x0"], g["dt"], u_cur,
                             u_prev, noise, g["vrange"], g["wrange"], arith=EXACT)
    assert (out.view(np.uint32) == want.view(np.uint32)).all(), int((out != want).sum())
