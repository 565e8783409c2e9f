"""Kernel-by-kernel parity against the UNMODIFIED reference's Numba-CUDA kernels running on the same GPU.

The reference cannot be committed to this repository; build() compiles it to git-ignored bytecode under
oracle/_ref/ where its sources are readable (oracle/ref_build.py).  When that was not built the tests skip.
What is asserted (same inputs on both sides: seed, PMFs, masks, params):
  * control noise: bit-identical;  sampled traction maps: bit-identical
  * det-dynamics and speed-map rollout costs: bit-identical, also with a nonzero lower traction bound on inputs where
    fusing lo + ratio*q (and the state's dv*cos + x) into one FMA decides the goal flag, and where fusing the speed
    map's lo + ratio*risk decides the time step -- what pins the exact oracle's FMAs; the speed map with bin values
    outside the traction bounds (its risk bytes truncated and wrapped)
  * the batched one-map kernels (MPPI_Batch of speed-map planners, MPPI_MixedBatch of det-dynamics and speed-map
    planners): every planner's costs bit-identical to the reference kernel's on that planner's noise and controls
  * visualisation rollouts (get_state_rollout of one planner and of a batch, V across the 32-thread blocks): every
    state bit-identical, for det dynamics, speed map and use_tdm, and on the directed boundary cases
  * the map-free notebook (barebone_mppi_numba.ipynb) kernels: costs and visualisation states bit-identical over the
    edge-case sweep of tests/barebone_edge_cases.py and its directed obstacle / goal boundaries
  Every trajectory compared bit for bit stays inside the padded map (asserted from the oracle's states), so no
  comparison depends on the engine's documented rule for cells outside it.
  * stochastic CVaR costs: within the CVaR kernel's bound plus the reference's pairwise tree's bound
    (tests/reduce_bounds.py), around the exact mean of the engine's per-(n, m) costs, plus the rounding of adding the
    control cost step by step (the reference) instead of pre-summed (the windowed kernel); including M > 1024
    against the reference's oversized kernel at cvar_alpha = 1
  * updated control sequence given the reference's costs: within 1e-4
"""
import io
import contextlib
import os
import sys

import numpy as np
import pytest

from tests import barebone_edge_cases as BE
from tests.gpu_harness import assert_all_equal, dev, directed_oracle, eng, quiet, run_directed, tdm_planner  # noqa: F401

pytestmark = pytest.mark.gpu
f32 = np.float32


def _quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


@pytest.fixture(scope="module")
def ref():
    from oracle.ref_build import compiled_reference
    root = compiled_reference()
    if root is None:
        pytest.skip("compiled reference not available (oracle/_ref absent)")
    if os.environ.get("NUMBA_ENABLE_CUDASIM") == "1":
        pytest.skip("numba is in simulator mode in this process")
    np.float = float                      # mppi.py:32-33 uses the removed alias
    if root not in sys.path:
        sys.path.insert(0, root)
    try:
        from numba import cuda
        if not cuda.is_available():
            pytest.skip("numba sees no CUDA device")
        from mppi_numba.config import Config
        from mppi_numba.terrain import TDM_Numba
        from mppi_numba.mppi import MPPI_Numba
    except Exception as e:                # numba / driver mismatch: not a failure of this repository
        pytest.skip("reference could not be imported on this GPU: %r" % (e,))
    return Config, TDM_Numba, MPPI_Numba, cuda


def OUTSIDE_BOUNDS(B):
    """Bin values of a speed-map scenario outside its traction bounds [0, 1] (the last, the nominal bin, at 1): risk
    bytes below 0 truncate towards 0, above 127 wrap, as the reference's astype(np.int8) does."""
    return np.r_[0.0, np.linspace(-0.9, 2.6, B - 2), 1.0]


def ref_planner(ref, sc):
    """The reference's MPPI_Numba of a scenario (tests/scenarios.make_scenario), set up as tests/gpu_harness.tdm_planner
    sets up the engine's: its TDMs are .lin_tdm and .ang_tdm, u_cur from sc["u0"] when the scenario has one."""
    RConfig, RTDM, RMPPI, cuda = ref
    rcfg = _quiet(RConfig, **sc["cfg"])
    rl, ra = _quiet(RTDM, rcfg), _quiet(RTDM, rcfg)
    _quiet(rl.set_TDM_from_PMF_grid, sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    _quiet(ra.set_TDM_from_PMF_grid, sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    rp = _quiet(RMPPI, rcfg)
    rp.setup(sc["params"], rl, ra)
    if "u0" in sc:
        rp.u_cur_d = cuda.to_device(sc["u0"])
    return rp


def one_map_rollout(ref, rp, mode, lin_g, ang_g, noise_d, u_d, costs_d):
    """rollout_det_dyn_numba ("det") or rollout_det_dyn_w_speed_map_numba ("spd") of planner rp on the given sampled
    maps, noise and controls, with the arguments (and so the types Numba specialises on) of solve_det_dyn /
    solve_nom_dyn_w_speed_map (mppi.py:245-291, 317-361)."""
    RMPPI = ref[2]
    (res_d, xl_d, yl_d, vr_d, wr_d, xg_d, vpost_d, tol_d, lam_d, ustd_d, _, x0_d, dt_d, obs_c, unk_c) = \
        rp.move_mppi_task_vars_to_device()
    dist_weight = 1.0 if "dist_weight" not in rp.params else rp.params["dist_weight"]
    rl, ra = rp.lin_tdm, rp.ang_tdm
    tail = (rl.bin_values_bounds_d, ra.bin_values_bounds_d, rl.obstacle_map_d, rl.unknown_map_d, res_d, xl_d, yl_d,
            vr_d, wr_d, xg_d, vpost_d, obs_c, unk_c, tol_d, lam_d, ustd_d, x0_d, dt_d, dist_weight, noise_d, u_d, costs_d)
    N = noise_d.shape[0]
    if mode == "spd":
        RMPPI.rollout_det_dyn_w_speed_map_numba[N, 1](lin_g, ang_g, rl.risk_traction_map_d, *tail)
    else:
        RMPPI.rollout_det_dyn_numba[N, 1](lin_g, ang_g, *tail)


def assert_inside(states, tdm):
    """Every state (the oracle's, (..., 3)) lies in a cell of the TDM's padded map: no comparison then rests on the
    engine's rule for lookups outside the map (wrap, then clamp; the reference reads outside its allocation)."""
    st = np.asarray(states, np.float64)
    Hp, Wp = tdm.pmf_grid_d.shape[1:]
    xi = np.floor((st[..., 0] - float(tdm.padded_xlimits[0])) / float(np.float32(tdm.res)))
    yi = np.floor((st[..., 1] - float(tdm.padded_ylimits[0])) / float(np.float32(tdm.res)))
    assert np.isfinite(st).all()
    assert (xi >= 1).all() and (xi < Wp - 1).all() and (yi >= 1).all() and (yi < Hp - 1).all(), \
        "a trajectory leaves the padded map: cells x %s, y %s of %d x %d" % (
            (xi.min(), xi.max()), (yi.min(), yi.max()), Hp, Wp)


@pytest.mark.parametrize("mode,N,M,T,H,res,B,det_alpha", [
    ("tdm", 1024, 64, 64, 512, 0.1, 12, 1.0),        # BASELINE config 3
    ("det", 4096, 1, 128, 512, 0.2, 32, 0.3),        # BASELINE config 4
    ("tdm", 8192, 256, 128, 1024, 0.1, 12, 1.0),     # BASELINE config 5, the headline workload, full size
    ("tdm", 128, 1100, 32, 128, 0.1, 12, 1.0),       # M > 1024: rollout_oversized_numba, cvar_alpha = 1 (its
                                                     # "sort" for alpha < 1 swaps unconditionally, SURVEY 9-B1)
    ("spd", 4096, 1, 128, 512, 0.2, 32, 0.3),        # speed map at config 4's size, risk from the CVaR at 0.3
    ("spd", 100, 1, 37, 160, 0.2, 12, 1.0),          # speed map at the reference's minimum N, ragged T, mean risk
])
def test_kernels_vs_reference_numba_cuda(ref, dev, mode, N, M, T, H, res, B, det_alpha):
    RConfig, RTDM, RMPPI, cuda = ref
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from tests.scenarios import make_scenario, oracle_rollout_costs
    sc = make_scenario(mode, N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=1, det_alpha=det_alpha, warm_start=True,
                       cvar_alpha=1.0 if M > 1024 else 0.5, bin_values=OUTSIDE_BOUNDS(B) if mode == "spd" else None)
    p = sc["params"]
    rp = ref_planner(ref, sc)
    rl, ra = rp.lin_tdm, rp.ang_tdm
    with quiet():
        ep = tdm_planner(E, sc)
    el, ea = ep.lin_tdm, ep.ang_tdm
    ep.move_mppi_task_vars_to_device()
    L = E._lib
    Hp, Wp = el.pmf_grid_d.shape[1:]
    # host preprocessing of the setter
    assert (rl.pmf_grid_d.copy_to_host() == el.pmf_grid_d.copy_to_host()).all()
    if mode == "spd":                     # the risk map truncates and wraps where the bin values leave the bounds
        risk = rl.risk_traction_map_d.copy_to_host()
        assert (risk < 0).any() and (risk == el.risk_traction_map_d.copy_to_host()).all()
    # replay the body of solve_* kernel by kernel on both sides (same seed -> same streams)
    (res_d, xl_d, yl_d, vr_d, wr_d, xg_d, vpost_d, tol_d, lam_d, ustd_d, cvar_d, x0_d, dt_d, obs_c, unk_c) = \
        rp.move_mppi_task_vars_to_device()
    alpha_dyn = 0.9 if mode == "tdm" else 1.0
    lin_g, ang_g = rl.sample_grids(alpha_dyn), ra.sample_grids(alpha_dyn)
    eg_l, eg_a = el.sample_grids(alpha_dyn).copy_to_host(), ea.sample_grids(alpha_dyn).copy_to_host()
    assert (lin_g.copy_to_host()[:, :Hp, :Wp] == eg_l[:, :Hp, :Wp]).all()
    assert (ang_g.copy_to_host()[:, :Hp, :Wp] == eg_a[:, :Hp, :Wp]).all()
    RMPPI.sample_noise_numba[N, T](rp.rng_states_d, ustd_d, rp.noise_samples_d)
    L.check(L.lib.b200mppi_planner_sample_noise(ep._handle))
    noise = rp.noise_samples_d.copy_to_host()
    assert (noise == ep.noise_samples_d.copy_to_host()).all()
    if mode == "tdm":
        kern = RMPPI.rollout_numba[N, M, 0, 4 * M] if M <= 1024 else RMPPI.rollout_oversized_numba[N, 1024, 0, 4 * M]
        kern(
            lin_g, ang_g, rl.bin_values_bounds_d, ra.bin_values_bounds_d, rl.obstacle_map_d, rl.unknown_map_d, res_d,
            xl_d, yl_d, vr_d, wr_d, xg_d, vpost_d, obs_c, unk_c, tol_d, lam_d, ustd_d, cvar_d, x0_d, dt_d, 1.0,
            rp.noise_samples_d, rp.u_cur_d, rp.costs_d)
    else:
        assert_inside(oracle_rollout_costs(sc, el, ea, noise, sc["u0"], arith=dev, return_states=True)[1], el)
        one_map_rollout(ref, rp, mode, lin_g, ang_g, rp.noise_samples_d, rp.u_cur_d, rp.costs_d)
    cuda.synchronize()
    ref_costs = rp.costs_d.copy_to_host().copy()
    L.check(L.lib.b200mppi_planner_rollout(ep._handle))
    got = ep.costs_d.copy_to_host()
    rel = np.abs(got - ref_costs) / np.maximum(np.abs(ref_costs), 1e-6)
    print("\n[%s] costs bit-identical %.4f, max rel %.2e" % (mode, float((got == ref_costs).mean()), float(rel.max())))
    if mode != "tdm":
        assert (got == ref_costs).all()
    else:
        check_cvar_vs_reference(got, ref_costs, ep.costs_nm_d.copy_to_host(), noise, sc["u0"], p)
    RMPPI.update_useq_numba[1, 32](lam_d, rp.costs_d, rp.noise_samples_d, rp.weights_d, vr_d, wr_d, rp.u_cur_d)
    cuda.synchronize()
    ref_u = rp.u_cur_d.copy_to_host()
    c = np.ascontiguousarray(ref_costs)
    L.check(L.lib.b200mppi_planner_update(ep._handle, L.ptr(c)))
    eu = ep.u_cur_d.copy_to_host()
    np.testing.assert_allclose(eu, ref_u, rtol=1e-4, atol=1e-5)


def check_cvar_vs_reference(got, ref_costs, costs_nm, noise, u_cur, p):
    """|engine - reference| <= (CVaR kernel bound + reference tree bound) around the exact mean of the engine's
    per-(n, m) costs, + R_n: the reference adds each step's control cost to a map's running cost, the windowed kernel
    adds their pre-summed total, so the per-(n, m) costs may differ by the roundings of T + 1 adds and of the
    presum, R_n = gamma(2T + 4) * (max_m |cost_nm| + 2 sum_t |c_nt|)."""
    from tests import reduce_bounds as RB
    alpha, M, T = p["cvar_alpha"], costs_nm.shape[1], noise.shape[1]
    std = np.asarray(p["u_std"], np.float64)
    ctrl = p["lambda_weight"] * (np.abs(u_cur[None, :, 0] / std[0] ** 2 * noise[:, :, 0]) +
                                 np.abs(u_cur[None, :, 1] / std[1] ** 2 * noise[:, :, 1]))
    roll = RB.gamma(2 * T + 4) * (np.abs(costs_nm.astype(np.float64)).max(axis=1) + 2 * ctrl.sum(axis=1)) * 1.001
    worst, worst_order = 0.0, 0.0
    for n, (mu, abs_sum, numel) in enumerate(RB.cvar_exact(costs_nm, alpha)):
        b = RB.cvar_bound(M, numel, abs_sum, mu, RB.kernel_kind(M)) + RB.cvar_bound(M, numel, abs_sum, mu, "tree")
        d = abs(float(got[n]) - float(ref_costs[n]))
        assert d <= b + roll[n], "n %d: engine %r, reference %r, |difference| %.3e > %.3e + %.3e" % (
            n, got[n], ref_costs[n], d, b, roll[n])
        worst = max(worst, d / (b + roll[n]))
        worst_order = max(worst_order, d / b)
    print("[cvar vs reference] largest |difference| / bound %.3g (%.3g of the summation bounds alone)"
          % (worst, worst_order))


@pytest.mark.parametrize("kind,method", [
    pytest.param(kind, method, id=kind if method == "det" else "%s-%s" % (kind, method))   # det: the plain kind
    for method in ("det", "spd") for kind in ("state", "traction", "speed")])
def test_reference_fuses_traction_and_state_updates(ref, dev, method, kind):
    """rollout_det_dyn_numba and rollout_det_dyn_w_speed_map_numba themselves on the directed cases of
    tests/directed_cases.py: rounding lo + ratio*q, or dt*vtr*v*cos + x, before the add would move the first step's x by
    one float32 ulp and flip the goal flag (kinds state, traction); rounding the speed map's lo + ratio*risk before the
    add would move its time step dt / (eff + 1e-6), the whole cost, by one float32 ulp (kind speed).  The reference's
    costs equal the engine's and the exact oracle's (device provider) bit for bit, so the reference fuses each as the
    oracle does."""
    RConfig, RTDM, RMPPI, cuda = ref
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from tests.directed_cases import boundary_case, directed_scenario
    case = boundary_case(dev, kind)
    if kind == "speed":
        assert case["cost_exact"] != case["cost_other"]
    else:
        assert case["x1_exact"] != case["x1_other"]
    s = directed_scenario(case, N=40, M=1)
    N, mode = s["N"], dict(det=1, spd=2)[method]
    lim = np.array([s["xlo"], s["xlo"] + s["Cc"] * s["res"]], f32)
    costs_d = cuda.device_array(N, dtype=f32)
    head = (cuda.to_device(s["lin"]), cuda.to_device(s["ang"]))
    if method == "spd":
        head += (cuda.to_device(s["risk"][None]),)
    kern = RMPPI.rollout_det_dyn_w_speed_map_numba if method == "spd" else RMPPI.rollout_det_dyn_numba
    kern[N, 1](
        *head, cuda.to_device(np.array(s["lb"], f32)),
        cuda.to_device(np.array(s["ab"], f32)), cuda.to_device(s["obs"]), cuda.to_device(s["unk"]), f32(s["res"]),
        cuda.to_device(lim), cuda.to_device(lim), cuda.to_device(np.array([0, 3], f32)),
        cuda.to_device(np.array([-np.pi, np.pi], f32)), cuda.to_device(np.array(s["goal"], f32)), f32(0.01), f32(1e5),
        f32(1e2), f32(s["tol"]), f32(1.0), cuda.to_device(np.array([2, 3], f32)), cuda.to_device(np.array(s["x0"], f32)),
        f32(s["dt"]), 1.0, cuda.to_device(s["noise"]), cuda.to_device(s["u_cur"]), costs_d)
    cuda.synchronize()
    ref_costs = costs_d.copy_to_host()[:, None]
    want = directed_oracle(s, mode, dev)
    assert_all_equal(ref_costs, want, "reference %s, %s boundary" % (method, kind))
    assert_all_equal(run_directed(E, s, mode), want, "engine %s, %s boundary" % (method, kind))
    if kind == "speed" and method == "spd":
        assert (ref_costs == case["cost_exact"]).all()


# ----------------------------------------------------------------------------- batched one-map rollouts
@pytest.mark.parametrize("kinds", [("spd", "spd", "spd"), ("det", "spd", "spd", "det")])
def test_batched_one_map_rollouts_vs_reference(ref, eng, dev, kinds):
    """One solve (num_opt 1) of an MPPI_Batch of speed-map planners (rollout_batch_kernel<2>) and of an MPPI_MixedBatch
    of det-dynamics and speed-map planners (rollout_batch_mixed_kernel), each planner with its own seed, maps, start,
    risk and controls: every planner's costs equal the reference kernel's on that planner's noise (itself equal to the
    reference's sample_noise_numba from the same seed), sampled maps and pre-solve u_cur, bit for bit."""
    RConfig, RTDM, RMPPI, cuda = ref
    E = eng
    from tests.scenarios import make_scenario, oracle_rollout_costs
    scs = [make_scenario(kind, N=256, M=1, T=40, H=200, W=200, res=0.2, B=8, seed=31 + 3 * k, warm_start=True,
                         det_alpha=[0.4, 1.0, 0.7][k % 3], bin_values=OUTSIDE_BOUNDS(8) if kind == "spd" else None)
           for k, kind in enumerate(kinds)]
    with quiet():
        pls = [tdm_planner(E, sc) for sc in scs]
        batch = E.MPPI_Batch(pls) if len(set(kinds)) == 1 else E.MPPI_MixedBatch(pls)
        batch.solve()
    for k, (kind, sc, pl) in enumerate(zip(kinds, scs, pls)):
        rp = ref_planner(ref, sc)
        ustd_d = rp.move_mppi_task_vars_to_device()[9]
        N, T = sc["N"], sc["T"]
        RMPPI.sample_noise_numba[N, T](rp.rng_states_d, ustd_d, rp.noise_samples_d)
        noise = pl.noise_samples_d.copy_to_host()
        assert (rp.noise_samples_d.copy_to_host() == noise).all(), "planner %d noise" % k
        lin_g, ang_g = rp.lin_tdm.sample_grids(1.0), rp.ang_tdm.sample_grids(1.0)
        Hp, Wp = pl.lin_tdm.pmf_grid_d.shape[1:]
        for r, e in ((lin_g, pl.lin_tdm), (ang_g, pl.ang_tdm)):
            assert (r.copy_to_host()[:, :Hp, :Wp] == e.sample_grid_batch_d.copy_to_host()[:1, :Hp, :Wp]).all()
        assert_inside(oracle_rollout_costs(sc, pl.lin_tdm, pl.ang_tdm, noise, sc["u0"], arith=dev,
                                           return_states=True)[1], pl.lin_tdm)
        costs_d = cuda.device_array(N, dtype=f32)
        one_map_rollout(ref, rp, kind, lin_g, ang_g, rp.noise_samples_d, cuda.to_device(sc["u0"]), costs_d)
        cuda.synchronize()
        assert_all_equal(pl.costs_d.copy_to_host(), costs_d.copy_to_host(), "%s batch planner %d (%s)" % (
            type(batch).__name__, k, kind))


# ----------------------------------------------------------------------------- visualisation rollouts
@pytest.mark.parametrize("mode", ["det", "spd", "tdm"])
@pytest.mark.parametrize("V", [1, 31, 32, 33, 100])
def test_state_rollouts_vs_reference(ref, eng, dev, mode, V):
    """get_state_rollout of one planner (state_rollout_kernel) and of a batch of two (state_rollout_batch_kernel)
    against the reference's get_state_rollout_across_control_noise (det, spd) and get_state_rollout_across_envs_numba
    (tdm), launched by the reference's own get_state_rollout: the same sampled maps, u_cur outside vrange / wrange (row 0
    does not clip), u_prev != u_cur and noise that pushes past the clip; every state bit for bit.  V spans one, and
    more than one, 32-thread block of the engine's launch."""
    RConfig, RTDM, RMPPI, cuda = ref
    E = eng
    from oracle import mppi_ref as MR
    from tests.scenarios import make_scenario
    N, M, T = 128, 128, 24
    pls, wants = [], []
    for k in range(2):
        sc = make_scenario(mode, N=N, M=M, T=T, H=200, W=200, res=0.2, B=6, seed=41 + 5 * k)
        sc["cfg"]["num_vis_state_rollouts"] = V
        rng = np.random.default_rng(60 + k)
        u_cur = np.stack([rng.uniform(-0.6, 3.6, T), rng.uniform(-4.0, 4.0, T)], 1).astype(f32)
        u_prev = np.stack([rng.uniform(-0.6, 3.6, T), rng.uniform(-4.0, 4.0, T)], 1).astype(f32)
        noise = (rng.standard_normal((N, T, 2)) * np.array([2.0, 3.0])).astype(f32)
        with quiet():
            pl = tdm_planner(E, sc)
        rp = ref_planner(ref, sc)
        assert pl.num_vis_state_rollouts == rp.num_vis_state_rollouts == V
        pl.u_cur_d.copy_to_device(u_cur)
        pl.u_prev_d.copy_to_device(u_prev)
        pl.noise_samples_d.copy_to_device(noise)
        rp.u_cur_d, rp.u_prev_d = cuda.to_device(u_cur), cuda.to_device(u_prev)
        rp.noise_samples_d.copy_to_device(noise)
        Hp, Wp = pl.lin_tdm.pmf_grid_d.shape[1:]
        maps = V if mode == "tdm" else 1
        for r, e in ((rp.lin_tdm, pl.lin_tdm), (rp.ang_tdm, pl.ang_tdm)):
            got, want = e.sample_grids(1.0).copy_to_host(), r.sample_grids(1.0).copy_to_host()
            assert (got[:maps, :Hp, :Wp] == want[:maps, :Hp, :Wp]).all()
        want = _quiet(rp.get_state_rollout).copy()
        lt = pl.lin_tdm
        grids = (lt.sample_grid_batch_d.copy_to_host()[:, :Hp, :Wp], pl.ang_tdm.sample_grid_batch_d.copy_to_host()[:, :Hp, :Wp])
        assert_all_equal(want, MR.state_rollouts(dict(tdm=MR.MODE_STOCHASTIC, det=MR.MODE_DET_DYN, spd=MR.MODE_SPEED_MAP)[mode],
                                                 V, *grids, lt.bin_values_bounds, pl.ang_tdm.bin_values_bounds, f32(lt.res),
                                                 lt.padded_xlimits, lt.padded_ylimits, pl.params["x0"], pl.params["dt"],
                                                 u_cur, u_prev, noise, pl.params["vrange"], pl.params["wrange"], arith=dev),
                         "oracle, %s V %d planner %d" % (mode, V, k))
        assert_inside(want, lt)
        with quiet():
            assert_all_equal(pl.get_state_rollout(), want, "get_state_rollout, %s V %d planner %d" % (mode, V, k))
        pls.append(pl)
        wants.append(want)
    cls = E.MPPI_StochasticBatch if mode == "tdm" else E.MPPI_Batch
    with quiet():
        got = cls(pls).get_state_rollout()
    for k in range(2):
        assert_all_equal(got[k], wants[k], "batch get_state_rollout, %s V %d planner %d" % (mode, V, k))


@pytest.mark.parametrize("kind", ["state", "traction"])
def test_state_rollouts_on_a_float32_rounding_boundary(ref, eng, dev, kind):
    """The directed state and traction cases through the reference's two visualisation kernels and the engine's
    (modes 1 and 0): the first saved x is the one-ulp decision itself."""
    RConfig, RTDM, RMPPI, cuda = ref
    from tests.directed_cases import directed_scenario, fma_boundary_case
    case = fma_boundary_case(dev, kind)
    s = directed_scenario(case, N=40, M=1)
    T = s["T"]
    lim = cuda.to_device(np.array([s["xlo"], s["xlo"] + s["Cc"] * s["res"]], f32))
    common = (cuda.to_device(s["lin"]), cuda.to_device(s["ang"]), cuda.to_device(np.array(s["lb"], f32)),
              cuda.to_device(np.array(s["ab"], f32)), f32(s["res"]), lim, lim, cuda.to_device(np.array(s["x0"], f32)),
              f32(s["dt"]))
    u_d = cuda.to_device(s["u_cur"])
    a = cuda.device_array((1, T + 1, 3), dtype=f32)
    RMPPI.get_state_rollout_across_control_noise[1, 1](a, *common, cuda.to_device(s["noise"]),
                                                       cuda.to_device(np.array([0, 3], f32)),
                                                       cuda.to_device(np.array([-np.pi, np.pi], f32)), u_d, u_d)
    b = cuda.device_array((1, T + 1, 3), dtype=f32)
    RMPPI.get_state_rollout_across_envs_numba[1, 1](b, *common, u_d)
    cuda.synchronize()
    a, b = a.copy_to_host(), b.copy_to_host()
    assert a[0, 1, 0] == b[0, 1, 0] == case["x1_exact"] != case["x1_other"]
    assert_all_equal(run_directed(eng, s, 1, states=True), a, "engine mode 1, %s boundary" % kind)
    assert_all_equal(run_directed(eng, s, 0, states=True), b, "engine mode 0, %s boundary" % kind)


# ----------------------------------------------------------------------------- the map-free notebook
@pytest.fixture(scope="module")
def notebook(ref):
    """MPPI_Numba of the compiled barebone_mppi_numba.ipynb (oracle/ref_build.py), whose kernels are its static
    methods."""
    from oracle.ref_build import compiled_notebook
    root = compiled_notebook()
    if root is None:
        pytest.skip("compiled notebook not available (oracle/_ref/barebone_mppi_numba.pyc absent)")
    if root not in sys.path:
        sys.path.insert(0, root)
    import barebone_mppi_numba
    return barebone_mppi_numba.MPPI_Numba


def notebook_run(ref, BMPPI, c, noise, u_cur, u_prev, V):
    """The notebook's rollout_numba and get_state_rollout_across_control_noise on an edge case, launched with the
    arguments its solve() and get_state_rollout() pass (without obstacles, its own host-array stand-ins)."""
    cuda = ref[3]
    to = cuda.to_device
    ob = c["obstacles"]
    if len(ob):
        pos, rad = to(np.ascontiguousarray(ob[:, :2], f32)), to(np.ascontiguousarray(ob[:, 2], f32))
    else:
        pos, rad = np.array([[1e5, 1e5]], dtype=f32), np.array([0], dtype=f32)
    vr, wr = to(np.asarray(c["vrange"], f32)), to(np.asarray(c["wrange"], f32))
    x0 = to(np.asarray(c["x0"], f32))
    noise_d, u_d = to(noise), to(u_cur)
    N, T = noise.shape[:2]
    costs = cuda.device_array(N, dtype=f32)
    BMPPI.rollout_numba[N, 1](vr, wr, to(np.asarray(c["goal"], f32)), f32(c["obs_cost"]), pos, rad, f32(c["tol"]),
                              f32(c["lam"]), to(np.asarray(c["u_std"], f32)), x0, f32(c["dt"]), float(c["dist_weight"]),
                              noise_d, u_d, costs)
    states = cuda.device_array((V, T + 1, 3), dtype=f32)
    BMPPI.get_state_rollout_across_control_noise[V, 1](states, x0, f32(c["dt"]), noise_d, vr, wr, to(u_prev), u_d)
    cuda.synchronize()
    return costs.copy_to_host(), states.copy_to_host()


def _notebook_cases():
    return [c["name"] for c in BE.CASES] + ["directed-obstacle-" + k for k in ("up", "up_ahead", "down", "on_circle")] + \
        ["directed-goal-" + k for k in ("on_tol", "split")]


@pytest.mark.parametrize("name", _notebook_cases())
def test_notebook_kernels_vs_engine(ref, notebook, eng, dev, name):
    """The map-free planner (mode 3, RawBarebone) against the notebook's own compiled kernels: every cost and every
    visualisation state bit for bit, over the edge-case sweep and the directed obstacle and goal boundaries (built with
    this GPU's cos / sin)."""
    from tests.test_gpu_barebone_edges import RawBarebone
    if name.startswith("directed-obstacle-"):
        case = BE.obstacle_boundary_case(dev, name[len("directed-obstacle-"):])
        assert case["alt_outside"] != case["exact_outside"]
        c, noise, u_cur, u_prev = BE.directed_inputs(case)
    elif name.startswith("directed-goal-"):
        case = BE.goal_boundary_case(dev, name[len("directed-goal-"):])
        assert case["alt_reached"] != case["exact_reached"]
        c, noise, u_cur, u_prev = BE.directed_inputs(case)
    else:
        c = next(c for c in BE.CASES if c["name"] == name)
        noise, u_cur, u_prev = BE.inputs(c)
    V = BE.vis_count(c)
    want_costs, want_states = notebook_run(ref, notebook, c, noise, u_cur, u_prev, V)
    rp = RawBarebone(eng, c, V)
    try:
        costs = rp.rollout(noise, u_cur)
        states = rp.states(u_prev)
    finally:
        rp.close()
    assert_all_equal(costs, want_costs, name + " costs")
    assert_all_equal(states, want_states, name + " states")
