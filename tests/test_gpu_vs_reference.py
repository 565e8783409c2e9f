"""Kernel-by-kernel parity against the UNMODIFIED reference's Numba-CUDA kernels running on the same GPU.

The reference cannot be committed to this repository; build() compiles it to git-ignored bytecode under
oracle/_ref/ where its sources are readable (oracle/ref_build.py).  When that was not built the tests skip.
What is asserted (same inputs on both sides: seed, PMFs, masks, params):
  * control noise: bit-identical;  sampled traction maps: bit-identical
  * deterministic-mode rollout costs: bit-identical
  * stochastic CVaR costs: within 1e-4 relative (only the summation order of the CVaR mean differs),
    including M > 1024 against the reference's oversized kernel at cvar_alpha = 1
  * updated control sequence given the reference's costs: within 1e-4
"""
import io
import contextlib
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


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


@pytest.mark.parametrize("mode,N,M,T,H,res,B,det_alpha", [
    ("tdm", 1024, 64, 64, 512, 0.1, 12, 1.0),        # BASELINE config 3
    ("det", 4096, 1, 128, 512, 0.2, 32, 0.3),        # BASELINE config 4
    ("tdm", 8192, 256, 128, 1024, 0.1, 12, 1.0),     # BASELINE config 5, the headline workload, full size
    ("tdm", 128, 1100, 32, 128, 0.1, 12, 1.0),       # M > 1024: rollout_oversized_numba, cvar_alpha = 1 (its
                                                     # "sort" for alpha < 1 swaps unconditionally, SURVEY 9-B1)
])
def test_kernels_vs_reference_numba_cuda(ref, mode, N, M, T, H, res, B, det_alpha):
    RConfig, RTDM, RMPPI, cuda = ref
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    from tests.scenarios import make_scenario
    sc = make_scenario(mode, N=N, M=M, T=T, H=H, W=H, res=res, B=B, seed=1, det_alpha=det_alpha, warm_start=True,
                       cvar_alpha=1.0 if M > 1024 else 0.5)
    p = sc["params"]
    rcfg = _quiet(RConfig, **sc["cfg"])
    rl, ra = _quiet(RTDM, rcfg), _quiet(RTDM, rcfg)
    _quiet(rl.set_TDM_from_PMF_grid, sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    _quiet(ra.set_TDM_from_PMF_grid, sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    rp = _quiet(RMPPI, rcfg)
    rp.setup(p, rl, ra)
    rp.u_cur_d = cuda.to_device(sc["u0"])
    cfg = _quiet(E.Config, **sc["cfg"])
    el, ea = _quiet(E.TDM_Numba, cfg), _quiet(E.TDM_Numba, cfg)
    _quiet(el.set_TDM_from_PMF_grid, sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    _quiet(ea.set_TDM_from_PMF_grid, sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    ep = _quiet(E.MPPI_Numba, cfg)
    ep.setup(p, el, ea)
    ep.u_cur_d.copy_to_device(sc["u0"])
    ep.move_mppi_task_vars_to_device()
    L = E._lib
    Hp, Wp = el.pmf_grid_d.shape[1:]
    Mg = M if mode == "tdm" else 1
    # host preprocessing of the setter
    assert (rl.pmf_grid_d.copy_to_host() == el.pmf_grid_d.copy_to_host()).all()
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
        RMPPI.rollout_det_dyn_numba[N, 1](
            lin_g, ang_g, rl.bin_values_bounds_d, ra.bin_values_bounds_d, rl.obstacle_map_d, rl.unknown_map_d, res_d,
            xl_d, yl_d, vr_d, wr_d, xg_d, vpost_d, obs_c, unk_c, tol_d, lam_d, ustd_d, x0_d, dt_d, 1.0,
            rp.noise_samples_d, rp.u_cur_d, rp.costs_d)
    cuda.synchronize()
    ref_costs = rp.costs_d.copy_to_host().copy()
    L.check(L.lib.b200mppi_planner_rollout(ep._handle))
    got = ep.costs_d.copy_to_host()
    rel = np.abs(got - ref_costs) / np.maximum(np.abs(ref_costs), 1e-6)
    print("\n[%s] costs bit-identical %.4f, max rel %.2e" % (mode, float((got == ref_costs).mean()), float(rel.max())))
    if mode == "det":
        assert (got == ref_costs).all()
    else:
        assert rel.max() < 1e-4
    RMPPI.update_useq_numba[1, 32](lam_d, rp.costs_d, rp.noise_samples_d, rp.weights_d, vr_d, wr_d, rp.u_cur_d)
    cuda.synchronize()
    ref_u = rp.u_cur_d.copy_to_host()
    c = np.ascontiguousarray(ref_costs)
    L.check(L.lib.b200mppi_planner_update(ep._handle, L.ptr(c)))
    eu = ep.u_cur_d.copy_to_host()
    np.testing.assert_allclose(eu, ref_u, rtol=1e-4, atol=1e-5)
