"""Run the UNMODIFIED reference (Numba-CUDA) on a real GPU next to the engine: timing of its
solve() at the BASELINE configs and kernel-level parity on identical inputs.  TEST INFRASTRUCTURE.

The reference is imported from the bytecode build() compiles under oracle/_ref/ (oracle/ref_build.py;
git-ignored, never committed).  If that is absent the script says so and exits 0.

    python -m oracle.ref_gpu_probe [c2 c3 c4 c5] [--out DIR]   -> DIR/ref_probe.json (default: runs/, git-ignored)
"""
import io
import contextlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def locate():
    from oracle.ref_build import compiled_reference
    return compiled_reference()


def out_dir():
    return sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else os.path.join(ROOT, "runs")


def quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def main():
    ref_root = locate()
    out_path = os.path.join(out_dir(), "ref_probe.json")
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    if ref_root is None:
        json.dump({"unavailable": "reference not found"}, open(out_path, "w"))
        print("reference not found; nothing to do")
        return
    np.float = float
    sys.path.insert(0, ref_root)
    sys.path.insert(0, ROOT)
    from numba import cuda
    from mppi_numba.config import Config as RConfig
    from mppi_numba.terrain import TDM_Numba as RTDM
    from mppi_numba.mppi import MPPI_Numba as RMPPI
    import mppi_numba_b200 as E
    from bench import WORKLOADS, build_scenario
    names = [a for a in sys.argv[1:] if a in WORKLOADS] or ["c2", "c3", "c4", "c5"]
    results = {"numba_cc": list(cuda.get_current_device().compute_capability), "workloads": {}}
    f32 = np.float32
    for name in names:
        sc = build_scenario(name)
        p = sc["params"]
        rcfg = quiet(RConfig, **sc["cfg"])
        rl, ra = quiet(RTDM, rcfg), quiet(RTDM, rcfg)
        quiet(rl.set_TDM_from_PMF_grid, sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        quiet(ra.set_TDM_from_PMF_grid, sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        rp = quiet(RMPPI, rcfg)
        rp.setup(p, rl, ra)
        N, M, T = sc["N"], (sc["M"] if sc["mode"] == "tdm" else 1), sc["T"]
        res = {"N": N, "M": M, "T": T}
        # ---- timing of the reference's public solve()
        t0 = time.perf_counter()
        quiet(rp.solve)
        res["first_solve_s (JIT)"] = time.perf_counter() - t0
        ts = []
        for _ in range(5 if name == "c5" else 10):
            cuda.synchronize()
            t0 = time.perf_counter()
            rp.solve()
            ts.append(time.perf_counter() - t0)
        res["solve_ms_median"] = 1e3 * float(np.median(ts))
        res["rate_state_steps_per_s"] = N * M * T / float(np.median(ts))
        # per-stage: sampling alone
        cuda.synchronize()
        t0 = time.perf_counter()
        rl.sample_grids(1.0)
        ra.sample_grids(1.0)
        cuda.synchronize()
        res["sample_grids_x2_ms"] = 1e3 * (time.perf_counter() - t0)

        # ---- kernel-level parity on identical inputs: replay the body of solve_* kernel by kernel
        (res_d, xl_d, yl_d, vr_d, wr_d, xg_d, vpost_d, tol_d, lam_d, ustd_d, cvar_d, x0_d, dt_d, obs_c, unk_c) = \
            rp.move_mppi_task_vars_to_device()
        lin_g = rl.sample_grids(1.0)
        ang_g = ra.sample_grids(1.0)
        RMPPI.sample_noise_numba[N, T](rp.rng_states_d, ustd_d, rp.noise_samples_d)
        cuda.synchronize()
        t0 = time.perf_counter()
        if sc["mode"] == "tdm":
            RMPPI.rollout_numba[N, M, 0, 4 * M](
                lin_g, ang_g, rl.bin_values_bounds_d, ra.bin_values_bounds_d, rl.obstacle_map_d, rl.unknown_map_d,
                res_d, xl_d, yl_d, vr_d, wr_d, xg_d, vpost_d, obs_c, unk_c, tol_d, lam_d, ustd_d, cvar_d, x0_d, dt_d,
                1.0, rp.noise_samples_d, rp.u_cur_d, rp.costs_d)
        else:
            RMPPI.rollout_det_dyn_numba[N, 1](
                lin_g, ang_g, rl.bin_values_bounds_d, ra.bin_values_bounds_d, rl.obstacle_map_d, rl.unknown_map_d,
                res_d, xl_d, yl_d, vr_d, wr_d, xg_d, vpost_d, obs_c, unk_c, tol_d, lam_d, ustd_d, x0_d, dt_d,
                1.0, rp.noise_samples_d, rp.u_cur_d, rp.costs_d)
        cuda.synchronize()
        res["rollout_kernel_ms"] = 1e3 * (time.perf_counter() - t0)
        ref_costs = rp.costs_d.copy_to_host().copy()
        noise = rp.noise_samples_d.copy_to_host()
        u_cur = rp.u_cur_d.copy_to_host()
        gl = lin_g.copy_to_host()
        ga = ang_g.copy_to_host()
        t0 = time.perf_counter()
        RMPPI.update_useq_numba[1, 32](lam_d, rp.costs_d, rp.noise_samples_d, rp.weights_d, vr_d, wr_d, rp.u_cur_d)
        cuda.synchronize()
        res["update_kernel_ms"] = 1e3 * (time.perf_counter() - t0)
        ref_u = rp.u_cur_d.copy_to_host()

        # the engine on the same noise / maps / warm start
        cfg = quiet(E.Config, **sc["cfg"])
        el, ea = quiet(E.TDM_Numba, cfg), quiet(E.TDM_Numba, cfg)
        quiet(el.set_TDM_from_PMF_grid, sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        quiet(ea.set_TDM_from_PMF_grid, sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        ep = quiet(E.MPPI_Numba, cfg)
        ep.setup(p, el, ea)
        ep.move_mppi_task_vars_to_device()
        Hp, Wp = el.pmf_grid_d.shape[1:]
        # did the engine's sampler produce the same maps as the reference's (same seed, same call count)?
        for _ in range(int(round(len(ts))) + 3):          # the reference sampled: 1 JIT + len(ts) + 1 + 1 times
            pass
        el.sample_grid_batch_d.copy_to_device(gl)
        ea.sample_grid_batch_d.copy_to_device(ga)
        ep.noise_samples_d.copy_to_device(noise)
        ep.u_cur_d.copy_to_device(u_cur)
        L = E._lib
        L.check(L.lib.b200mppi_planner_rollout(ep._handle))
        got = ep.costs_d.copy_to_host()
        rel = np.abs(got - ref_costs) / np.maximum(np.abs(ref_costs), 1e-6)
        res["costs_bit_identical_frac"] = float((got == ref_costs).mean())
        res["costs_within_1e-4_frac"] = float((rel < 1e-4).mean())
        res["costs_rel_median"] = float(np.median(rel))
        res["costs_rel_max"] = float(rel.max())
        c = np.ascontiguousarray(ref_costs)
        L.check(L.lib.b200mppi_planner_update(ep._handle, L.ptr(c)))
        eu = ep.u_cur_d.copy_to_host()
        res["u_max_abs_diff_given_ref_costs"] = float(np.abs(eu - ref_u).max())
        res["u_max_rel_diff_given_ref_costs"] = float((np.abs(eu - ref_u) / np.maximum(np.abs(ref_u), 1e-3)).max())
        # noise generator: engine stream vs the reference stream for a fresh planner pair with the same seed
        rp2 = quiet(RMPPI, rcfg)
        RMPPI.sample_noise_numba[N, T](rp2.rng_states_d, ustd_d, rp2.noise_samples_d)
        ep2 = quiet(E.MPPI_Numba, cfg)
        ep2.setup(p, el, ea)
        ep2.move_mppi_task_vars_to_device()
        L.check(L.lib.b200mppi_planner_sample_noise(ep2._handle))
        n_ref, n_eng = rp2.noise_samples_d.copy_to_host(), ep2.noise_samples_d.copy_to_host()
        res["noise_bit_identical_frac"] = float((n_ref == n_eng).mean())
        res["noise_max_abs_diff"] = float(np.abs(n_ref - n_eng).max())
        # map sampler: fresh TDMs with the same seed
        rl2 = quiet(RTDM, rcfg)
        quiet(rl2.set_TDM_from_PMF_grid, sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        el2 = quiet(E.TDM_Numba, cfg)
        quiet(el2.set_TDM_from_PMF_grid, sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        g_ref = rl2.sample_grids(0.9).copy_to_host()[:, :Hp, :Wp]
        g_eng = el2.sample_grids(0.9).copy_to_host()[:, :Hp, :Wp]
        res["sampled_maps_bit_identical"] = bool((g_ref == g_eng).all())
        res["sampled_maps_mismatch_frac"] = float((g_ref != g_eng).mean())
        results["workloads"][name] = res
        print(name, json.dumps(res))
        del rp, rl, ra, rp2, rl2, ep, ep2, el, ea, el2
    json.dump(results, open(out_path, "w"), indent=1)


if __name__ == "__main__":
    main()
