"""Debug aid (TEST INFRASTRUCTURE): per-step state traces of the reference's Numba-CUDA kernels vs the
engine on a real GPU, to localise the first diverging step of the rare rollouts whose costs differ.

    python -m oracle.ref_gpu_trace c4 [--out DIR]   -> DIR/trace_<name>.json (default: runs/, git-ignored)
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def main():
    from oracle.ref_gpu_probe import locate, out_dir, quiet
    ref_root = locate()
    if ref_root is None:
        print("reference not found")
        return
    np.float = float
    sys.path.insert(0, ref_root)
    sys.path.insert(0, ROOT)
    from numba import cuda
    from mppi_numba.config import Config as RConfig
    from mppi_numba.terrain import TDM_Numba as RTDM
    from mppi_numba.mppi import MPPI_Numba as RMPPI
    import mppi_numba_b200 as E
    from bench import build_scenario
    from tests.test_gpu_parity import RawPlanner
    name = sys.argv[1] if len(sys.argv) > 1 else "c4"
    sc = build_scenario(name)
    p = sc["params"]
    f32 = np.float32
    rcfg = quiet(RConfig, **sc["cfg"])
    rl, ra = quiet(RTDM, rcfg), quiet(RTDM, rcfg)
    quiet(rl.set_TDM_from_PMF_grid, sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    quiet(ra.set_TDM_from_PMF_grid, sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    rp = quiet(RMPPI, rcfg)
    rp.setup(p, rl, ra)
    N, T = sc["N"], sc["T"]
    V = min(N, 4096)
    (res_d, xl_d, yl_d, vr_d, wr_d, xg_d, vpost_d, tol_d, lam_d, ustd_d, cvar_d, x0_d, dt_d, obs_c, unk_c) = \
        rp.move_mppi_task_vars_to_device()
    lin_g = rl.sample_grids(1.0)
    ang_g = ra.sample_grids(1.0)
    RMPPI.sample_noise_numba[N, T](rp.rng_states_d, ustd_d, rp.noise_samples_d)
    u0 = np.stack([np.linspace(0.5, 2.5, T), np.linspace(-0.5, 0.5, T)], 1).astype(f32)
    u_d = cuda.to_device(u0)
    out_d = cuda.device_array((V, T + 1, 3), dtype=f32)
    RMPPI.get_state_rollout_across_control_noise[V, 1](
        out_d, lin_g, ang_g, rl.bin_values_bounds_d, ra.bin_values_bounds_d, res_d, xl_d, yl_d, x0_d, dt_d,
        rp.noise_samples_d, vr_d, wr_d, u_d, u_d)
    ref_states = out_d.copy_to_host()
    noise = rp.noise_samples_d.copy_to_host()
    gl, ga = lin_g.copy_to_host(), ang_g.copy_to_host()

    Rmax, Cmax = sc["cfg"]["max_map_dim"]
    e = RawPlanner(E, 1, N, 1, T, Rmax, Cmax, V=V)
    pad_pmf = rl.pmf_grid_d.copy_to_host()
    for which in ("lin", "ang"):
        e.set_map(which, pad_pmf, rl.bin_values, rl.bin_values_bounds, rl.res, rl.padded_xlimits, rl.padded_ylimits,
                  rl.obstacle_map_d.copy_to_host(), rl.unknown_map_d.copy_to_host())
    e.set_grids("lin", gl)
    e.set_grids("ang", ga)
    e.copy_in(E._lib.BUF_NOISE, noise)
    e.copy_in(E._lib.BUF_U_CUR, u0)
    e.copy_in(E._lib.BUF_U_PREV, u0)
    e.set_params(x0=list(np.asarray(p["x0"], dtype=f32)), xgoal=list(np.asarray(p["xgoal"], dtype=f32)), dt=0.1)
    mine = np.empty((V, T + 1, 3), dtype=f32)
    E._lib.check(E._lib.lib.b200mppi_planner_get_state_rollout(e.pl, E._lib.ptr(mine), mine.nbytes))
    same = (mine == ref_states).all(axis=(1, 2))
    res = {"workload": name, "V": V, "bit_identical_rollouts": int(same.sum())}
    cases = []
    xlo, ylo, rs = f32(rl.padded_xlimits[0]), f32(rl.padded_ylimits[0]), f32(rl.res)
    for b in np.where(~same)[0][:12]:
        t = int(np.argmax((mine[b] != ref_states[b]).any(axis=1)))       # first differing state index
        prev = ref_states[b, t - 1]
        ax, ay = f32(prev[0] - xlo), f32(prev[1] - ylo)
        cases.append(dict(b=int(b), first_diff_step=t, prev_state=[float(v) for v in prev],
                          prev_state_hex=[hex(int(np.float32(v).view(np.uint32))) for v in prev],
                          ref=[float(v) for v in ref_states[b, t]], mine=[float(v) for v in mine[b, t]],
                          ax_over_res=float(np.float64(ax) / np.float64(rs)), ay_over_res=float(np.float64(ay) / np.float64(rs)),
                          ax_hex=hex(int(ax.view(np.uint32))), ay_hex=hex(int(ay.view(np.uint32)))))
    res["cases"] = cases
    os.makedirs(out_dir(), exist_ok=True)
    out = os.path.join(out_dir(), "trace_%s.json" % name)
    json.dump(res, open(out, "w"), indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
