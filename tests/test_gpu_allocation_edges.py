"""Maps smaller than their TDM allocation on the GPU (run with ``-m gpu``): max_map_dim is a capacity (the Config
default is 250 x 250, the reference benchmark runs an 11 x 11 padded map in a 15 x 15 allocation), so the kernels see
the sampled maps' geometry (allocation rows, columns and pitch) next to the masks' (the padded map's).  Every
allocation byte beyond the map holds a sentinel (tests/allocation_cases.py) or, after a map change, the samples of a
larger map; rollouts that leave the map read them through the wrap and the clamp.  Checked against the exact oracle
(device provider, wrap + clamp, the whole allocation as the sampled maps, the map-shaped masks), every element bit for
bit:

1. C-ABI rollouts in modes 0 (windowed and generic), 1 and 2 from the centre, the corners heading out and the padding,
   on allocations larger in rows, in columns and in both, and on a map larger than the window; the state rollouts of
   get_state_rollout; the allocation is unchanged afterwards.
2. Batches (MPPI_Batch of det / speed-map planners, MPPI_StochasticBatch) whose planners' allocations differ from their
   maps and from each other.
3. Window-first solves whose rollouts stay inside the sampled rectangle, escape into the map, or read beyond the map
   only through the wrap (no flag: those bytes are never sampled); a map change inside one allocation, whose rollouts
   are clamped onto the old map's samples beyond the new map.
4. A planner re-bound to a TDM pair of another allocation shape with the same byte count (the windowed rollout's
   tensor maps are keyed on the allocation shapes, not only on the buffer addresses).
5. The reference benchmark's shape (9 x 9 cells at 1 m in a 15 x 15 allocation) in a closed loop."""
import ctypes

import numpy as np
import pytest

from tests import allocation_cases as AC
from tests import reduce_bounds as RB
from tests import rollout_edge_cases as EC
from tests.gpu_harness import (RawPlanner, assert_all_equal, dev, eng, quiet, replay,  # noqa: F401
                               solve_in_batch_of_one, tdm_planner, tdm_scenario, vary)
from tests.scenarios import make_scenario, oracle_rollout_costs
from tests.test_gpu_window_first_edges import _planners, _solve

pytestmark = pytest.mark.gpu

F32 = np.float32


# ----------------------------------------------------------------------------- 1. raw C-ABI rollouts
def _launches(rp):
    n = ctypes.c_int64()
    rp.L.check(rp.lib.b200mppi_planner_launch_count(rp.pl, ctypes.byref(n)))
    return int(n.value)


def _bind(rp, s):
    """Map, masks, risk, the whole allocations, noise, controls and parameters of raw case s."""
    pxl, pyl = AC.limits(s)
    dummy = np.zeros((2, s["R"], s["C"]), np.int8)
    dummy[1] = 100
    rp.set_map("lin", dummy, [0.0, 1.0], s["lb"], s["res"], pxl, pyl, s["obs"], s["unk"], s["risk"] if s["mode"] == 2 else None)
    rp.set_map("ang", dummy, [0.0, 1.0], s["ab"], s["res"], pxl, pyl, s["obs"], s["unk"], None)
    rp.set_grids("lin", s["lin"])
    rp.set_grids("ang", s["ang"])
    rp.copy_in(rp.L.BUF_NOISE, s["noise"])
    rp.copy_in(rp.L.BUF_U_CUR, s["u_cur"])
    rp.copy_in(rp.L.BUF_U_PREV, s["u_prev"])
    rp.set_params(x0=list(s["x0"]), xgoal=list(s["goal"]), goal_tolerance=s["tol"], vrange=list(s["vrange"]),
                  dt=float(s["dt"]), cvar_alpha=s["alpha"])


def _costs(rp, s, launches=None):
    """One rollout stage: per-(n, m) costs (mode 0) or costs (N, 1); `launches`: what it must issue."""
    before = _launches(rp)
    rp.call("rollout")
    assert launches is None or _launches(rp) - before == launches, "the rollout stage took another kernel"
    if s["mode"] == 0:
        return rp.copy_out(rp.L.BUF_COSTS_NM, (s["N"], s["M"]))
    return rp.copy_out(rp.L.BUF_COSTS, (s["N"],))[:, None]


VARIANTS = ["window", "generic", "mode1", "mode2"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("geom", list(AC.GEOMETRIES))
def test_raw_rollouts(eng, dev, monkeypatch, geom, variant):
    """Mode 0 windowed (3 launches: controls, windowed rollout, CVaR) and generic (B200MPPI_NO_WINDOW: rollout,
    CVaR), modes 1 and 2; then V state rollouts; the allocation is left as set."""
    mode = dict(window=0, generic=0, mode1=1, mode2=2)[variant]
    V = 8
    for spot in AC.SPOTS:
        s = AC.raw_case(geom, spot, mode)
        if variant == "generic":
            monkeypatch.setenv("B200MPPI_NO_WINDOW", "1")
        rp = RawPlanner(eng, mode, s["N"], s["M"], s["T"], s["Rmax"], s["Cmax"], V=V)
        monkeypatch.delenv("B200MPPI_NO_WINDOW", raising=False)
        try:
            _bind(rp, s)
            got = _costs(rp, s, dict(window=3, generic=2).get(variant))
            vis = np.empty((V, s["T"] + 1, 3), F32)
            rp.call("get_state_rollout", rp.L.ptr(vis), vis.nbytes)
            after = rp.get_grids("lin"), rp.get_grids("ang")
            cvar = rp.copy_out(rp.L.BUF_COSTS, (s["N"],))
        finally:
            rp.close()
        what = "%s %s %s" % (geom, spot, variant)
        order = "sequential" if variant == "generic" else None
        assert_all_equal(got, AC.oracle(s, dev, ctrl_order=order), what)
        assert_all_equal(vis, AC.state_oracle(s, V, dev), what + ": state rollouts")
        assert after[0].tobytes() == s["lin"].tobytes() and after[1].tobytes() == s["ang"].tobytes(), what
        if mode == 0:
            RB.check_cvar(cvar, got, s["alpha"], label=what)


# ----------------------------------------------------------------------------- 2. batches
def _grow(sc, extra):
    """Scenario sc in an allocation `extra` = (rows, cols) larger than its padded map."""
    R, C = sc["cfg"]["max_map_dim"]
    return dict(sc, cfg=dict(sc["cfg"], max_map_dim=(R + extra[0], C + extra[1])))


BATCH_MAPS = [(24, 0.2, (5, 19)), (37, 0.1, (13, 0)), (9, 0.5, (0, 6))]     # (cells, res, allocation beyond the map)


def _batch_scenarios(mode, N=256, M=8, T=40):
    """Planner k starts in the map's first cell heading out of it: steps of up to 1.2 m (dt 0.4 s, forward controls
    2.5 m/s) jump its traction-0 padding, so rollouts read beyond the map in the axis its allocation extends."""
    scs = []
    for k, (n, res, extra) in enumerate(BATCH_MAPS):
        sc = _grow(make_scenario(mode, N=N, M=M, T=T, H=n, W=n + 3 * k, res=res, B=5, seed=71 + k), extra)
        sc["params"]["x0"] = np.array([0.6 * res, 0.4 * res, [3.6, -1.9, np.pi][k]])
        sc["params"]["dt"] = 0.4
        sc["u0"] = np.stack([np.full(T, 2.5), np.zeros(T)], 1).astype(F32)
        scs.append(sc)
    return scs


@pytest.mark.parametrize("mode", ["det", "spd", "tdm"])
def test_batches_against_oracle(eng, dev, mode):
    """One MPPI_Batch (det, spd) or MPPI_StochasticBatch (tdm) solve, num_opt 1: each planner's costs from its
    pre-solve u_cur, the noise it drew and its maps as read after the solve."""
    scs = _batch_scenarios(mode)
    with quiet():
        pls = [tdm_planner(eng, sc) for sc in scs]
        u0 = [p.u_cur_d.copy_to_host() for p in pls]
        (eng.MPPI_StochasticBatch if mode == "tdm" else eng.MPPI_Batch)(pls).solve()
    shapes = set()
    for k, (sc, p) in enumerate(zip(scs, pls)):
        lin, ang = p.lin_tdm, p.ang_tdm
        gl, ga = lin.sample_grid_batch_d.copy_to_host(), ang.sample_grid_batch_d.copy_to_host()
        assert gl.shape[1:] != lin.obstacle_map_d.shape
        shapes.add(gl.shape[1:])
        want, states = oracle_rollout_costs(sc, lin, ang, p.noise_samples_d.copy_to_host(), u0[k], grids=(gl, ga),
                                            arith=dev, ctrl_order="presummed" if mode == "tdm" else "sequential",
                                            wrap_clamp=True, return_states=True)
        R, C = lin.obstacle_map_d.shape
        reads = AC.beyond_reads(states, dict(xlo=lin.padded_xlimits[0], ylo=lin.padded_ylimits[0], res=lin.res, R=R, C=C,
                                             Rmax=gl.shape[1], Cmax=gl.shape[2]), dev)
        assert any(reads.values()), "%s batch, planner %d: no read beyond the map" % (mode, k)
        if mode == "tdm":
            got = p.costs_nm_d.copy_to_host()
            RB.check_cvar(p.costs_d.copy_to_host(), got, sc["params"]["cvar_alpha"], label="planner %d" % k)
        else:
            got = p.costs_d.copy_to_host()[:, None]
        assert_all_equal(got, want, "%s batch, planner %d" % (mode, k))
    assert len(shapes) == len(scs)


# ----------------------------------------------------------------------------- 3. window-first solves
def _keep(p):
    return dict(lin=p.lin_tdm.sample_grid_batch_d.copy_to_host(), ang=p.ang_tdm.sample_grid_batch_d.copy_to_host())


def _place(pls, case):
    x0, u = AC.wf_start(case)
    for p in pls.values():
        p.params["x0"] = x0.copy()
        p.u_cur_d.copy_to_device(u)


def _check_wf(r, case, what):
    """The outcome WF_CASES states: flagged or not, reads beyond the map or not.  Returns the beyond-map cells read."""
    assert r is not None, what
    hit = AC.beyond_cells(r["cells"], r["rows"], r["cols"], (r["states"].shape[1],) + AC.WF_ALLOC)
    flagged, beyond = AC.WF_CASES[case][-1]
    assert (r["flags"] > 0) == flagged, (what, r["flags"])
    assert beyond is None or hit.any() == beyond, what
    return hit


@pytest.mark.parametrize("case", [c for c in AC.WF_CASES if c != "old-samples"])
def test_window_first(eng, dev, monkeypatch, case):
    sc = AC.wf_scenario(*AC.WF_MAP)
    pls = _planners(eng, sc, monkeypatch)
    _place(pls, case)
    lin = pls["window"].lin_tdm
    shape, (rows_p, cols_p) = lin.sample_grid_batch_d.shape, lin.obstacle_map_d.shape
    _check_wf(_solve(pls, sc, dev, case, fill=lambda p: AC.sentinel_grids(shape, rows_p, cols_p)), case, case)


def test_map_change_inside_one_allocation(eng, dev, monkeypatch):
    """An escaping solve on the large map; reset() and the small map in the same allocation, whose rollouts run off its
    right edge and are clamped onto the large map's old samples (unflagged); then the large map again.  The pre-solve
    maps are what the allocation holds, so the oracle samples over the old bytes."""
    sc = AC.wf_scenario(*AC.WF_MAP)
    pls = _planners(eng, sc, monkeypatch)
    _place(pls, "escape")
    _check_wf(_solve(pls, sc, dev, "large map", fill=_keep), "escape", "large map")

    def rebind(m):
        for p in pls.values():
            lin, ang, params = p.lin_tdm, p.ang_tdm, dict(p.params)
            with quiet():
                p.reset()
                lin.reset()
                ang.reset()
                lin.set_TDM_from_PMF_grid(m["pmf_lin"], m["tdm_dict"], m["obstacle"], m["unknown"])
                ang.set_TDM_from_PMF_grid(m["pmf_ang"], m["tdm_dict"], m["obstacle"], m["unknown"])
                p.setup(dict(params, x0=np.array([1.0, 1.0, 0.0])), lin, ang)
    rebind(AC.wf_scenario(*AC.WF_SMALL))
    _place(pls, "old-samples")
    old = _keep(pls["window"])
    r = _solve(pls, sc, dev, "small map", fill=_keep)
    hit = _check_wf(r, "old-samples", "small map")
    assert (r["rows"], r["cols"]) == (AC.WF_SMALL[0] + 10, AC.WF_SMALL[1] + 10)
    sampled = np.zeros(hit.shape, bool)
    sampled[:, :AC.WF_MAP[0] + 10, :AC.WF_MAP[1] + 10] = True             # where the large padded map was sampled
    assert (hit & sampled & (old["lin"] != 0)).any(), "no read lands on the large map's samples"
    rebind(sc)
    _place(pls, "escape")
    _check_wf(_solve(pls, sc, dev, "large map again", fill=_keep), "escape", "large map again")


# ----------------------------------------------------------------------------- 4. re-binding to another shape
def test_rebind_to_another_allocation_shape(eng, dev):
    """Solve on a 64 x 80 allocation; destroy the TDM pair; create a 80 x 64 pair (the same bytes), set_tdms; solve
    again.  The windowed rollout's tensor maps must be encoded for the new shape even where cudaMalloc hands back the
    freed addresses."""
    s = AC.raw_case("both", "low-left", 0, N=256, M=8, T=100)
    rows, cols = s["R"], s["C"]
    L = eng._lib
    rp = RawPlanner(eng, 0, s["N"], s["M"], s["T"], 64, 80)
    try:
        results, bases = [], []
        for Rmax, Cmax in ((64, 80), (80, 64)):
            if Rmax != rp.Rmax:
                rp.lib.b200mppi_tdm_destroy(rp.lin)
                rp.lib.b200mppi_tdm_destroy(rp.ang)
                rp.lin, rp.ang = ctypes.c_void_p(), ctypes.c_void_p()
                pod = L.ConfigPOD.from_buffer_copy(rp.pod)
                pod.max_map_rows, pod.max_map_cols = Rmax, Cmax
                L.check(rp.lib.b200mppi_tdm_create(ctypes.byref(pod), ctypes.byref(rp.lin)))
                L.check(rp.lib.b200mppi_tdm_create(ctypes.byref(pod), ctypes.byref(rp.ang)))
                rp.Rmax, rp.Cmax = Rmax, Cmax
            for w in ("lin", "ang"):
                g = AC.fill_beyond(np.zeros((s["M"], Rmax, Cmax), np.int8), rows, cols, w)
                g[:, :rows, :cols] = s[w][:, :rows, :cols]
                s[w] = g
            s["Rmax"], s["Cmax"] = Rmax, Cmax
            _bind(rp, s)
            base, pitch = ctypes.c_void_p(), ctypes.c_int32()
            L.check(rp.lib.b200mppi_tdm_sample_grid_view(rp.lin, ctypes.byref(base), ctypes.byref(pitch)))
            bases.append(base.value)
            results.append((_costs(rp, s, 3), AC.oracle(s, dev)))
    finally:
        rp.close()
    print("\n[rebind] lin grid base %#x -> %#x: %s" % (bases[0], bases[1],
                                                       "old address reused" if bases[0] == bases[1] else "new address"))
    for k, (got, want) in enumerate(results):
        assert_all_equal(got, want, "allocation %s" % ["64 x 80", "80 x 64"][k])


# ----------------------------------------------------------------------------- 5. the reference benchmark's shape
def _bench_setup(E, k, N=1024, M=1024, T=100):
    """tdm_trial_setup's planners 1 (nearby goal) and 2 (goal out of reach) on 9 x 9 cells at 1 m (11 x 11 padded) in
    a 15 x 15 allocation."""
    sc = tdm_scenario(k, N=N, M=M, T=T, H=9, res=1.0)
    sc["cfg"] = dict(sc["cfg"], max_map_dim=(15, 15))
    p = sc["params"]
    x0 = np.asarray(p["x0"], dtype=np.float64)
    p["xgoal"] = x0[:2] + (np.array([0.9, -0.4]) if k == 1 else 50.0)
    pl = tdm_planner(E, vary(sc, k))
    rng = np.random.default_rng(300 + k)
    return pl, E.TractionGrid(rng.uniform(0.2, 1.0, (9, 9)), rng.uniform(0.2, 1.0, (9, 9)), res=1.0), sc


def test_reference_benchmark_shape(eng, dev):
    """The first step's per-(n, m) costs against the oracle (on the maps where CTA shares begin and end), then
    run_stochastic_trials against the host loop."""
    import torch
    with quiet():
        p, _, sc = _bench_setup(eng, 2)
        u0 = p.u_cur_d.copy_to_host()
        eng.MPPI_StochasticBatch([p]).solve()
    lin, ang = p.lin_tdm, p.ang_tdm
    assert lin.sample_grid_batch_d.shape[1:] == (15, 15) and lin.obstacle_map_d.shape == (11, 11)
    maps = EC.share_edge_maps(1024, 1024, torch.cuda.get_device_properties(0).multi_processor_count, limit=8)
    gl, ga = lin.sample_grid_batch_d.copy_to_host()[maps], ang.sample_grid_batch_d.copy_to_host()[maps]
    want = oracle_rollout_costs(sc, lin, ang, p.noise_samples_d.copy_to_host(), u0, grids=(gl, ga), arith=dev,
                                ctrl_order="presummed", wrap_clamp=True)
    assert_all_equal(p.costs_nm_d.copy_to_host()[:, maps], want, "benchmark shape, first step")
    with quiet():
        first = [_bench_setup(eng, k) for k in (1, 2)]
        A, grids = [f[0] for f in first], [f[1] for f in first]
        B = [_bench_setup(eng, k)[0] for k in (1, 2)]
        out = eng.MPPI_StochasticBatch(A).run_stochastic_trials(grids, 3)
    replay(A, B, out, solve_in_batch_of_one, check_next=False)
