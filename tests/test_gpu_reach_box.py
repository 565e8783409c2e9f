"""The reach box where it is tight (run with ``-m gpu``): boxed map sampling (B200MPPI_SAMPLE_BOX static / dynamic)
against whole maps (off), bit for bit, for rollouts that run the full reach -- straight lines (w = 0) with every step's
displacement between 0.5 and 1.5 ulp of the coordinate on maps far from the origin, where float32 rounding makes the
robot move up to twice as far as its exact path -- and at the reach disc's edge near the origin.

Before every sampling both TDMs' sampled maps are filled with byte 0 (traction 0) while every sampled cell decodes to
traction 1 inside the map: a rollout that reads a cell the boxed launch did not write stops there, which changes its
cost."""
import numpy as np
import pytest

from tests.gpu_harness import assert_same, eng, quiet, tdm_planner  # noqa: F401

pytestmark = pytest.mark.gpu


# origin (both axes), res, map cells a side, T, start inside the map (m), heading, vrange, u_cur[v], u_std[v]
CASES = {
    "far": (4096.0, 0.01, 256, 512, 1.2, np.pi / 2, (0.0025, 0.003), 0.00275, 2e-4),
    "utm": (4.0e5, 0.1, 128, 64, 5.0, np.pi / 2, (0.16, 0.17), 0.165, 0.004),
    "disc": (0.0, 0.1, 256, 32, 12.8, np.pi / 4, (0.0, 3.0), 3.0, 0.3),
}


def scenario(case, seed=3, heading=None):
    origin, res, cells, T, inside, th, vr, u, us = CASES[case]
    dt = 0.1
    pad = int(np.ceil(5.0 * dt / res))
    cfg = dict(T=T * dt + dt / 2, dt=dt, num_grid_samples=4, num_control_rollouts=64, seed=seed,
               max_map_dim=(cells + 2 * pad, cells + 2 * pad), tdm_sample_thread_dim=(16, 16), max_speed_padding=5.0,
               num_vis_state_rollouts=4, use_tdm=True)
    pmf = np.zeros((2, cells, cells), dtype=np.int8)
    pmf[1] = 100                                             # every map cell: traction 1 (padding: bin 0, traction 0)
    zero = np.zeros((cells, cells), dtype=np.int8)           # no obstacle, nothing unknown
    lim = np.array([origin, origin + cells * res])
    tdm_dict = dict(res=res, xlimits=lim, ylimits=lim, bin_values=np.array([0.0, 1.0]),
                    bin_values_bounds=np.array([0.0, 1.0]), det_dynamics_cvar_alpha=1.0)
    x0 = np.array([origin + inside, origin + inside, th if heading is None else heading])
    params = dict(dt=dt, x0=x0, xgoal=x0[:2] - 50.0, goal_tolerance=0.01, v_post_rollout=0.01, cvar_alpha=0.5,
                  alpha_dyn=1.0, dist_weight=1.0, lambda_weight=1.0, num_opt=1, u_std=np.array([us, 0.1]),
                  vrange=np.array(vr), wrange=np.array([0.0, 0.0]))
    u0 = np.zeros((T, 2), dtype=np.float32)
    u0[:, 0] = u
    return dict(cfg=cfg, pmf_lin=pmf, pmf_ang=pmf, obstacle=zero, unknown=zero, tdm_dict=tdm_dict, params=params, u0=u0,
                T=T, res=res, cells=cells, lim=lim)


def planner(E, sc, box, monkeypatch):
    with quiet():
        return tdm_planner(E, sc, box=box, monkeypatch=monkeypatch)


def zero_maps(pl):
    for t in (pl.lin_tdm, pl.ang_tdm):
        t.sample_grid_batch_d.copy_to_device(np.zeros(t.sample_grid_batch_d.shape, dtype=np.int8))


def closed_loop(E, sc, box, monkeypatch, solves=3):
    pl = planner(E, sc, box, monkeypatch)
    hist, boxes = [], []
    x = np.asarray(sc["params"]["x0"], dtype=np.float64)
    with quiet():
        for _ in range(solves):
            zero_maps(pl)
            u = pl.solve()
            boxes.append(pl.sample_box())
            hist.append(dict(u=u.copy(), costs=pl.costs_d.copy_to_host(), costs_nm=pl.costs_nm_d.copy_to_host(),
                             noise=pl.noise_samples_d.copy_to_host(), rng=pl.rng_states_d.copy_to_host(),
                             lin_rng=pl.lin_tdm.rng_states_d.copy_to_host(),
                             ang_rng=pl.ang_tdm.rng_states_d.copy_to_host()))
            step = sc["params"]["dt"] * float(u[0, 0])       # plant step on traction 1
            x = x + np.array([step * np.cos(x[2]), step * np.sin(x[2]), 0.0])
            pl.shift_and_update(x, u, 1)
    return hist, boxes


def assert_boxed_equals_off(E, sc, monkeypatch):
    ref, ref_boxes = closed_loop(E, sc, "off", monkeypatch)
    assert all(b[0] == 0 for b in ref_boxes)
    for box, how in (("static", 1), ("dynamic", 2)):
        hist, boxes = closed_loop(E, sc, box, monkeypatch)
        assert all(b[0] == how for b in boxes), (box, boxes)  # a real box, not whole maps
        side = sc["cells"] + 2 * int(np.ceil(0.5 / sc["res"]))
        assert all(b[2] - b[1] < side and b[4] - b[3] < side for b in boxes), (box, boxes)
        for k, (h, h0) in enumerate(zip(hist, ref)):
            assert_same(h, h0, "%s solve %d, against whole-map sampling (box %s)" % (box, k, boxes[k]))


@pytest.mark.parametrize("case", ["far", "utm"])
def test_far_origin_boxed_solve_equals_whole_maps(eng, monkeypatch, case):
    """A map at 4096 m at 1 cm (T 512, 0.5 - 0.6 ulp per step) and one at 4e5 m at 10 cm (T 64): every step rounds to a
    whole ulp, so the rollouts travel up to twice dt * traction * sum |v|.  Per-(n, m) and CVaR costs, u, noise and every
    RNG state equal whole-map sampling's."""
    assert_boxed_equals_off(eng, scenario(case), monkeypatch)


def test_disc_edge_boxed_solve_equals_whole_maps(eng, monkeypatch):
    """Near the origin, heading pi/4 at the speed limit on traction 1: the rollouts end on the reach disc, in the box
    corner the disc narrowing leaves out."""
    sc = scenario("disc")
    assert_boxed_equals_off(eng, sc, monkeypatch)


def _batch_twins(E, box, monkeypatch):
    scs = [scenario("far", seed=3), scenario("far", seed=8, heading=0.0)]
    return [planner(E, sc, box, monkeypatch) for sc in scs], scs


def test_device_decided_box_far_origin(eng, monkeypatch):
    """The batched trial sampler decides each planner's box on the device: run_stochastic_trials (K = 2, far-origin
    map) with the dynamic box against whole maps -- xhist, uhist, the sampled maps and every RNG state bit-identical --
    and MPPI_StochasticBatch.solve() the same way."""
    E = eng
    runs = {}
    for box in ("off", "dynamic"):
        pls, scs = _batch_twins(E, box, monkeypatch)
        grids = [E.TractionGrid(np.ones((sc["cells"], sc["cells"])), np.ones((sc["cells"], sc["cells"])), res=sc["res"],
                                xlimits=tuple(sc["lim"]), ylimits=tuple(sc["lim"])) for sc in scs]
        for p in pls:
            zero_maps(p)
        with quiet():
            out = E.MPPI_StochasticBatch(pls).run_stochastic_trials(grids, 4)
        assert list(out["steps"]) == [4, 4], out["status"]
        runs[box] = dict(xhist=out["xhist"], uhist=out["uhist"], boxes=[p.sample_box() for p in pls],
                         state=[dict(rng=p.rng_states_d.copy_to_host(), lin_rng=p.lin_tdm.rng_states_d.copy_to_host(),
                                     ang_rng=p.ang_tdm.rng_states_d.copy_to_host(),
                                     lin_map=p.lin_tdm.sample_grid_batch_d.copy_to_host(),
                                     ang_map=p.ang_tdm.sample_grid_batch_d.copy_to_host()) for p in pls])
    assert all(b[0] == 0 for b in runs["off"]["boxes"])
    assert all(b[0] == 2 for b in runs["dynamic"]["boxes"]), runs["dynamic"]["boxes"]
    assert_same({key: runs["dynamic"][key] for key in ("xhist", "uhist")},
                {key: runs["off"][key] for key in ("xhist", "uhist")}, "trials")
    for k in range(2):
        assert_same(runs["dynamic"]["state"][k], runs["off"]["state"][k], "trials, planner %d" % k)

    solved = {}
    for box in ("off", "dynamic"):
        pls, _ = _batch_twins(E, box, monkeypatch)
        batch = E.MPPI_StochasticBatch(pls)
        hist = []
        with quiet():
            for r in range(3):
                for p in pls:
                    zero_maps(p)
                u = batch.solve()
                hist.append(dict(u=u.copy(), boxes=[p.sample_box()[0] for p in pls],
                                 costs_nm=[p.costs_nm_d.copy_to_host() for p in pls],
                                 costs=[p.costs_d.copy_to_host() for p in pls],
                                 rng=[p.rng_states_d.copy_to_host() for p in pls],
                                 lin_rng=[p.lin_tdm.rng_states_d.copy_to_host() for p in pls]))
                for k, p in enumerate(pls):
                    x = np.asarray(p.params["x0"], dtype=np.float64)
                    step = p.params["dt"] * float(u[k, 0, 0])
                    p.shift_and_update(x + np.array([step * np.cos(x[2]), step * np.sin(x[2]), 0.0]), u[k], 1)
        solved[box] = hist
    for r, (h, h0) in enumerate(zip(solved["dynamic"], solved["off"])):
        assert h["boxes"] == [2, 2] and h0["boxes"] == [0, 0], (h["boxes"], h0["boxes"])
        assert_same(dict(u=h["u"]), dict(u=h0["u"]), "batch solve round %d" % r)
        for k in range(2):
            keys = ("costs_nm", "costs", "rng", "lin_rng")
            assert_same({key: h[key][k] for key in keys}, {key: h0[key][k] for key in keys},
                        "batch solve round %d planner %d" % (r, k))
