"""Window-first map sampling (include/b200mppi.h, b200mppi_planner_sample_window): solve() samples only the rollout
window plus a ring up front, flags the maps whose rollouts read outside it, completes those maps and reruns their
rollouts.  Against whole-map sampling over a closed loop with a moving robot, everything a solve writes is
bit-identical, with and without escapes, and sample_box() reports the reach box a reach-box solve samples."""
import numpy as np
import pytest

from tests.gpu_harness import eng, tdm_planner  # noqa: F401
from tests.scenarios import make_scenario

pytestmark = pytest.mark.gpu


def _loop(pl, sc, steps, dx):
    lin, ang = pl.lin_tdm, pl.ang_tdm
    x0 = sc["params"]["x0"].copy()
    hist = []
    for _ in range(steps):
        l0 = pl.launch_count()
        u = pl.solve()
        hist.append(dict(u=u.copy(), costs=pl.costs_d.copy_to_host(), costs_nm=pl.costs_nm_d.copy_to_host(),
                         noise=pl.noise_samples_d.copy_to_host(), rng=pl.rng_states_d.copy_to_host(),
                         lin_rng=lin.rng_states_d.copy_to_host(), ang_rng=ang.rng_states_d.copy_to_host(),
                         box=pl.sample_box(), window=pl.sample_window(), launches=pl.launch_count() - l0))
        x0 = x0 + np.asarray(dx)
        pl.shift_and_update(x0, u, 1)
    grids = (lin.sample_grid_batch_d.copy_to_host(), ang.sample_grid_batch_d.copy_to_host())
    return hist, grids


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "%s: %d of %d elements differ" % (
        what, int((a != b).sum()), a.size)


def _compare(runs, mode):
    ref, got = runs["off"], runs[mode]
    for k, (h0, h1) in enumerate(zip(ref[0], got[0])):
        for key in ("u", "costs", "costs_nm", "noise", "rng", "lin_rng", "ang_rng"):
            _same(h1[key], h0[key], "solve %d: %s" % (k, key))
    _same(got[1][0], ref[1][0], "lin maps")
    _same(got[1][1], ref[1][1], "ang maps")


@pytest.mark.parametrize("escape", [False, True])
def test_window_first_identical_to_whole_maps(eng, monkeypatch, escape):  # noqa: F811
    T = 128
    sc = make_scenario("tdm", N=1024, M=32, T=T, H=600, W=600, res=0.1, B=12, seed=7)
    params = dict(sc["params"])
    if escape:
        # heading +x at full speed from the first solve: the rollouts run ~38 m, far past the window's 12 m
        params["x0"] = np.array([params["x0"][0], params["x0"][1], 0.0])
        sc["u0"] = np.stack([np.full(T, 3.0), np.zeros(T)], 1).astype(np.float32)
        sc["params"] = params
    runs = {}
    for mode in ("off", "dynamic", None):
        monkeypatch.delenv("B200MPPI_SAMPLE_BOX", raising=False)
        pl = tdm_planner(eng, sc, box=mode, monkeypatch=monkeypatch)
        runs[mode or "window"] = _loop(pl, sc, 4, [0.37, -0.21, 0.05])
    _compare(runs, "window")
    _compare(runs, "dynamic")
    win = runs["window"][0]
    assert all(h["window"][0] == 1 for h in win), [h["window"] for h in win]
    assert all(h["launches"] == 8 for h in win), [h["launches"] for h in win]
    # sample_box() keeps its meaning: the reach box a reach-box solve samples
    assert [h["box"] for h in win] == [h["box"] for h in runs["dynamic"][0]]
    flagged = [h["window"][5] for h in win]
    if escape:
        assert flagged[0] > 0, flagged
    else:
        assert flagged == [0] * 4, flagged
    for h in win:
        r0, r1, c0, c1 = h["window"][1:5]
        assert 0 <= r0 < r1 <= 600 + 10 and 0 <= c0 < c1 <= 600 + 10


def test_window_first_some_maps_escape(eng, monkeypatch):  # noqa: F811
    """Every rollout drives straight along one row through a gate cell whose linear traction is 0 with probability
    0.9 and 1 otherwise (every other cell: 1).  A closed gate stops every rollout of that map inside the window; an open
    one lets them all run out of it.  Steps are shorter than a cell, so no rollout skips the gate.  So exactly the maps
    whose sampled gate cell is open escape: the flag count must equal their number, some but not all of the M maps
    (the redo takes the u-th flagged map, the completion skips groups of maps without a flag), and everything a solve
    writes must be bit-identical to whole-map sampling."""
    T, M, res, H = 200, 64, 0.4, 600
    sc = make_scenario("tdm", N=256, M=M, T=T, H=H, W=H, res=res, B=2, seed=5)
    gate_r, gate_c = 300, 340                         # PMF cell of the gate, 40 cells ahead of the robot
    sc["pmf_lin"][:, gate_r, gate_c] = [90, 10]
    x0 = np.array([300 * res + res / 2, gate_r * res + res / 2, 0.0])
    sc["obstacle"][:] = 0
    sc["params"] = dict(sc["params"], x0=x0, xgoal=x0[:2] + np.array([150.0, 0.0]), u_std=np.array([0.2, 0.001]))
    u0 = np.stack([np.full(T, 3.0), np.zeros(T)], 1).astype(np.float32)
    pad = int(np.ceil(5.0 * 0.1 / res))
    runs = {}
    for mode in ("off", None):
        monkeypatch.delenv("B200MPPI_SAMPLE_BOX", raising=False)
        pl = tdm_planner(eng, sc, box=mode, monkeypatch=monkeypatch)
        lin, ang = pl.lin_tdm, pl.ang_tdm
        hist = []
        for _ in range(4):
            pl.u_cur_d.copy_to_device(u0)
            u = pl.solve()
            lg = lin.sample_grid_batch_d.copy_to_host()
            hist.append(dict(u=u.copy(), costs=pl.costs_d.copy_to_host(), costs_nm=pl.costs_nm_d.copy_to_host(),
                             noise=pl.noise_samples_d.copy_to_host(), rng=pl.rng_states_d.copy_to_host(),
                             lin_rng=lin.rng_states_d.copy_to_host(), ang_rng=ang.rng_states_d.copy_to_host(),
                             lin=lg, ang=ang.sample_grid_batch_d.copy_to_host(), window=pl.sample_window(),
                             open=int((lg[:, gate_r + pad, gate_c + pad] != 0).sum())))
        runs[mode or "window"] = hist
    partial = 0
    for k, (h0, h1) in enumerate(zip(runs["off"], runs["window"])):
        for key in ("u", "costs", "costs_nm", "noise", "rng", "lin_rng", "ang_rng", "lin", "ang"):
            _same(h1[key], h0[key], "solve %d: %s" % (k, key))
        assert h1["window"][0] == 1
        assert h1["window"][5] == h1["open"], (k, h1["window"], h1["open"])
        partial += 0 < h1["open"] < M
    assert partial >= 3, [h["open"] for h in runs["window"]]


def test_window_first_fallbacks(eng, monkeypatch):  # noqa: F811
    """Maps no larger than the window, and num_opt != 1, keep the reach-box path."""
    small = make_scenario("tdm", N=256, M=8, T=32, H=100, W=100, res=0.1, B=12, seed=3)
    pl = tdm_planner(eng, small, monkeypatch=monkeypatch)
    pl.solve()
    assert pl.sample_window()[0] == 0
    sc = make_scenario("tdm", N=256, M=8, T=32, H=400, W=400, res=0.1, B=12, seed=3)
    p2 = dict(sc["params"], num_opt=2)
    pl = tdm_planner(eng, sc, params=p2, monkeypatch=monkeypatch)
    pl.solve()
    assert pl.sample_window()[0] == 0
    pl = tdm_planner(eng, sc, monkeypatch=monkeypatch)
    pl.solve()
    assert pl.sample_window()[0] == 1
