"""Window-first sampling through solve() at its edges (run with ``-m gpu``): ragged N (padding lanes over whatever
the allocator left in ctrl), maps larger than the window in one or both axes with the robot at the centre, the corners
and in the padding, the ring's boundary on all four sides, the 224-row window, one map, a map count that is no multiple
of the sampler's maps per CTA, masks 0..3, and closed loops that alternate solves with and without escapes between
public samplings, visualisation rollouts, new maps and a reach-box solve.

Before every solve both TDMs' sampled maps hold a sentinel code, so a rollout that trusted a byte outside the sampled
rectangle would read it.  Per window-first solve: every per-(n, m) cost equals the exact oracle (device provider) on
the maps the oracle samples whole from the pre-solve generator states, with the solve's noise and the pre-solve
controls; the CVaR stays within its bound; the flag count equals the escapes predicted from the oracle's trajectories
(tests/window_first_cases.py); the reported rectangle is the restated one and the solve issues 8 launches; u, noise,
every generator state and the completed maps are byte-identical to whole-map sampling (B200MPPI_SAMPLE_BOX=off) and
sample_box() reports what a reach-box (dynamic) solve reports."""
import numpy as np
import pytest

from oracle import terrain_ref as TR
from tests import reduce_bounds as RB
from tests import rollout_edge_cases as EC
from tests import window_first_cases as WF
from tests.gpu_harness import assert_all_equal, dev, eng, quiet, tdm_planner  # noqa: F401
from tests.scenarios import make_scenario, oracle_rollout_costs

pytestmark = pytest.mark.gpu

F32 = np.float32
SENTINEL = -77                       # no sampled code, and not -128 (the detecting kernel's escape code)
MODES = ("window", "off", "dynamic")
MOVING = np.array([0.0, 0.6, 0.7, 0.85, 1.0])    # bin values of the escape scenarios (bin 0 emptied by _moving)


def _moving(sc):
    """No traction-0 cell: bin 0's mass moved to bin 1, so no rollout stops before it can leave the window."""
    for key in ("pmf_lin", "pmf_ang"):
        sc[key][1] += sc[key][0]
        sc[key][0] = 0
    return sc


def _fill(pl):
    for t in (pl.lin_tdm, pl.ang_tdm):
        t.sample_grid_batch_d.copy_to_device(np.full(t.sample_grid_batch_d.shape, SENTINEL, np.int8))


def _planners(E, sc, monkeypatch):
    out = {}
    with quiet():
        for mode in MODES:
            monkeypatch.delenv("B200MPPI_SAMPLE_BOX", raising=False)
            out[mode] = tdm_planner(E, sc, box=None if mode == "window" else mode, monkeypatch=monkeypatch)
    return out


def _state(pl):
    lin, ang = pl.lin_tdm, pl.ang_tdm
    return dict(u=pl.u_cur_d.copy_to_host(), noise=pl.noise_samples_d.copy_to_host(), rng=pl.rng_states_d.copy_to_host(),
                lin_rng=lin.rng_states_d.copy_to_host(), ang_rng=ang.rng_states_d.copy_to_host(),
                lin_map=lin.sample_grid_batch_d.copy_to_host(), ang_map=ang.sample_grid_batch_d.copy_to_host())


def _solve(pls, sc, dev, what, expect_flags=None, sentinel_read=False):
    """One solve of the three twins with sentinel maps; every check of the module docstring.  Returns None when the
    window planner did not take window-first sampling, else dict(flags (the count), reads (WF.escapes), cells
    (WF.executed_cells), rows, cols, rect).  ``sentinel_read``: some escaping read lies outside the cells the
    window-first sampling writes, so the byte there is the sentinel until the completion."""
    pl = pls["window"]
    lin, ang = pl.lin_tdm, pl.ang_tdm
    u_pre = pl.u_cur_d.copy_to_host()
    st_pre = lin.rng_states_d.copy_to_host()
    fused = np.array_equal(st_pre, ang.rng_states_d.copy_to_host())
    snaps, us = {}, {}
    for mode in MODES:
        p = pls[mode]
        _fill(p)
        n0 = p.launch_count()
        with quiet():
            us[mode] = p.solve()
        snaps[mode] = dict(_state(p), box=np.asarray(p.sample_box()), window=np.asarray(p.sample_window()),
                           launches=p.launch_count() - n0)
    w = snaps["window"]
    for key in ("u", "noise", "rng", "lin_rng", "ang_rng", "lin_map", "ang_map"):
        assert w[key].tobytes() == snaps["off"][key].tobytes(), "%s: %s differs from whole-map sampling" % (what, key)
    assert us["window"].tobytes() == us["off"].tobytes(), what
    assert tuple(w["box"]) == tuple(snaps["dynamic"]["box"]), (what, w["box"], snaps["dynamic"]["box"])
    if w["window"][0] == 0:
        return None
    assert fused, what
    assert w["launches"] == 8, (what, w["launches"])
    # the oracle: both TDMs sampled whole from lin's pre-solve stream (the fused pair), on sentinel maps
    cfg_tile, M = lin.thread_dim, lin.sample_grid_batch_d.shape[0]
    grids = []
    for t in (lin, ang):
        g = np.full(t.sample_grid_batch_d.shape, SENTINEL, np.int8)
        TR.sample_grids(g, t.pmf_grid_d.copy_to_host(), st_pre.copy(), t.bin_values, t.bin_values_bounds,
                        float(pl.params.get("alpha_dyn", 1.0)), cfg_tile, M)
        grids.append(g)
    assert w["lin_map"].tobytes() == grids[0].tobytes() and w["ang_map"].tobytes() == grids[1].tobytes(), what
    want, states = oracle_rollout_costs(dict(sc, params=pl.params), lin, ang, w["noise"], u_pre, grids=grids, arith=dev,
                                        ctrl_order="presummed", wrap_clamp=True, return_states=True)
    costs_nm = pl.costs_nm_d.copy_to_host()
    assert_all_equal(costs_nm, want, what + ": costs")
    RB.check_cvar(pl.costs_d.copy_to_host(), costs_nm, float(pl.params["cvar_alpha"]), label=what)
    # the rectangle and the escapes
    rows, cols = lin.obstacle_map_d.shape
    x0 = pl.params["x0"]
    wx0, wy0, ww, wh = EC.window_origin(x0[0], x0[1], lin.padded_xlimits[0], lin.padded_ylimits[0], lin.res, cols,
                                        rows, EC.window_height(states.shape[2] - 1))
    rect = WF.window_rect(wx0, wy0, ww, wh, rows, cols)
    assert tuple(w["window"][1:5]) == rect, (what, w["window"], rect)
    flags, reads = WF.escapes(states, lin.padded_xlimits[0], lin.padded_ylimits[0], lin.res, pl.params["xgoal"],
                              pl.params["goal_tolerance"], rect, rows, cols, grids[0].shape[1], grids[0].shape[2], dev)
    assert w["window"][5] == int(flags.sum()), (what, w["window"], flags)
    if expect_flags is not None:
        assert int(flags.sum()) == expect_flags, (what, int(flags.sum()), expect_flags)
    if sentinel_read:                                 # an escape trusted without a flag would read the sentinel
        r0, r1, c0, c1 = WF.window_sampled(rect, cols, lin.thread_dim[1])
        assert any(not (r0 <= gy < r1 and c0 <= gx < c1) for *_, gy, gx in reads), (what, rect, reads[:4])
    cells = WF.executed_cells(states, lin.padded_xlimits[0], lin.padded_ylimits[0], lin.res, pl.params["xgoal"],
                              pl.params["goal_tolerance"], dev)
    return dict(flags=int(flags.sum()), reads=reads, cells=cells, rows=rows, cols=cols, rect=rect)


# ----------------------------------------------------------------------------- 1. ragged N
@pytest.mark.parametrize("N", [33, 200, 1000])
@pytest.mark.parametrize("escape", [False, True])
def test_ragged_n(eng, dev, monkeypatch, N, escape):
    import torch
    junk = torch.full((4 << 20,), float("nan"), device="cuda")      # best effort: leave NaN where ctrl may land
    del junk
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    T = 128
    sc = _moving(make_scenario("tdm", N=N, M=8, T=T, H=600, W=600, res=0.1, B=5, seed=11 + N, bin_values=MOVING))
    x0 = sc["params"]["x0"]
    sc["params"] = dict(sc["params"], x0=np.array([x0[0], x0[1], 0.3]), u_std=np.array([0.3, 0.3]))
    sc["u0"] = np.stack([np.full(T, 3.0 if escape else 0.4), np.zeros(T)], 1).astype(F32)
    pls = _planners(eng, sc, monkeypatch)
    r = _solve(pls, sc, dev, "N %d" % N)
    assert r is not None and (r["flags"] > 0) == escape, r and r["flags"]


# ----------------------------------------------------------------------------- 2. map edges
EDGE_MAPS = [c for c in EC.MAP_CASES if EC.padded_grid(*c)[0] > 232 or EC.padded_grid(*c)[1] > 240] + \
    [(600, 600, 0.1), (100, 600, 0.1), (600, 100, 0.1)]


def _crop(sc, rows, cols, res):
    """make_scenario draws square maps: keep the rows x cols corner."""
    pad = EC.pad_cells(res)
    for key in ("pmf_lin", "pmf_ang"):
        sc[key] = np.ascontiguousarray(sc[key][:, :rows, :cols])
    for key in ("obstacle", "unknown"):
        sc[key] = np.ascontiguousarray(sc[key][:rows, :cols])
    sc["tdm_dict"] = dict(sc["tdm_dict"], xlimits=np.array([0.0, cols * res]), ylimits=np.array([0.0, rows * res]))
    sc["cfg"] = dict(sc["cfg"], max_map_dim=(rows + 2 * pad, cols + 2 * pad))
    sc["params"] = dict(sc["params"], x0=np.array([cols * res / 2, rows * res / 2, 0.0]))
    return sc


# heading of each robot spot: out of the map across the nearest edge (the corners), so that steps of up to 1.2 m
# (dt 0.4 s) jump the 0.5 m of traction-0 padding: x < 0 from low-left, y < 0 from low-right (wrapped to the far side),
# y beyond the top from high-left, x beyond the right edge from high-right (clamped)
SPOT_HEADING = {"centre": 0.7, "low-left": np.pi, "low-right": -np.pi / 2, "high-left": np.pi / 2, "high-right": 0.0,
                "padding": -2.4}


@pytest.mark.parametrize("rows,cols,res", EDGE_MAPS, ids=["%dx%d" % c[:2] for c in EDGE_MAPS])
@pytest.mark.parametrize("spot", EC.MAP_SPOTS)
def test_map_edges(eng, dev, monkeypatch, rows, cols, res, spot):
    T, n = 100, max(rows, cols)
    sc = _moving(make_scenario("tdm", N=64, M=4, T=T, H=n, W=n, res=res, B=5, seed=41, bin_values=MOVING))
    if rows != cols:
        sc = _crop(sc, rows, cols, res)
    sc["params"] = dict(sc["params"], dt=0.4)
    sc["u0"] = np.stack([np.full(T, 3.0), np.zeros(T)], 1).astype(F32)
    x, y = EC.map_spot(spot, rows, cols, res, EC.pad_cells(res))
    pls = _planners(eng, sc, monkeypatch)
    for p in pls.values():                              # setup() takes x0 inside the map only; a closed loop goes anywhere
        p.params["x0"] = np.array([x, y, SPOT_HEADING[spot]])
    r = _solve(pls, sc, dev, "%dx%d %s" % (rows, cols, spot))
    assert r is not None
    R, C, (r0, r1, c0, c1), pad = r["rows"], r["cols"], r["rect"], EC.pad_cells(res)
    if spot == "low-left" and C - pad >= c1:            # every far-side cell a wrapped lane can land on is outside
        assert any(xi < 0 for _, _, _, _, xi, _, _ in r["reads"]), r["reads"][:4]
    if spot == "low-right" and R - pad >= r1:
        assert any(yi < 0 for _, _, _, yi, _, _, _ in r["reads"]), r["reads"][:4]
    if spot == "high-left":                             # clamped into the top row
        assert any((live & (yi >= R)).any() for live, yi, _ in r["cells"])
    if spot == "high-right":                            # clamped into the last column
        assert any((live & (xi >= C)).any() for live, _, xi in r["cells"])


# ----------------------------------------------------------------------------- 3. the ring's boundary
def _wall_scenario(side, past):
    """Straight rollouts (heading along +-x or +-y, u_std on w tiny, steps of at most 0.3 m on 0.4 m cells) from the
    centre of a 600 x 600 map towards a wall of traction-0 cells on the last ring row / column of that side (past
    False) or one cell beyond it (past True)."""
    T, res, H = 200, 0.4, 600
    sc = make_scenario("tdm", N=64, M=4, T=T, H=H, W=H, res=res, B=2, seed=5)
    pad = EC.pad_cells(res)
    sc["obstacle"][:] = 0
    sc["unknown"][:] = 0
    c = H // 2
    x0 = np.array([c * res + res / 2, c * res + res / 2, dict(px=0.0, nx=np.pi, py=np.pi / 2, ny=-np.pi / 2)[side]])
    wx0, wy0, ww, wh = EC.window_origin(x0[0], x0[1], -pad * res, -pad * res, res, H + 2 * pad, H + 2 * pad,
                                        EC.window_height(T))
    r0, r1, c0, c1 = WF.window_rect(wx0, wy0, ww, wh, H + 2 * pad, H + 2 * pad)
    line = dict(px=c1 - 1 + past, nx=c0 - past, py=r1 - 1 + past, ny=r0 - past)[side] - pad   # PMF coordinates
    if side in ("px", "nx"):
        sc["pmf_lin"][:, :, line] = [[100], [0]]
    else:
        sc["pmf_lin"][:, line, :] = [[100], [0]]
    d = np.array(dict(px=(1, 0), nx=(-1, 0), py=(0, 1), ny=(0, -1))[side], float)
    sc["params"] = dict(sc["params"], x0=x0, xgoal=x0[:2] + 200.0 * d, u_std=np.array([0.2, 0.001]))
    sc["u0"] = np.stack([np.full(T, 3.0), np.zeros(T)], 1).astype(F32)
    return sc


@pytest.mark.parametrize("side", ["px", "nx", "py", "ny"])
@pytest.mark.parametrize("past", [0, 1])
def test_ring_boundary(eng, dev, monkeypatch, side, past):
    sc = _wall_scenario(side, past)
    pls = _planners(eng, sc, monkeypatch)
    r = _solve(pls, sc, dev, "wall %s%s" % (side, " + 1" if past else ""), expect_flags=4 if past else 0,
               sentinel_read=bool(past) and side in ("py", "ny"))
    assert r is not None


# ----------------------------------------------------------------------------- 4. shapes
@pytest.mark.parametrize("N,M,T,masks03", [(64, 4, 703, False), (256, 1, 64, False), (128, 37, 48, False),
                                           (200, 8, 64, True)], ids=["T703", "M1", "M37", "masks03"])
def test_shapes(eng, dev, monkeypatch, N, M, T, masks03):
    sc = make_scenario("tdm", N=N, M=M, T=T, H=400, W=400, res=0.1, B=5, seed=17 + M, warm_start=True)
    if masks03:
        rng = np.random.default_rng(90)
        sc["obstacle"] = (rng.integers(0, 4, sc["obstacle"].shape) * (rng.random(sc["obstacle"].shape) < 0.05)).astype(np.int8)
    if T > 100:
        sc["params"]["vrange"] = np.array([0.0, 0.3])
    pls = _planners(eng, sc, monkeypatch)
    assert _solve(pls, sc, dev, "N %d M %d T %d" % (N, M, T)) is not None


def test_m2048(eng, dev, monkeypatch):
    """2048 maps (the large-M CVaR kernel; the completion counts the flags over eight 256-thread passes): N 32, T 16,
    steps of up to 15 cells (dt 0.5 s) heading +y from the centre of a 260 x 240 map, so most maps escape through the
    rectangle's top rows."""
    T = 16
    sc = _moving(_crop(make_scenario("tdm", N=32, M=2048, T=T, H=260, W=260, res=0.1, B=5, seed=3, bin_values=MOVING),
                       260, 240, 0.1))
    sc["params"] = dict(sc["params"], x0=np.array([120 * 0.1 + 0.05, 130 * 0.1 + 0.05, np.pi / 2]), dt=0.5,
                        u_std=np.array([0.3, 0.3]))
    sc["u0"] = np.stack([np.full(T, 3.0), np.zeros(T)], 1).astype(F32)
    pls = _planners(eng, sc, monkeypatch)
    r = _solve(pls, sc, dev, "M 2048", sentinel_read=True)
    assert r is not None and r["flags"] > 256, r and r["flags"]


# ----------------------------------------------------------------------------- 5. sequences
def test_closed_loop_flag_parities(eng, dev, monkeypatch):
    """Seven solves, escaping (E) or not (N): E, N, N, E, then one that takes the reach box (lin alone sampled in public:
    the pair is no longer fused), then N, N once ang's public sampling has brought the pair's streams together again.
    Between them: a public sampling of both TDMs, a visualisation rollout, new maps for both TDMs.  The flag buffer
    alternates between two parities from one window-first solve to the next, so solves 2 and 6 (N) reuse the buffers of
    solves 0 and 3 (E): a flag left over from two window-first solves back would show as a count above 0."""
    T = 128
    sc = _moving(make_scenario("tdm", N=200, M=8, T=T, H=600, W=600, res=0.1, B=5, seed=29, bin_values=MOVING))
    x0 = sc["params"]["x0"]
    sc["params"] = dict(sc["params"], x0=np.array([x0[0], x0[1], 0.0]), u_std=np.array([0.3, 0.3]))
    pls = _planners(eng, sc, monkeypatch)
    counts = []
    for k in range(7):
        u = np.stack([np.full(T, 3.0 if k in (0, 3) else 0.3), np.zeros(T)], 1).astype(F32)
        for p in pls.values():
            p.u_cur_d.copy_to_device(u)
            if k == 1:
                p.lin_tdm.sample_grids()
                p.ang_tdm.sample_grids()
            elif k == 2:
                with quiet():
                    p.get_state_rollout()
            elif k == 3:
                p.lin_tdm.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
                p.ang_tdm.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
            elif k == 4:
                p.lin_tdm.sample_grids()
            elif k == 5:
                p.ang_tdm.sample_grids()
        r = _solve(pls, sc, dev, "solve %d" % k)
        counts.append(None if r is None else r["flags"])
        for p in pls.values():
            p.params["x0"] = p.params["x0"] + np.array([0.11, -0.07, 0.0])
    assert counts[4] is None and all(c is not None for i, c in enumerate(counts) if i != 4), counts
    assert counts[0] > 0 and counts[3] > 0 and counts[1] == counts[2] == counts[5] == counts[6] == 0, counts
