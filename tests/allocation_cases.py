"""Maps smaller than their allocation (TEST INFRASTRUCTURE): the geometries, sentinels and directed rollout inputs of
tests/test_gpu_allocation_edges.py and tests/test_allocation_cases_cpu.py.

A TDM's sampled maps live in an allocation of max_map_dim = (Rmax, Cmax) rows and columns, row pitch
round_up(Cmax, 16); the padded map it holds has rows x cols cells and its obstacle / unknown / risk planes have row
pitch round_up(cols, 16).  When the allocation is larger than the map the kernels work with both geometries at once: a
cell index outside the map wraps (negative) and clamps by (Rmax, Cmax) for the sampled maps and by (rows, cols) for
the masks (csrc/rollout.cu wrap_clamp, csrc/rollout_win.cu lookup_slow), so a rollout that leaves the map reads
allocation bytes beyond the map, which no sampler writes.  Here those bytes hold sentinels: one value beyond the map's
columns and another beyond its rows, different for the linear and the angular maps and from every sampled code, so a
wrap or clamp by the wrong dimension, or a read with the wrong pitch, changes the cost."""
import numpy as np

from oracle import mppi_ref as MR
from oracle import terrain_ref as TR
from oracle import xoroshiro as X
from tests import rollout_edge_cases as EC
from tests import window_first_cases as WF
from tests.scenarios import make_scenario

F32, F64 = np.float32, np.float64

# name: (rows, cols, Rmax, Cmax, res) -- the padded map and the allocation around it.  Where the columns differ the
# two pitches differ, neither equals cols, and cols is no multiple of 16 (37: mask pitch 48, 70: grid pitch 80;
# 261: 272, 290: 304).  "large" is larger than the 232 x 240 window in both axes: the staged window is clamped at the
# map's edge, inside the allocation.
GEOMETRIES = {
    "rows": (30, 37, 52, 37, 0.1),
    "cols": (30, 37, 30, 70, 0.1),
    "both": (30, 37, 52, 70, 0.1),
    "large": (300, 261, 333, 290, 0.05),
}
SMALL = ("rows", "cols", "both")
MASKS03 = "both"                     # the geometry whose masks hold 0..3 (the windowed kernel's general variant)

# (beyond the map's columns, beyond its rows) of each map; sampled codes are 0..100, the escape code is -128
SENTINELS = dict(lin=(111, 123), ang=(117, 126))

SPOTS = EC.MAP_SPOTS
# out of the map across the nearest edge: x < 0 from low-left and y < 0 from low-right (wrapped by the allocation
# to beyond the map), y past the top from high-left and x past the right edge from high-right (clamped into the
# allocation's last row / column)
HEADING = {"centre": 0.7, "low-left": np.pi, "low-right": -np.pi / 2, "high-left": np.pi / 2, "high-right": 0.0,
           "padding": -2.4}
# the side each corner leaves through, and the allocation axis its reads beyond the map need
SIDE = {"low-left": ("x", "low"), "low-right": ("y", "low"), "high-left": ("y", "high"), "high-right": ("x", "high")}


def pitch(n):
    return (n + 15) // 16 * 16


def beyond(shape, rows, cols):
    """(beyond the columns, beyond the rows): boolean masks of a (..., Rmax, Cmax) array's cells outside the map."""
    R, C = shape[-2:]
    r, c = np.arange(R)[:, None], np.arange(C)[None, :]
    return (np.broadcast_to((r < rows) & (c >= cols), shape), np.broadcast_to(r >= rows, shape))


def fill_beyond(grids, rows, cols, which):
    """Write map `which`'s sentinels into every allocation cell of `grids` (..., Rmax, Cmax) beyond the map."""
    bc, br = beyond(grids.shape, rows, cols)
    grids[bc], grids[br] = SENTINELS[which]
    return grids


def sentinel_grids(shape, rows, cols, inside=-77):
    """dict(lin, ang) of whole allocations: `inside` on the map, the sentinels beyond it."""
    return {w: fill_beyond(np.full(shape, inside, np.int8), rows, cols, w) for w in ("lin", "ang")}


def raw_case(geom, spot, mode, N=128, M=8, T=100, seed=0, masks03=None):
    """Inputs of one C-ABI rollout on geometry `geom`: random sampled codes on the map (0 in the padding ring, so the
    traction floor lb[0] = 0.2 carries rollouts across it), sentinels beyond it, random masks (0..3 on the MASKS03
    geometry) and risk, the robot at `spot` heading out of the map, forward controls fast enough to leave it."""
    rows, cols, Rmax, Cmax, res = GEOMETRIES[geom]
    masks03 = (geom == MASKS03) if masks03 is None else masks03
    pad = EC.pad_cells(res)
    rng = np.random.default_rng(1000 * seed + 10 * SPOTS.index(spot) + mode + len(geom))
    Mk = M if mode == 0 else 1
    maps = {}
    for w in ("lin", "ang"):
        g = fill_beyond(np.zeros((Mk, Rmax, Cmax), np.int8), rows, cols, w)
        g[:, pad:rows - pad, pad:cols - pad] = rng.integers(0, 101, (Mk, rows - 2 * pad, cols - 2 * pad))
        maps[w] = g
    hit = rng.random((2, rows, cols)) < 0.05
    vals = rng.integers(1, 4, (2, rows, cols)) if masks03 else 1
    obs, unk = (hit * vals).astype(np.int8)
    x, y = EC.map_spot(spot, rows - 2 * pad, cols - 2 * pad, res, pad)
    th = HEADING[spot]
    T_ = np.arange(T)
    u_cur = np.stack([1.5 + 0.5 * np.cos(0.3 * T_), 0.2 * np.sin(0.2 * T_)], 1).astype(F32)
    return dict(mode=mode, N=N, M=Mk, T=T, R=rows, C=cols, Rmax=Rmax, Cmax=Cmax, res=F32(res), xlo=F32(-pad * res),
                ylo=F32(-pad * res), lb=[0.2, 1.3], ab=[0.15, 0.9], obs=obs, unk=unk,
                risk=rng.integers(0, 101, (rows, cols)).astype(np.int8), lin=maps["lin"], ang=maps["ang"],
                noise=(rng.standard_normal((N, T, 2)) * [1.0, 0.4]).astype(F32), u_cur=u_cur,
                u_prev=(u_cur + F32(0.1)).astype(F32), x0=[x, y, th],
                goal=[x + 40.0 * np.cos(th), y + 40.0 * np.sin(th)], tol=0.5, dt=F32(0.1), vrange=[0.0, 3.0],
                alpha=0.5, masks03=masks03)


def limits(s):
    """Padded map limits (pxl, pyl) of a raw case, float32 as the planner holds them."""
    return (np.array([s["xlo"], F64(s["xlo"]) + s["C"] * F64(s["res"])], F32),
            np.array([s["ylo"], F64(s["ylo"]) + s["R"] * F64(s["res"])], F32))


def oracle(s, arith, grids=None, return_states=False, ctrl_order=None):
    """MR.rollout_costs of a raw case: the whole allocations as the sampled maps (or `grids`), the map-shaped masks and
    risk, wrap + clamp, the windowed kernel's control-cost order in mode 0 (pre-summed), the generic one's otherwise."""
    lin, ang = (s["lin"], s["ang"]) if grids is None else grids
    pxl, pyl = limits(s)
    return MR.rollout_costs(s["mode"], lin, ang, s["lb"], s["ab"], s["obs"], s["unk"], s["res"], pxl, pyl, s["vrange"],
                            [-np.pi, np.pi], s["goal"], 0.01, 1e5, 1e2, s["tol"], 1.0, [2, 3], s["x0"], s["dt"], 1.0,
                            s["noise"], s["u_cur"], risk_map=s["risk"][None], return_states=return_states, arith=arith,
                            ctrl_order=ctrl_order or ("presummed" if s["mode"] == 0 else "sequential"), wrap_clamp=True)


def state_oracle(s, V, arith):
    """MR.state_rollouts of a raw case (get_state_rollout): V sequences over the whole allocations."""
    pxl, pyl = limits(s)
    return MR.state_rollouts(s["mode"], V, s["lin"], s["ang"], s["lb"], s["ab"], s["res"], pxl, pyl, s["x0"], s["dt"],
                             s["u_cur"], s["u_prev"], s["noise"], s["vrange"], [-np.pi, np.pi], arith=arith,
                             wrap_clamp=True)


def beyond_reads(states, s, arith):
    """Which allocation cells beyond the map the oracle's trajectories read, per way of getting there: dict of
    booleans wrap_x (x < 0 wrapped past cols), wrap_y, clamp_x (x >= cols clamped into a column >= cols), clamp_y.
    States (N, M, T + 1, 3); every step's read counts (the goal is out of reach)."""
    xs, ys = states[..., :-1, 0], states[..., :-1, 1]
    xi = MR.floor_div_f32(arith.sub32(xs, F32(s["xlo"])), F32(s["res"]), arith)
    yi = MR.floor_div_f32(arith.sub32(ys, F32(s["ylo"])), F32(s["res"]), arith)
    gx, gy = MR._wrap_clamp(xi, s["Cmax"]), MR._wrap_clamp(yi, s["Rmax"])
    return dict(wrap_x=bool(((xi < 0) & (gx >= s["C"])).any()), wrap_y=bool(((yi < 0) & (gy >= s["R"])).any()),
                clamp_x=bool(((xi >= s["C"]) & (gx >= s["C"])).any()), clamp_y=bool(((yi >= s["R"]) & (gy >= s["R"])).any()))


# ----------------------------------------------------------------------------- window-first solves
# The large map (padded 400 x 197: the window spans every column, so x never escapes) and the smaller one set in the
# same allocation afterwards (padded 310 x 123: still taller than the window, so solves take window-first sampling).
WF_RES = 0.1
WF_MAP = (390, 187)
WF_SMALL = (300, 113)
WF_ALLOC = (450, 290)
# name: (map, robot (x, y) in map cells, heading, forward control, (flagged, reads beyond the map)).  Steps of up to
# 1.2 m (dt 0.4 s) jump the 0.5 m of traction-0 padding.  "old-samples": +x from the small map's right edge, clamped
# into the columns where the large map was sampled.
WF_CASES = {
    "inside": (WF_MAP, (93.5, 195.5), 0.7, 0.05, (False, False)),
    "escape": (WF_MAP, (93.5, 195.5), np.pi / 2, 3.0, (True, None)),
    "wrap": (WF_MAP, (1.5, 195.5), np.pi, 3.0, (False, True)),
    "old-samples": (WF_SMALL, (111.5, 150.5), 0.0, 3.0, (False, True)),
}


def wf_scenario(rows, cols, T=100):
    """The window-first scenario on the rows x cols corner of one 390 x 390 draw, in the WF_ALLOC allocation."""
    sc = WF.moving(WF.crop(make_scenario("tdm", N=64, M=4, T=T, H=WF_MAP[0], W=WF_MAP[0], res=WF_RES, B=5, seed=43,
                                         bin_values=WF.MOVING), rows, cols, WF_RES))
    sc["cfg"] = dict(sc["cfg"], max_map_dim=WF_ALLOC)
    sc["params"] = dict(sc["params"], dt=0.4, u_std=np.array([0.2, 0.001]))
    return sc


def wf_start(case):
    """(x0, u_cur) of window-first case `case`."""
    _, (cx, cy), th, u, _ = WF_CASES[case]
    T = 100
    return np.array([cx * WF_RES, cy * WF_RES, th]), np.stack([np.full(T, u), np.zeros(T)], 1).astype(F32)


def beyond_cells(cells, rows, cols, shape):
    """(M, Rmax, Cmax) mask of the allocation cells beyond the rows x cols map that executed reads land on (cells:
    WF.executed_cells, (live (N, M), yi, xi) per step)."""
    out = np.zeros(shape, bool)
    m = np.broadcast_to(np.arange(shape[0])[None, :], cells[0][0].shape) if cells else None
    for live, yi, xi in cells:
        gy, gx = MR._wrap_clamp(yi, shape[1]), MR._wrap_clamp(xi, shape[2])
        hit = live & ((gy >= rows) | (gx >= cols))
        out[m[hit], gy[hit], gx[hit]] = True
    return out


def wf_outcome(case, arith, base=None, seed=0):
    """Case `case` on the host: both maps sampled whole over `base` (default zeros) from the TDM's initial generator
    states (lin's stream for both: the fused pair), the exact oracle's rollouts with random noise.  Returns (flags (M,),
    beyond_cells mask, grids, costs)."""
    sc = wf_scenario(*WF_CASES[case][0])
    pad = EC.pad_cells(WF_RES)
    M = sc["M"]
    grids = host_maps(sc, np.zeros((M,) + WF_ALLOC, np.int8) if base is None else base)
    rows, cols = sc["obstacle"].shape[0] + 2 * pad, sc["obstacle"].shape[1] + 2 * pad
    x0, u_cur = wf_start(case)
    p = sc["params"]
    noise = (np.random.default_rng(seed).standard_normal((sc["N"], 100, 2)) * p["u_std"]).astype(F32)
    xlo = F32(-pad * WF_RES)
    lim = np.array([xlo, F32(F64(xlo) + cols * WF_RES)], F32), np.array([xlo, F32(F64(xlo) + rows * WF_RES)], F32)
    costs, states = MR.rollout_costs(MR.MODE_STOCHASTIC, grids[0], grids[1], [0, 1], [0, 1], np.pad(sc["obstacle"], pad),
                                     np.pad(sc["unknown"], pad), F32(WF_RES), lim[0], lim[1], p["vrange"], p["wrange"],
                                     p["xgoal"], p["v_post_rollout"], 1e5, 1e2, p["goal_tolerance"], p["lambda_weight"],
                                     p["u_std"], x0, p["dt"], 1.0, noise, u_cur, return_states=True, arith=arith,
                                     ctrl_order="presummed", wrap_clamp=True)
    wx0, wy0, ww, wh = EC.window_origin(x0[0], x0[1], xlo, xlo, WF_RES, cols, rows, EC.window_height(100))
    rect = WF.window_rect(wx0, wy0, ww, wh, rows, cols)
    flags, _ = WF.escapes(states, xlo, xlo, WF_RES, p["xgoal"], p["goal_tolerance"], rect, rows, cols, *WF_ALLOC, arith)
    cells = WF.executed_cells(states, xlo, xlo, WF_RES, p["xgoal"], p["goal_tolerance"], arith)
    return flags, beyond_cells(cells, rows, cols, grids[0].shape), grids, costs


def host_maps(sc, base):
    """(lin, ang): scenario sc's maps sampled whole over copies of `base`, as a fused TDM pair's first sampling."""
    pad = EC.pad_cells(sc["tdm_dict"]["res"])
    M, tile = sc["M"], tuple(sc["cfg"]["tdm_sample_thread_dim"])
    states = X.create_states(tile[0] * tile[1] * M, sc["cfg"]["seed"])
    out = []
    for key in ("pmf_lin", "pmf_ang"):
        pmf = np.pad(sc[key], ((0, 0), (pad, pad), (pad, pad)))
        pmf[0, :pad], pmf[0, -pad:], pmf[0, :, :pad], pmf[0, :, -pad:] = 100, 100, 100, 100
        g = base.copy()
        TR.sample_grids(g, pmf, states.copy(), np.asarray(sc["tdm_dict"]["bin_values"], F32),
                        np.asarray(sc["tdm_dict"]["bin_values_bounds"], F32), 1.0, tile, M)
        out.append(g)
    return out
