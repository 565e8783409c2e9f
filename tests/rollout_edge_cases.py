"""Edge cases of the windowed stochastic rollout (TEST INFRASTRUCTURE): the launch rules of csrc/rollout_win.cu
restated as functions of N, M, T and the SM count, the tables of shapes that reach each work-share regime, window
height and map geometry, and the directed cell-corner inputs.

Work share (launch_rollout_win, launch_rollout_win_batch; kernel: rollout_win_body): the work list is the unit-major
sequence of 32-rollout chunks, units = maps (single launch) or (planner, map) pairs (batched launch), npad = N rounded
up to 32.  The persistent grid is min(max(chunks / 8, 1), SMs) CTAs; the share unit is 32 chunks when a CTA's share is
at least 4 passes of 32 chunks, else 0 when there is at least one CTA per unit (shares never cross a unit: unit m gets
q or q + 1 CTAs), else 1 (chunk-granular shares that may cross units).  Window height: 232 rows while the shared-memory
layout (4 byte planes of 240 x WH, the traction tables, 2T controls, the barrier) fits 232 448 bytes, else 224; the
batched launch also keeps one planner record (sizeof(RolloutWinArgs)) there."""
import numpy as np

F32, F64 = np.float32, np.float64

WIN_WW = 240
WIN_MAX_SMEM = 232448
H100_SXM_SMS = 132


def win_smem_total(WH, T):
    """win_smem_layout(240, WH, T).total."""
    planes = (4 * WIN_WW * WH + 127) & ~127
    off_bar = (planes + 2 * 256 * 8 + 2 * T * 4 + 15) & ~15
    return off_bar + 16


def window_height(T, record_bytes=0):
    """Rows of the staged window: the single launch (record_bytes 0) or the batched one (record_bytes =
    sizeof(RolloutWinArgs) > 0)."""
    return 232 if win_smem_total(232, T) + record_bytes <= WIN_MAX_SMEM else 224


def share_regime(N, M, sms, count=1):
    """The launch's persistent grid and share unit for `count` planners (count 1: the single launch) of N control
    sequences and M maps: dict(npad, cpm (chunks per unit), units, chunks, grid, unit, passes (chunks per CTA / 32))."""
    npad = (N + 31) // 32 * 32
    cpm = npad // 32
    units = count * M
    chunks = units * cpm
    grid = min(max(chunks // 8, 1), sms)
    unit = 32 if chunks // (32 * grid) >= 4 else (0 if grid >= units else 1)
    return dict(npad=npad, cpm=cpm, units=units, chunks=chunks, grid=grid, unit=unit, passes=chunks / (32.0 * grid))


def share_bounds(N, M, sms, count=1):
    """[(w_lo, w_hi)] chunk range of every CTA (rotate 0), as rollout_win_body computes it."""
    r = share_regime(N, M, sms, count)
    G, cpm, units, total, unit = r["grid"], r["cpm"], r["units"], r["chunks"], r["unit"]
    out = []
    for b in range(G):
        if unit == 0:
            q = G // units
            rem = G - q * units
            if b < rem * (q + 1):
                m, j, k = b // (q + 1), b % (q + 1), q + 1
            else:
                b2 = b - rem * (q + 1)
                m, j, k = rem + b2 // q, b2 % q, q
            out.append((m * cpm + cpm * j // k, m * cpm + cpm * (j + 1) // k))
        else:
            n_units = (total + unit - 1) // unit
            out.append((min(total, n_units * b // G * unit), min(total, n_units * (b + 1) // G * unit)))
    return out


def share_edge_maps(N, M, sms, limit=16):
    """Maps to check against the oracle when M is large: the first, the last and those where CTA shares begin and
    end (at most `limit`, spread over the launch)."""
    r = share_regime(N, M, sms)
    edges = set()
    for lo, hi in share_bounds(N, M, sms):
        if hi > lo:
            edges.update((lo // r["cpm"], (hi - 1) // r["cpm"]))
    edges = sorted(edges - {0, M - 1})
    if len(edges) > limit - 2:
        edges = [edges[i] for i in np.linspace(0, len(edges) - 1, limit - 2).round().astype(int)]
    return np.array(sorted({0, M - 1, *edges}))


ORACLE_BUDGET = 8192 * 8 * 128         # lane-steps of the config-5 subset check (tests/test_gpu_exact_oracle.py)


def oracle_maps(N, M, T, sms):
    """Maps the oracle checks: every map while the N * M * T lane-steps fit ORACLE_BUDGET, else share_edge_maps."""
    return np.arange(M) if N * M * T <= ORACLE_BUDGET else share_edge_maps(N, M, sms)


def mid_share_switches(N, M, sms, count):
    """CTAs of a batched launch whose share holds units of more than one planner."""
    r = share_regime(N, M, sms, count)
    per = M * r["cpm"]
    return [b for b, (lo, hi) in enumerate(share_bounds(N, M, sms, count)) if hi > lo and lo // per != (hi - 1) // per]


# ----------------------------------------------------------------------------- the tables
# (N, M, T, grid, unit, what it exercises) with grid and unit on a 132-SM H100 SXM
REGIME_CASES = [
    (1, 1, 24, 1, 0, "one live lane"),
    (1, 8, 24, 1, 1, "one CTA walks all 8 maps"),
    (33, 100, 24, 25, 1, "shares cross maps; the last warp has 1 live lane"),
    (33, 100, 1, 25, 1, "one step"),
    (33, 100, 2, 25, 1, "two steps"),
    (200, 24, 24, 21, 1, "tdm_scenario's shape"),
    (1000, 131, 16, 132, 0, "one map gets 2 CTAs"),
    (1000, 133, 16, 132, 1, "unit 1 over more maps than CTAs"),
    (1000, 600, 16, 132, 32, "4.5 passes per CTA"),
    (64, 4, 703, 1, 1, "T 703: the single launch's 224-row window"),
    (64, 4, 1024, 1, 1, "T 1024: the configured maximum"),
]

# map sizes (rows, cols, res) of the map-geometry cases.  The window is laid over the PADDED grid (pad_cells(res) cells
# on every side), which is 11 x 11 and 8 x 14 (smaller than the window), 232 x 240 (equal to it: the window is the whole
# grid), 233 x 241 (one row and one column more) and 250 x 250 (larger, 250 - 240 not a multiple of 16)
MAP_CASES = [(9, 9, 1.0), (6, 12, 1.0), (222, 230, 0.1), (223, 231, 0.1), (240, 240, 0.1)]
MAP_SPOTS = ["centre", "low-left", "low-right", "high-left", "high-right", "padding"]

# batched launches: (N, M, T) of 3 planners on three different maps; M 20 rather than 24 at T 20 so that a CTA's share
# holds the end of one planner and the start of the next (at M 24 every planner ends on a share boundary)
BATCH_MAPS = [(9, 1.0), (64, 0.2), (300, 0.05)]
BATCH_CASES = [(200, 20, 20), (200, 4, 702)]

NOISE_N = [1, 33, 200, 1000]
NOISE_T = [1, 3, 100, 129]

CORNER_RES = [0.1, 0.05, 0.3, 1.0, 0.0625, 0.7]
CORNER_KINDS = ["small", "+2^20", "-2^20", "+2^21", "-2^21"]


def pad_cells(res):
    """Cells of padding on every side of a tests/scenarios.make_scenario map (pad_speed 5 m/s, dt 0.1 s)."""
    return int(np.ceil(5.0 * 0.1 / res))


def padded_grid(rows, cols, res):
    """(R, C): the planner's grid of a rows x cols map, padding included."""
    return rows + 2 * pad_cells(res), cols + 2 * pad_cells(res)


def window_origin(x, y, pxl, pyl, res, cols, rows, WH=232):
    """win_origin (kernels.h): (wx0, wy0, ww, wh) of the window centred on the robot's cell, clamped into the map,
    wx0 rounded down to a multiple of 16; columns from wx0 + ww on are read from global memory."""
    xi0 = int(np.floor((F64(F32(x)) - F64(F32(pxl))) / F64(F32(res))))
    yi0 = int(np.floor((F64(F32(y)) - F64(F32(pyl))) / F64(F32(res))))
    cx = max(min(xi0 - WIN_WW // 2, cols - WIN_WW), 0)
    cy = max(min(yi0 - WH // 2, rows - WH), 0)
    wx0 = cx & ~15
    return wx0, cy, min(WIN_WW, cols - wx0), min(WH, rows - cy)


def map_spot(spot, rows, cols, res, pad):
    """Robot position (x, y) in map coordinates (the unpadded map spans [0, cols*res] x [0, rows*res])."""
    w, h = cols * res, rows * res
    return dict(centre=(w / 2 + 0.13 * res, h / 2 - 0.21 * res),
                **{"low-left": (1.3 * res, 2.6 * res), "low-right": (w - 2.4 * res, 1.7 * res),
                   "high-left": (2.2 * res, h - 1.4 * res), "high-right": (w - 1.6 * res, h - 2.3 * res),
                   "padding": (-0.5 * min(pad, 1) * res, -0.4 * min(pad, 1) * res)})[spot]


# ----------------------------------------------------------------------------- directed cell corners
def _wrap_clamp(i, n):
    return min(max(i + n if i < 0 else i, 0), n - 1)


def corner_case(res, kind, mode, N=64, T=12, seed=0):
    """Inputs whose rollouts random-walk across both edges of a four-cell corner, about one float32 ulp per step.

    The corner is (i, j) in cells from (xlo, ylo); x0 is the float32 nearest to it.  vrange is +-e with e such that a
    step moves the state by at most ~2 ulps of its coordinate (traction 0.64 to 1.3 around the corner), so the noise
    (clipped to +-e) makes every rollout wander around the corner.  u_cur is small but not 0 (+-e/4 forward, up to
    1 rad/s of turn): the control cost is then not 0, and its summation order (pre-summed in the windowed kernel,
    sequential in the generic one) shows in the costs.  The four cells around it differ in
    obstacle, unknown, both traction bytes and risk; everything else is uniform, so a wrong cell changes the cost.
    kind "small": i = j = 8 on a 16 x 64 map;
    "+-2^20", "+-2^21": x index near (or just beyond) +-2^20 or 2^21 on a map of 2^20 + 64 or 2^21 + 64 columns, so a
    negative index wraps back into the map, y index 8 with ylo placed so that y has x's magnitude (and ulp)."""
    rng = np.random.default_rng(seed)
    res = F32(res)
    R = 16
    if kind == "small":
        C, i, xlo = 64, 8, F32(-3.0)
    else:
        big = 1 << (20 if "20" in kind else 21)
        C = big + 64
        i = {"+2^20": big - 3, "-2^20": -(big - 5), "+2^21": big + 16, "-2^21": -(big + 16)}[kind]
        xlo = F32(0.0)
    j = 8
    x0 = F32(F64(xlo) + i * F64(res))
    ylo = F32(-3.0) if kind == "small" else F32(F64(x0) - j * F64(res))
    y0 = F32(F64(ylo) + j * F64(res))
    ulp = F64(max(np.spacing(abs(x0)), np.spacing(abs(y0))))
    dt = F32(0.1)
    lb, ab = [0.2, 1.3], [0.0, 1.0]
    e = F32(2.0 * ulp / (F64(dt) * 1.3))
    M = 2 if mode == 0 else 1
    lin = np.full((M, R, C), 50, np.int8)
    ang = np.full((M, R, C), 50, np.int8)
    obs = np.zeros((R, C), np.int8)
    unk = np.zeros((R, C), np.int8)
    risk = np.full((R, C), 50, np.int8)
    gx = [_wrap_clamp(i - 1, C), _wrap_clamp(i, C)]
    gy = [_wrap_clamp(j - 1, R), _wrap_clamp(j, R)]
    assert gx[0] != gx[1] and gy[0] != gy[1]
    quad = [(gy[a], gx[b]) for a in (0, 1) for b in (0, 1)]
    for k, (r_, c_) in enumerate(quad):
        lin[0, r_, c_], ang[0, r_, c_] = (40, 95, 60, 75)[k], (90, 10, 60, 25)[k]
        if M > 1:
            lin[1, r_, c_], ang[1, r_, c_] = (85, 45, 100, 55)[k], (0, 100, 45, 55)[k]
        obs[r_, c_] = (1, 0, 0, 0)[k]
        unk[r_, c_] = (0, 0, 1, 0)[k]
        risk[r_, c_] = (15, 95, 55, 30)[k]
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(F32)
    th0 = F32(rng.uniform(-np.pi, np.pi))
    u_cur = np.stack([rng.choice([-0.25, 0.25], T) * e, rng.uniform(-1, 1, T)], 1).astype(F32)
    return dict(mode=mode, N=N, M=M, T=T, R=R, C=C, i=i, j=j, res=res, xlo=xlo, ylo=ylo, x0=[x0, y0, th0],
                edge=(F64(xlo) + i * F64(res), F64(ylo) + j * F64(res)),
                ulp=(F64(np.spacing(abs(x0))), F64(np.spacing(abs(y0)))),
                lb=lb, ab=ab, dt=dt, vrange=[-e, e], goal=[F32(x0 + F32(3.0)), F32(y0 + F32(4.0))], tol=0.5,
                lin=lin, ang=ang, obs=obs, unk=unk, risk=risk, noise=noise, u_cur=u_cur)
