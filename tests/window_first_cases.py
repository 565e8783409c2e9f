"""Window-first sampling (TEST INFRASTRUCTURE): the sampled rectangle and the escape rule of csrc/rollout_win.cu
restated once, for the CPU test of the kernels' source (tests/test_window_first_emulated_cpu.py) and the GPU test of
solve() (tests/test_gpu_window_first_edges.py).

The rectangle (stage_sample_window, api.cu): the staged window (win_origin; tests/rollout_edge_cases.window_origin)
plus a ring of WIN_SAMPLE_RING cells on every side, clipped to the map.  The escape rule (lookup_slow): a lane reads the
sampled maps at cell (wrap_clamp(yi, grid_rows), wrap_clamp(xi, grid_cols)); the read is an escape when that cell lies
inside the map (rows x cols) but outside the rectangle.  A map is flagged when some live lane escapes at a step it
executes: steps 0 .. T - 1, up to and including the step that reaches the goal.  The completion (the sampler's
window_complete kernel) re-walks the maps of every map group (gm maps per CTA) that holds a flagged map."""
import numpy as np

from oracle import mppi_ref as MR
from tests import rollout_edge_cases as EC

F32 = np.float32
WIN_SAMPLE_RING = 8
MOVING = np.array([0.0, 0.6, 0.7, 0.85, 1.0])    # bin values of the escape scenarios (bin 0 emptied by moving())


def moving(sc):
    """No traction-0 cell: bin 0's mass moved to bin 1, so no rollout stops before it can leave the window."""
    for key in ("pmf_lin", "pmf_ang"):
        sc[key][1] += sc[key][0]
        sc[key][0] = 0
    return sc


def crop(sc, rows, cols, res):
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


def window_rect(wx0, wy0, ww, wh, rows, cols, ring=WIN_SAMPLE_RING):
    """(row_lo, row_hi, col_lo, col_hi) of the sampled rectangle, as sample_window() reports it in [1:5]."""
    return (max(wy0 - ring, 0), min(wy0 + wh + ring, rows), max(wx0 - ring, 0), min(wx0 + ww + ring, cols))


def executed_cells(states, xlo, ylo, res, xgoal, tol, arith, n_live=None):
    """The cells the lanes read, from the oracle's trajectories ``states`` (N, M, T + 1, 3) (MR.rollout_costs with
    return_states=True, wrap_clamp=True, the same ``arith``): per step t, (live (N, M) bool -- the lane executes step
    t: live, and the goal not reached before it --, yi, xi) with the raw cell indices before wrap and clamp."""
    N, M, T1, _ = states.shape
    n_live = N if n_live is None else n_live
    xg, yg = F32(xgoal[0]), F32(xgoal[1])
    tol2 = F32(F32(tol) * F32(tol))
    active = np.zeros((N, M), bool)
    active[:n_live] = True
    out = []
    for t in range(T1 - 1):
        if not active.any():
            break
        x, y = states[:, :, t, 0], states[:, :, t, 1]
        xi = MR.floor_div_f32(arith.sub32(x, F32(xlo)), F32(res), arith)
        yi = MR.floor_div_f32(arith.sub32(y, F32(ylo)), F32(res), arith)
        out.append((active.copy(), yi, xi))
        xn, yn = states[:, :, t + 1, 0], states[:, :, t + 1, 1]
        dx, dy = arith.sub32(xg, xn), arith.sub32(yg, yn)
        d2 = arith.fma32(dx, dx, arith.mul32(dy, dy))
        active &= ~(d2 <= tol2)                        # the goal step's read counts; none after it
    return out


def escapes(states, xlo, ylo, res, xgoal, tol, rect, rows, cols, grid_rows, grid_cols, arith, n_live=None):
    """Escaping reads predicted from the oracle's trajectories (see executed_cells).  Returns (flags (M,) bool,
    reads): reads is a list of (n, m, t, yi, xi, gy, gx), the first escaping read of every (n, m) that escapes, with
    the raw and the wrapped + clamped cell."""
    r0, r1, c0, c1 = rect
    seen = np.zeros(states.shape[:2], bool)
    reads = []
    for t, (active, yi, xi) in enumerate(executed_cells(states, xlo, ylo, res, xgoal, tol, arith, n_live)):
        gy, gx = MR._wrap_clamp(yi, grid_rows), MR._wrap_clamp(xi, grid_cols)
        esc = active & (gy < rows) & (gx < cols) & ((gy < r0) | (gy >= r1) | (gx < c0) | (gx >= c1))
        for n, m in np.argwhere(esc & ~seen):
            reads.append((int(n), int(m), t, int(yi[n, m]), int(xi[n, m]), int(gy[n, m]), int(gx[n, m])))
        seen |= esc
    return seen.any(axis=0), reads


def window_sampled(rect, cols, ty):
    """(row_lo, row_hi, col_lo, col_hi) of the cells the window-first sampling writes: the rectangle's rows, and the
    whole tile columns (ceil(cols / ty) cells wide) that hold its columns."""
    r0, r1, c0, c1 = rect
    ncol = -(-cols // ty)
    return r0, r1, c0 // ncol * ncol, min(((c1 - 1) // ncol + 1) * ncol, cols)


def completed_maps(flags, gm):
    """Maps the completion re-walks: every map of a group of gm consecutive maps that holds a flagged map."""
    flags = np.asarray(flags, bool)
    out = np.zeros(len(flags), bool)
    for g0 in range(0, len(flags), gm):
        out[g0:g0 + gm] = flags[g0:g0 + gm].any()
    return out


def outside_rect(shape, rect):
    """Boolean mask of the cells of a (..., R, C) map array outside the rectangle."""
    r0, r1, c0, c1 = rect
    R, C = shape[-2:]
    inside = np.zeros((R, C), bool)
    inside[r0:r1, c0:c1] = True
    return np.broadcast_to(~inside, shape)
