"""The tables of tests/rollout_edge_cases.py (run on the GPU by tests/test_gpu_rollout_edges.py) still reach every
work-share regime, window height and map geometry they are there for: an edit that drops one fails here."""
import numpy as np
import pytest

from tests import rollout_edge_cases as EC

SMS = EC.H100_SXM_SMS


@pytest.mark.parametrize("N,M,T,grid,unit,what", EC.REGIME_CASES)
def test_regime_rows_at_132_sms(N, M, T, grid, unit, what):
    r = EC.share_regime(N, M, SMS)
    assert (r["grid"], r["unit"]) == (grid, unit), what
    bounds = EC.share_bounds(N, M, SMS)                  # the shares tile the work list, in order
    assert bounds[0][0] == 0 and bounds[-1][1] == r["chunks"]
    assert all(a[1] == b[0] for a, b in zip(bounds, bounds[1:]) if unit != 0)
    assert sorted(bounds) == bounds and sum(hi - lo for lo, hi in bounds) == r["chunks"]


def test_regime_table_covers_every_regime():
    rows = [(N, M, T, EC.share_regime(N, M, SMS)) for N, M, T, *_ in EC.REGIME_CASES]
    assert any(r["grid"] == 1 and M > 1 for N, M, T, r in rows)                          # one CTA walks every map
    assert any(r["grid"] == 1 and N == 1 and M == 1 for N, M, T, r in rows)              # one live lane
    # unit 0 with a remainder: some maps get one CTA more than the others
    assert any(r["unit"] == 0 and r["grid"] % M != 0 and r["grid"] > M for N, M, T, r in rows)
    # unit 1 at a ragged N: shares that cross maps, a partly empty last warp per map
    assert any(r["unit"] == 1 and N % 32 != 0 and r["grid"] < M for N, M, T, r in rows)
    assert any(r["unit"] == 32 and r["passes"] != int(r["passes"]) for N, M, T, r in rows)    # fractional passes
    assert {1, 2} <= {T for N, M, T, r in rows}
    assert max(T for N, M, T, r in rows) == 1024
    single = {EC.window_height(T) for N, M, T, r in rows}
    assert single == {224, 232}
    assert EC.window_height(702) == 232 and EC.window_height(703) == 224


def test_batch_cases_cover_both_heights_and_a_mid_share_switch():
    """The batched launch keeps a planner record of sizeof(RolloutWinArgs) bytes (between 1 and 4096) behind the
    window: T 702 fits the single launch's 232 rows exactly, so the batch runs 224 there; T 20 runs 232."""
    heights = set()
    for N, M, T in EC.BATCH_CASES:
        lo, hi = EC.window_height(T, 1), EC.window_height(T, 4096)
        assert lo == hi
        heights.add(lo)
        assert EC.mid_share_switches(N, M, SMS, len(EC.BATCH_MAPS)), (N, M, T)
    assert heights == {224, 232}
    assert any(EC.window_height(T, 1) != EC.window_height(T) for N, M, T in EC.BATCH_CASES)
    assert len({res for n, res in EC.BATCH_MAPS}) == len(EC.BATCH_MAPS) >= 3


def _windows(rows, cols, res):
    """(R, C) of the padded grid and the window (wx0, wy0, ww, wh) at every spot."""
    pad = EC.pad_cells(res)
    R, C = EC.padded_grid(rows, cols, res)
    lo = -pad * res
    return (R, C), {s: EC.window_origin(*EC.map_spot(s, rows, cols, res, pad), lo, lo, res, C, R) for s in EC.MAP_SPOTS}


def test_map_cases_reach_every_window_edge():
    """On the padded grid the window is laid over: one smaller than the window, one equal to it (the window is the
    whole grid, nothing on the global path), one a row and a column larger (the last row and column on the global
    path at the high spots), one larger with the 16-aligned origin short of the right edge."""
    grids = {EC.padded_grid(r, c, res): _windows(r, c, res)[1] for r, c, res in EC.MAP_CASES}
    assert any(R < 232 and C < 240 for R, C in grids)
    assert all(w == (0, 0, 240, 232) for w in grids[(232, 240)].values())
    hi = grids[(233, 241)]
    assert hi["high-right"] == (0, 1, 240, 232) and hi["low-left"] == (0, 0, 240, 232)     # column 240 outside
    assert any(C > 241 and (C - 240) % 16 for R, C in grids)
    for rows, cols, res in EC.MAP_CASES:
        (R, C), spots = _windows(rows, cols, res)
        assert spots["padding"][:2] == (0, 0) and spots["low-left"][:2] == (0, 0)
        for s in ("low-right", "high-right"):                  # origin clamped to the right edge, then 16-aligned
            wx0, _, ww, _ = spots[s]
            assert wx0 == max(C - EC.WIN_WW, 0) & ~15 and wx0 + ww <= C
            assert (wx0 + ww < C) == (C > EC.WIN_WW and (C - EC.WIN_WW) % 16 != 0)   # columns on the global path
        for s in ("high-left", "high-right"):
            assert spots[s][1] + spots[s][3] == R


def test_oracle_checks_every_map_of_the_small_launches():
    for N, M, T, *_ in EC.REGIME_CASES:
        maps = EC.oracle_maps(N, M, T, SMS)
        assert len(maps) == M or N * M * T > EC.ORACLE_BUDGET
    assert len(EC.oracle_maps(33, 100, 24, SMS)) == 100 and len(EC.oracle_maps(1000, 133, 16, SMS)) == 133


@pytest.mark.parametrize("kind", EC.CORNER_KINDS)
def test_corner_cases(kind):
    s = EC.corner_case(0.7, kind, 0)
    x0, y0 = s["x0"][:2]
    assert abs(np.float64(x0) - s["edge"][0]) <= s["ulp"][0] / 2
    assert abs(np.float64(y0) - s["edge"][1]) <= s["ulp"][1] / 2
    i = s["i"]
    assert (abs(i) < 2 ** 21) == (kind != "+2^21" and kind != "-2^21")      # beyond 2^21: the exact sequence
    if kind != "small":
        assert abs(i) > 2 ** 20 - 8
    gx = sorted({EC._wrap_clamp(i - 1, s["C"]), EC._wrap_clamp(i, s["C"])})
    gy = [s["j"] - 1, s["j"]]
    for name in ("lin", "ang"):
        quad = s[name][:, gy][:, :, gx].reshape(s["M"], 4)
        assert all(len(set(q)) == 4 for q in quad)
    for name in ("obs", "unk", "risk"):
        assert len(set(s[name][gy][:, gx].ravel())) > 1
    e = max(abs(v) for v in s["vrange"])
    assert e * 0.1 * 1.3 <= 2.01 * max(s["ulp"])
    u = s["u_cur"]                      # a control cost that is not 0, forward commands well inside +-e
    assert (u[:, 0] != 0).all() and (np.abs(u[:, 0]) <= e / 4).all() and (u[:, 1] != 0).any()
