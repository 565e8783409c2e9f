"""The map sampler's launch plan restated (TEST INFRASTRUCTURE) and the tables of cases that reach every variant of it.

Plan (csrc/api.cu plan_sampling, fill_v2, tdm_prepare_jump; csrc/kernels.h sample_v2_fits_hd, sample_v2_smem_hd):
  * bpad = B rounded up to 4; the staged kernel sample_grids_v2_kernel<NT, NW> runs with NW = bpad / 4 for 1, 3 and 8
    words and the runtime-width loop NW = 0 otherwise;
  * a whole-map launch takes gm = 8 maps per CTA, cut to 256 / ty for wide thread tiles; threads = ty * gm rounded up to
    a warp; it fits when 1 <= gm <= 32, threads <= 256, bpad <= 32, its shared memory <= 200 KB and, fused, both TDMs
    have the same bpad;
  * the staged kernel runs when the PMF is well-formed (entries >= 0, running sums <= 127), alpha's bucket table builds
    against the smallest column total, and the launch fits; otherwise the generic kernel sample_grids_kernel runs;
  * row segments: 4096 CTAs' worth, (4096 + tx * groups - 1) // (tx * groups) with groups = ceil(M / 8), or
    B200MPPI_SAMPLE_SEGS; then at most 33, at most nrow, at least 1; seg_rows = ceil(nrow / segs);
  * a lin/ang pair is sampled by one fused launch (NT = 2) when both TDMs hold the same generator states, both tables
    build and the fused launch fits; otherwise each TDM on its own.
A boxed launch (reach box, solve() only) keeps the staged kernel but narrows it to the box (apply_box): tile columns
[col_lo // ncol, (col_hi - 1) // ncol], gm = 128 / nact cut to [1, min(32, M)], the staged column window starting at
the first active tile column rounded down to 16 cells."""
import math

import numpy as np

SG_GM = 8
SG_GM_MAX = 32
SAMPLE_MAX_SEGS = 33
SAMPLE_TABLE_WORDS = 256
SENTINEL = -77                        # bytes the sampler must never write


# ----------------------------------------------------------------------------- the plan
def bpad_of(B):
    return (B + 3) // 4 * 4


def nw_of(bpad):
    """The template width of sample_grids_v2_kernel (launch_v2_nt)."""
    return bpad // 4 if bpad // 4 in (1, 3, 8) else 0


def smem_bytes(tiy_lo, nact, ty, cols, bpad, gm, nt):
    """sample_v2_smem_hd."""
    ncol = -(-cols // ty)
    cfirst = min(tiy_lo * ncol, cols)
    cs1 = min((tiy_lo + nact) * ncol, cols)
    wcols = cs1 - (cfirst & ~15)
    row_bytes_al = (wcols * bpad + 15) & ~15
    stage = max(nt * gm * ((wcols + 15) & ~15), 2 * 128 * 16)
    return nt * row_bytes_al + stage + SAMPLE_TABLE_WORDS * 8 + nt * 128


def fits(tiy_lo, nact, ty, cols, bpad0, bpad1, gm, nt):
    """sample_v2_fits_hd."""
    return (1 <= gm <= SG_GM_MAX and nact >= 1 and tiy_lo >= 0 and tiy_lo + nact <= ty and
            (nact * gm + 31) // 32 * 32 <= 256 and bpad0 <= 32 and
            smem_bytes(tiy_lo, nact, ty, cols, bpad0, gm, nt) <= 200 * 1024 and (nt == 1 or bpad0 == bpad1))


def segments(rows, tile, M, forced=None):
    """(segs, seg_rows) of tdm_prepare_jump; forced: the B200MPPI_SAMPLE_SEGS value."""
    tx = tile[0]
    nrow = -(-rows // tx)
    groups = (M + 7) // 8
    segs = (4096 + tx * groups - 1) // (tx * groups) if forced is None else int(forced)
    segs = max(min(segs, SAMPLE_MAX_SEGS, nrow), 1)
    return segs, -(-nrow // segs)


def plan(B, shape, tile, M, table_ok, forced_segs=None, B1=None, same_stream=False, box=None):
    """The launch one sampling call issues for one TDM (B1 None) or a lin/ang pair (B1: the second TDM's bin count; its
    table is taken to build whenever the first one's does).  box = (row_lo, row_hi, col_lo, col_hi): a boxed launch.
    Returns a dict: kernel ("staged" / "generic"), nt, NW, gm, segs, seg_rows and the geometry the launch meets."""
    rows, cols = shape
    tx, ty = tile
    nrow, ncol = -(-rows // tx), -(-cols // ty)
    bpad = bpad_of(B)
    segs, seg_rows = segments(rows, tile, M, forced_segs)
    gm = SG_GM if ty * SG_GM <= 256 else 256 // ty
    tiy_lo, nact, cs0 = 0, ty, 0
    if box is not None:
        tiy_lo = box[2] // ncol
        nact = (box[3] - 1) // ncol - tiy_lo + 1
        gm = max(min(128 // nact, SG_GM_MAX, M), 1)
        cs0 = min(tiy_lo * ncol, cols)
    nt = 1
    if B1 is not None and same_stream and table_ok and fits(tiy_lo, nact, ty, cols, bpad, bpad_of(B1), gm, 2):
        nt = 2
    staged = table_ok and fits(tiy_lo, nact, ty, cols, bpad, bpad, gm, nt)
    widths = [min((iy + 1) * ncol, cols) - min(iy * ncol, cols) for iy in range(ty)]
    heights = [min((ix + 1) * nrow, rows) - min(ix * nrow, rows) for ix in range(tx)]
    nonempty = [w for w in widths if w > 0]
    return dict(
        kernel="staged" if staged else "generic", nt=nt if staged else 1, NW=nw_of(bpad) if staged else None,
        bpad=bpad, gm=gm, segs=segs, seg_rows=seg_rows, nrow=nrow, ncol=ncol, threads=(nact * gm + 31) // 32 * 32,
        ragged_col=nonempty[-1] < ncol,                      # the last non-empty tile column is narrower
        empty_col=len(nonempty) < ty,                        # tile columns right of the map: no cells
        ragged_row=[h for h in heights if h > 0][-1] < nrow,
        segs_over=segs * seg_rows > nrow,                    # the last segments are short or empty (last_seg)
        partial_group=gm > 0 and M % gm != 0,
        gm_cut=gm < SG_GM and box is None,                   # wide thread tiles: fewer maps per CTA
        chunk_tail=(cols - cs0) % 16 != 0,                   # the window's last 16-byte chunk is partial
        cs0_unaligned=cs0 % 16 != 0,                         # the window starts inside a 16-byte chunk
        boxed=box is not None)


def table_builds(lib_mod, alpha, q_cap):
    """build_sample_thresholds(alpha, q_cap) through b200mppi_debug_sample_threshold (no GPU needed)."""
    r = np.zeros(1, np.uint64)
    out = np.zeros(1, np.uint8)
    return lib_mod.lib.b200mppi_debug_sample_threshold(float(alpha), int(q_cap), lib_mod.ptr(r), 1, lib_mod.ptr(out)) == 0


def pmf_valid(pmf):
    """set_pmf's well-formedness test and the smallest column total (the table's q cap)."""
    acc = np.cumsum(pmf.astype(np.int64), axis=0)
    ok = bool((pmf >= 0).all() and (acc <= 127).all())
    return ok, int(acc[-1].min()) if ok else 0


def case_table_ok(lib_mod, pmf, alpha):
    ok, cap = pmf_valid(pmf)
    return ok and table_builds(lib_mod, alpha, cap)


# ----------------------------------------------------------------------------- PMFs
def sweep_pmf(seed, B, rows, cols, kind="sum100"):
    """(B, rows, cols) int8.  sum100 / sum127: random columns with that total, plus columns with all their mass on the
    first or the last bin (the SIMD count then reaches ge = bpad and ge = bpad - B + 1); ill: running sums that pass
    127 and go below zero."""
    rng = np.random.default_rng(seed)
    if kind == "ill":
        lo, hi = (-128, 128) if B == 1 else (-31, 33) if B < 64 else (-14, 15)
        return rng.integers(lo, hi, (B, rows, cols)).astype(np.int8)
    total = 100 if kind == "sum100" else 127
    if B == 1:
        return np.full((1, rows, cols), total, np.int8)
    cuts = np.sort(rng.integers(0, total + 1, (B - 1, rows, cols)), axis=0)
    pmf = np.diff(np.concatenate([np.zeros((1, rows, cols), np.int64), cuts,
                                  np.full((1, rows, cols), total, np.int64)]), axis=0)
    flat = pmf.reshape(B, -1)
    n = flat.shape[1]
    for i in range(0, n, 5):                           # every fifth cell: all mass on the first bin
        flat[:, i] = 0
        flat[0, i] = total
    for i in range(2, n, 7):                           # every seventh from the third: all mass on the last bin
        flat[:, i] = 0
        flat[-1, i] = total
    return flat.reshape(B, rows, cols).astype(np.int8)


def bin_values(B):
    """Ascending, not representable in binary: the compiled float64 truncation of the quantised values matters."""
    return np.linspace(0.05, 1.0, B).astype(np.float32)


BOUNDS = np.array([0.0, 1.0], np.float32)

# ----------------------------------------------------------------------------- 1. whole-map sampling of one TDM
# name: B, (rows, cols), (max rows, max cols), (tx, ty), M, alphas of consecutive calls, forced segments ("nrow": the
# number of tile rows; None: the automatic choice), PMF kind.  The comment says what the case is meant to reach.
CASES = [
    # NW = 1
    ("b1_1x1", 1, (1, 1), (3, 20), (1, 1), 7, (1.0, 0.6), None, "sum100"),          # one cell, one bin
    ("b2_1xN", 2, (1, 45), (2, 64), (1, 40), 9, (0.6,), 1, "sum100"),               # one row; gm 6 cut by ty 40
    ("b3_Nx1", 3, (45, 1), (48, 16), (16, 16), 1, (1.0,), 2, "sum100"),             # one column: 15 empty tile columns
    ("b4_seq", 4, (37, 41), (40, 50), (3, 5), 33, (1.0, 0.01, 0.6), 2, "sum100"),   # M beyond SG_GM_MAX, three calls
    ("b4_127", 4, (20, 23), (20, 23), (3, 5), 9, (1.27,), 3, "sum127"),             # largest alpha with a table
    # NW = 0 (runtime width 2, 4, 7 words)
    ("b5_small_alpha", 5, (20, 50), (24, 60), (3, 5), 9, (0.004,), 3, "sum100"),    # tight table
    ("b7_tile1", 7, (30, 23), (31, 33), (1, 1), 7, (0.6,), "nrow", "sum100"),       # 1 x 1 tiles, segs = nrow
    ("b8_16x16", 8, (64, 70), (64, 80), (16, 16), 9, (1.27, 1.0), None, "sum127"),  # automatic segments
    ("b13_ragged", 13, (50, 29), (50, 29), (3, 5), 1, (0.6,), 1, "sum100"),        # M = 1, last tile column 5 of 6
    ("b16_segs33", 16, (70, 17), (72, 20), (1, 40), 7, (1.0,), 33, "sum100"),       # 33 segments of 3 rows over 70
    ("b28", 28, (33, 60), (35, 61), (4, 4), 33, (0.01, 1.0), "nrow", "sum100"),
    # NW = 3
    ("b9", 9, (31, 47), (40, 64), (3, 5), 9, (0.6,), 2, "sum100"),
    ("b12_tile16", 12, (16, 16), (16, 16), (16, 16), 33, (0.01,), None, "sum100"),  # one cell per tile
    ("b12_cols13", 12, (26, 13), (30, 13), (2, 3), 7, (1.0, 0.6), 3, "sum100"),     # cols < 16: one partial chunk
    # NW = 8
    ("b29", 29, (40, 35), (41, 35), (3, 5), 7, (1.0,), 3, "sum100"),
    ("b32_ty40", 32, (17, 100), (20, 112), (1, 40), 9, (0.004, 1.0), "nrow", "sum100"),  # ragged + empty columns
    # generic kernel on well-formed PMFs: more than 32 bins, wide tiles, alphas without a table
    ("b33", 33, (20, 30), (22, 30), (3, 5), 7, (0.6,), None, "sum100"),
    ("b64", 64, (25, 19), (25, 32), (16, 16), 2, (1.0,), None, "sum100"),
    ("b127", 127, (12, 13), (12, 13), (3, 5), 9, (1.27,), None, "sum127"),
    ("b28_ty300", 28, (12, 600), (12, 608), (2, 300), 2, (1.0,), None, "sum100"),   # gm 256 / 300 = 0
    ("b12_refused", 12, (21, 27), (24, 32), (3, 5), 9, (1.1, 0.0, 0.6), 2, "sum100"),  # q above every total; q = 0
    # generic kernel on ill-formed PMFs: the int8 clamp of the cumulative table
    ("ill_b1", 1, (19, 23), (19, 23), (3, 5), 5, (1.0, 1.27), None, "ill"),
    ("ill_b33", 33, (17, 21), (20, 21), (3, 5), 5, (1.27, 1.0), None, "ill"),
    ("ill_b127", 127, (9, 11), (9, 16), (2, 3), 3, (1.0, 1.27), None, "ill"),
]


def case_dict(row):
    name, B, shape, maxdim, tile, M, alphas, segs, kind = row
    return dict(name=name, B=B, shape=shape, maxdim=maxdim, tile=tile, M=M, alphas=alphas, segs=segs, kind=kind,
                seed=1000 + sum(map(ord, name)))


def forced_segs(c):
    if c["segs"] == "nrow":
        return -(-c["shape"][0] // c["tile"][0])
    return c["segs"]


def case_pmf(c):
    return sweep_pmf(c["seed"], c["B"], *c["shape"], kind=c["kind"])


def case_plans(c, lib_mod):
    """The plan of every call of case c."""
    pmf = case_pmf(c)
    return [plan(c["B"], c["shape"], c["tile"], c["M"], case_table_ok(lib_mod, pmf, a), forced_segs(c)) for a in c["alphas"]]


# ----------------------------------------------------------------------------- 2. lin/ang pairs through solve()
# name: lin bins, ang bins, map side (cells before padding), res, (tx, ty), M, alpha_dyn, forced segments, diverged
PAIRS = [
    ("p4", 4, 4, 40, 0.25, (3, 5), 9, 1.0, 2, False),
    ("p8", 8, 8, 44, 0.25, (4, 4), 10, 0.7, "nrow", False),
    ("p12", 12, 12, 50, 0.2, (16, 16), 33, 1.0, None, False),
    ("p32", 32, 32, 36, 0.25, (2, 3), 7, 0.6, 1, False),
    ("p12_segs33", 12, 12, 60, 0.2, (1, 8), 3, 1.0, 33, False),
    ("p8_diverged", 8, 8, 44, 0.25, (4, 4), 10, 0.7, 2, True),
    ("p32_diverged", 32, 32, 36, 0.25, (2, 3), 7, 1.0, None, True),
    ("p9_12", 9, 12, 40, 0.25, (3, 5), 9, 1.0, 2, False),          # unequal B, equal bpad: still fused
    ("p4_8", 4, 8, 40, 0.25, (3, 5), 9, 1.0, 2, False),            # unequal bpad: no fused launch
]

PAD_SPEED, DT = 5.0, 0.1


def pair_dict(row):
    name, B0, B1, H, res, tile, M, alpha, segs, diverged = row
    pad = int(math.ceil(PAD_SPEED * DT / res))
    return dict(name=name, B0=B0, B1=B1, H=H, res=res, tile=tile, M=M, alpha=alpha, segs=segs, diverged=diverged,
                pad=pad, shape=(H + 2 * pad, H + 2 * pad))


def pair_plan(p):
    """The plan of the pair's solve() (both PMFs sum to 100 per column: the table builds for alpha <= 1)."""
    segs = -(-p["shape"][0] // p["tile"][0]) if p["segs"] == "nrow" else p["segs"]
    return plan(p["B0"], p["shape"], p["tile"], p["M"], True, segs, B1=p["B1"], same_stream=not p["diverged"])


# ----------------------------------------------------------------------------- 3. boxed solves
# name: bins, map side, res, (tx, ty), M, T, reach disc on
BOXES = [
    ("box_nw1", 4, 80, 0.2, (16, 16), 5, 8, False),
    ("box_nw0", 6, 70, 0.2, (7, 5), 9, 8, False),
    ("box_nw3", 12, 90, 0.2, (4, 12), 12, 10, False),
    ("box_nw8", 32, 64, 0.25, (3, 5), 3, 8, False),
    ("box_disc", 12, 120, 0.1, (16, 16), 4, 12, True),              # the disc parks the box's corner tiles
]


def box_dict(row):
    name, B, H, res, tile, M, T, disc = row
    pad = int(math.ceil(PAD_SPEED * DT / res))
    return dict(name=name, B=B, H=H, res=res, tile=tile, M=M, T=T, disc=disc, pad=pad, shape=(H + 2 * pad, H + 2 * pad))


def static_box(T, vrange, dt, tr_abs_max, res, pxl, pyl, rows, cols, x0):
    """reach_box_decide (csrc/kernels.h) with the static bound: (row_lo, row_hi, col_lo, col_hi) or None (whole maps),
    and the reach disc (cx, cy, r) in cells.  Every input as the planner holds it (float32), the arithmetic in float64."""
    f = lambda v: float(np.float32(v))
    u = 5.9605e-8
    S = float(T) * max(abs(f(vrange[0])), abs(f(vrange[1])))
    Tu = float(T) * u
    x, y, res, pxl, pyl = f(x0[0]), f(x0[1]), f(res), f(pxl), f(pyl)
    R0 = f(dt) * f(tr_abs_max) * S * 1.0002
    D = (R0 + Tu * (abs(x) + abs(y))) / (1.0 - Tu)
    R = D + u * ((abs(x - pxl) + abs(y - pyl)) + 2.0 * D)
    fx0, fx1 = ((x - R) - pxl) / res, ((x + R) - pxl) / res
    fy0, fy1 = ((y - R) - pyl) / res, ((y + R) - pyl) / res
    if not (fx0 > 2.0 and fy0 > 2.0 and fx1 < cols - 3.0 and fy1 < rows - 3.0):
        return None, None
    box = (math.floor(fy0) - 1, math.floor(fy1) + 3, math.floor(fx0) - 1, math.floor(fx1) + 3)
    disc = (np.float32((x - pxl) / res), np.float32((y - pyl) / res), np.float32(np.float32(R / res + 3.0) * np.float32(1.0001)))
    return box, disc


def box_x0(b):
    """The robot's start: off-centre, so the box's first tile column starts inside a 16-cell chunk."""
    L = b["H"] * b["res"]
    return np.array([0.43 * L + 0.37 * b["res"], 0.55 * L - 0.21 * b["res"], 0.3])


def box_plan(b):
    """(plan, box, disc) of the boxed solve of case b (bounds [0, 1]: the largest traction is 1.0)."""
    rows, cols = b["shape"]
    pxl = -b["pad"] * b["res"]
    box, disc = static_box(b["T"], (0.0, 3.0), DT, 1.0, b["res"], pxl, pxl, rows, cols, box_x0(b))
    return plan(b["B"], b["shape"], b["tile"], b["M"], True, None, B1=b["B"], same_stream=True, box=box), box, disc
