"""Window-first sampling's kernel chain, executed on the host from the real source: the detecting windowed rollout
(rollout_win_kernel<..., WIN_DETECT>), the completion of the flagged maps (sample_window_complete_kernel) and the redo
of their rollouts (<..., WIN_REDO>), on maps just larger than the window whose cells outside the sampled rectangle
hold a sentinel -- what the rollout sees after the window-first sampling.  Against the exact oracle (libm provider,
the windowed kernel's order, wrap + clamp): the flags equal the escapes predicted from the oracle's trajectories
(tests/window_first_cases.py), the costs of unflagged maps and, after completion and redo, of every map equal the
oracle's bit for bit, and the completion re-walks exactly the map groups that hold a flag.

Buffers the planner allocates without clearing hold NaN here (ctrl beyond N): at N not a multiple of 32 the padding
lanes of the last chunk add that NaN to a cost they never store, which flagged every map before the flag store was
limited to live lanes -- the kernel compiled with the old store shows it."""
import numpy as np
import pytest

from oracle import mppi_ref as MR
from oracle import terrain_ref as TR
from oracle import xoroshiro as X
from tests import emu_rollout_win, emu_sampler
from tests import rollout_edge_cases as EC
from tests import window_first_cases as WF
from tests.emu_sampler import cumulative_table
from tests.test_exact_oracle_cpu import EXACT, assert_equal
from tests.test_rollout_emulated_cpu import _c, _fparams, _p, _ratios

F32 = np.float32
ROWS, COLS = 250, 256                 # the map (and its allocation): just larger than the 240 x 232 window
TILE = (4, 64)                        # sampler tiles: 64 threads per tile row, so 256 / 64 = 4 maps per CTA
SENTINEL = -77                        # not -128 (the detecting kernel's own escape code), no sampled code
BINS, BOUNDS = np.array([0.0, 1.0]), np.array([0.0, 1.0], F32)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("emu_window_first"))
    return dict(win=emu_rollout_win.build(d), any_lane=emu_rollout_win.build(d, flag_any_lane=True),
                sampler=emu_sampler.build(d, more=("window_complete",)))


def _random_pmf(rng):
    """Two bins (traction 0 and 1) with a random split of the mass in every cell."""
    p0 = rng.integers(0, 101, (ROWS, COLS))
    return np.stack([p0, 100 - p0]).astype(np.int8)


def _whole_maps(pmf, states, M):
    g = np.full((M, ROWS, COLS), SENTINEL, np.int8)
    TR.sample_grids(g, pmf, states.copy(), BINS, BOUNDS, 1.0, TILE, M)
    return g


def _gate_row(pmf_gate, states, M, col, want):
    """A row whose gate cell (row, col) samples closed (code 0) / open (100) in the maps as `want` (M booleans: open)."""
    w = _whole_maps(pmf_gate, states, M)
    for r in range(20, ROWS - 20):
        if ((w[:, r, col] == 100) == np.asarray(want)).all():
            return r
    raise AssertionError("no row with gate pattern %s" % (want,))


# name: (N, M, T, res, robot cell (col, row) or "gate", heading, u_v, u_std, expected flags: "none" | "last" | "all")
CASES = {
    "none": (40, 6, 40, 0.4, (128.5, 125.5), 0.7, 1.0, (0.5, 0.5), "none"),
    "last-map": (40, 6, 40, 0.4, "gate", np.pi, 3.0, (0.2, 0.001), "last"),
    "all-maps-y": (33, 6, 50, 0.1, (128.5, 125.5), np.pi / 2, 3.0, (0.2, 0.001), "all"),
    "wrapped-negative-x": (40, 6, 30, 0.4, (3.5, 60.5), np.pi, 3.0, (0.2, 0.001), "all"),
    "ragged-nan-33": (33, 5, 20, 0.4, (128.5, 125.5), -2.0, 1.0, (0.5, 0.5), "none"),
    "ragged-nan-40": (40, 6, 20, 0.4, (100.5, 140.5), 2.5, 1.0, (0.5, 0.5), "none"),
}


def _case(name, seed=5):
    N, M, T, res, cell, th, u, us, expect = CASES[name]
    states = X.create_states(TILE[0] * TILE[1] * M, seed)
    pmf = np.zeros((2, ROWS, COLS), np.int8)
    pmf[1] = 100                                          # traction 1 everywhere
    rng = np.random.default_rng(seed + len(name))
    pmf_ang = _random_pmf(rng)              # random angular traction: lin and ang maps differ
    if expect == "none":                                  # and random linear traction where nothing must escape
        pmf = _random_pmf(rng)
    if cell == "gate":                                    # a gate cell at column 2 closed in every map but the last
        gate = pmf.copy()
        gate[:, :, 2] = [[50], [50]]
        r = _gate_row(gate, states, M, 2, [False] * (M - 1) + [True])
        pmf[:, r, 2] = [50, 50]
        cell = (5.5, r + 0.5)
    x0 = [cell[0] * res, cell[1] * res, th]
    return dict(N=N, M=M, T=T, res=F32(res), x0=x0, expect=expect, states=states, pmf=pmf, pmf_ang=pmf_ang,
                noise=(rng.standard_normal((N, T, 2)) * us).astype(F32),
                u_cur=np.stack([np.full(T, u), np.zeros(T)], 1).astype(F32), u_std=us, goal=[x0[0] + 300.0, x0[1]],
                obs=np.zeros((ROWS, COLS), np.int8), unk=np.zeros((ROWS, COLS), np.int8))


def _oracle(s, lin, ang):
    lim_x, lim_y = [0.0, COLS * float(s["res"])], [0.0, ROWS * float(s["res"])]
    return MR.rollout_costs(MR.MODE_STOCHASTIC, lin, ang, BOUNDS, BOUNDS, s["obs"], s["unk"], s["res"], lim_x, lim_y,
                            [0.0, 3.0], [-np.pi, np.pi], s["goal"], 0.01, 1e5, 1e2, 0.5, 1.0, s["u_std"], s["x0"], 0.1,
                            1.0, s["noise"], s["u_cur"], return_states=True, arith=EXACT, ctrl_order="presummed",
                            wrap_clamp=True)


def _rollout(lib, s, lin, ang, costs_mn, esc, mode, ctrl_pad):
    N, M, T = s["N"], s["M"], s["T"]
    f = _fparams(s["res"], 0.0, 0.0, 0.1, s["x0"], s["goal"], 0.5, 0.01, 1.0, s["u_std"], [0.0, 3.0], [-np.pi, np.pi],
                 1e5, 1e2, 1.0, BOUNDS[0], BOUNDS[0])
    geo = _c([ROWS, COLS, ROWS, COLS, COLS, COLS, T, N, M], np.int32)
    origin = np.zeros(4, np.int32)
    rc = lib.emu_rollout_win_esc(_p(f), _p(geo), _p(_ratios(BOUNDS, BOUNDS)), _p(lin), _p(ang), _p(s["obs"]),
                                 _p(s["unk"]), _p(s["noise"]), _p(s["u_cur"]), _p(costs_mn), _p(esc), mode,
                                 float(ctrl_pad), 1, _p(origin))
    assert rc == 0
    return tuple(int(v) for v in origin)


def _chain(emu, name, rollout_lib="win"):
    s = _case(name)
    N, M, res = s["N"], s["M"], s["res"]
    whole = [_whole_maps(s["pmf"], s["states"], M), _whole_maps(s["pmf_ang"], s["states"], M)]   # fused: lin's stream
    want, states = _oracle(s, *whole)
    wx0, wy0, ww, wh = EC.window_origin(s["x0"][0], s["x0"][1], 0.0, 0.0, res, COLS, ROWS)
    rect = WF.window_rect(wx0, wy0, ww, wh, ROWS, COLS)
    flags, reads = WF.escapes(states, 0.0, 0.0, res, s["goal"], 0.5, rect, ROWS, COLS, ROWS, COLS, EXACT)
    out = np.where(WF.outside_rect(whole[0].shape, rect), np.int8(SENTINEL), 0)
    maps = [_c(np.where(out != 0, out, w), np.int8) for w in whole]
    esc = np.zeros(M, np.uint8)
    costs = np.full((M, N), np.nan, F32)
    origin = _rollout(emu[rollout_lib], s, maps[0], maps[1], costs, esc, 1, np.nan)
    assert origin == (wx0, wy0, ww, wh)
    return dict(s=s, whole=whole, want=want, rect=rect, flags=flags, reads=reads, maps=maps, esc=esc, costs=costs)


@pytest.mark.parametrize("name", [n for n in CASES if not n.startswith("ragged")])
def test_detect_complete_redo_chain_equals_oracle(emu, name):
    c = _chain(emu, name)
    s, flags, M, N = c["s"], c["flags"], c["s"]["M"], c["s"]["N"]
    expect = dict(none=[False] * M, last=[False] * (M - 1) + [True], all=[True] * M)[s["expect"]]
    assert list(flags) == expect, (name, flags, c["rect"])
    assert (c["whole"][0] != c["whole"][1]).any()         # lin and ang maps differ: a swap would show
    if name == "wrapped-negative-x":                      # every escaping read comes from an index below 0
        assert c["reads"] and all(xi < 0 <= c["rect"][3] <= gx for _, _, _, _, xi, _, gx in c["reads"])
    for n, m, t, yi, xi, gy, gx in c["reads"][:1]:                # an escape would read a byte that differs from the whole map's
        assert c["maps"][0][m, gy, gx] == SENTINEL != c["whole"][0][m, gy, gx]
    # detect: the flags, and the costs of the unflagged maps
    assert list(c["esc"] != 0) == list(flags), (c["esc"], flags)
    assert_equal(c["costs"][~flags].T.copy(), c["want"][:, ~flags].copy(), "%s: unflagged maps after detect" % name)
    # completion from the pre-call states
    cums = [cumulative_table(s["pmf"], 4), cumulative_table(s["pmf_ang"], 4)]
    qv = np.zeros(128, np.int8)
    qv[:2] = TR.quantise_bin_values(BINS, BOUNDS)
    clear = np.ones(M, np.uint8)
    record = np.full(6, -1, np.int32)
    before = [m.copy() for m in c["maps"]]
    states = np.ascontiguousarray(s["states"].copy())     # the pre-call states: read, never written (write_states 0)
    gm = emu["sampler"].emu_window_complete(_p(c["maps"][0]), _p(c["maps"][1]), _p(cums[0]), _p(cums[1]),
                                            _p(states), _p(qv), _p(qv), 4, ROWS, COLS,
                                            ROWS, COLS, TILE[0], TILE[1], M, 1.0, 100, _p(c["esc"]), _p(clear),
                                            _p(record))
    assert gm == 4, gm
    assert (states == s["states"]).all()
    walked = WF.completed_maps(flags, gm)
    for k in range(2):
        assert (c["maps"][k][walked] == c["whole"][k][walked]).all(), (name, k)
        assert (c["maps"][k][~walked] == before[k][~walked]).all(), (name, k)
    assert list(record) == [0, 0, ROWS, 0, COLS, int(flags.sum())], record
    assert (clear == 0).all()
    # redo of the flagged maps on the completed maps: every cost is the oracle's
    _rollout(emu["win"], s, c["maps"][0], c["maps"][1], c["costs"], c["esc"], 2, np.nan)
    assert_equal(c["costs"].T.copy(), c["want"], "%s: every map after the redo" % name)


@pytest.mark.parametrize("name", ["ragged-nan-33", "ragged-nan-40"])
def test_padding_lanes_flag_no_map(emu, name):
    """N 33 / 40 with NaN in ctrl beyond N and no escape: no flag, and every cost the oracle's.  With the flag store of
    every lane (the kernel before padding lanes were excluded) the same launch flags every map."""
    c = _chain(emu, name)
    assert not c["flags"].any()
    assert not c["esc"].any(), c["esc"]
    assert_equal(c["costs"].T.copy(), c["want"], name)
    old = _chain(emu, name, rollout_lib="any_lane")
    assert (old["esc"] == 1).all(), old["esc"]
    assert_equal(old["costs"].T.copy(), old["want"], name + ", every lane flags")
