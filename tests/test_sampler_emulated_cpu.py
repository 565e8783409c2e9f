"""The sampler kernel's REAL source, executed on the host by tests/emu_sampler.py, against the oracle's
restatement of sample_grids_numba (terrain.py:633-694): sampled maps and advanced generator states bit for bit,
for the template variants solve() uses (12 bins = 3 words, fused lin+ang), the generic-width variant, row
segments with GF(2) jump-ahead, partial map groups and ragged tiles."""
import numpy as np
import pytest

from oracle import terrain_ref as TR
from oracle import xoroshiro as X
from tests.emu_sampler import build, cumulative_table
from tests.scenarios import random_pmf


@pytest.fixture(scope="module", params=["as-built", "values-in-registers", "one-popc"])
def emu(request, tmp_path_factory):
    """The kernel as built, and with its compile-time A/B switches flipped (value lookup through a register table;
    the bytes >= q counted with shifts + one POPC instead of one POPC per word)."""
    import __graft_entry__
    __graft_entry__.build_engine()
    d = str(tmp_path_factory.mktemp("emu"))
    if request.param == "values-in-registers":
        return build(d, values_in_registers=True)
    if request.param == "one-popc":
        return build(d, popc_per_word=False)
    return build(d)


def _ptr(a):
    return a.ctypes.data_as(__import__("ctypes").c_void_p)


@pytest.mark.parametrize("B,nt,segs,alpha,M,shape,tdim", [
    (12, 2, 1, 1.0, 10, (37, 41), (4, 4)),      # the variant solve() runs at config 5 (<2,3>), partial map group
    (12, 2, 3, 0.6, 9, (37, 41), (4, 4)),       # row segments: jump-ahead, double-buffered states
    (12, 1, 2, 0.9, 3, (21, 50), (3, 5)),       # single TDM, ragged tiles (last tile column narrower)
    (5, 2, 2, 1.0, 8, (19, 23), (2, 4)),        # 5 bins -> 2 words: generic-width variant (NW = 0)
    (32, 1, 1, 0.3, 2, (12, 18), (2, 2)),       # 32 bins -> 8 words (config 4's PMF width)
    (4, 2, 4, 1.27, 17, (16, 16), (4, 2)),      # 1 word, largest representable alpha, 3 map groups
])
def test_sampler_kernel_source_matches_oracle(emu, B, nt, segs, alpha, M, shape, tdim):
    rows, cols = shape
    tx, ty = tdim
    rng = np.random.default_rng(B * 100 + M)
    bpad = (B + 3) // 4 * 4
    bin_values = np.linspace(0, 1, B)
    bounds = np.array([0.0, 1.0], dtype=np.float32)
    pmfs = [random_pmf(rng, B, rows, cols) for _ in range(nt)]
    if alpha > 1.0:                                  # thresholds up to 127: column totals must reach them
        pmfs = [np.concatenate([p[:-1], (p[-1:] + 27)], axis=0).astype(np.int8) for p in pmfs]
    grid_rows, pitch = rows + 3, (cols + 5 + 15) // 16 * 16
    states0 = X.create_states(tx * ty * M, 7)
    q = np.zeros(128, dtype=np.int8)
    q[:B] = TR.quantise_bin_values(bin_values, bounds)
    grids = [np.full((M, grid_rows, pitch), -7, dtype=np.int8) for _ in range(nt)]
    cums = [cumulative_table(p, bpad) for p in pmfs]
    st_in = np.ascontiguousarray(states0.copy())
    st_out = np.zeros_like(st_in)
    q_cap = int(min(int(np.cumsum(p.astype(np.int64), axis=0)[-1].min()) for p in pmfs))
    rc = emu.emu_sample_v2(nt, _ptr(grids[0]), _ptr(grids[nt - 1]), _ptr(cums[0]), _ptr(cums[nt - 1]), _ptr(st_in),
                           _ptr(st_out), _ptr(q), _ptr(q), bpad, rows, cols, grid_rows, pitch, tx, ty, M, segs,
                           float(alpha), min(q_cap, 127), None, None)
    assert rc == 0
    for k in range(nt):
        want = np.full((M, grid_rows, pitch), -7, dtype=np.int8)
        st = states0.copy()
        TR.sample_grids(want, pmfs[k], st, bin_values, bounds, alpha, (tx, ty), M)
        assert (grids[k][:, :rows, :cols] == want[:, :rows, :cols]).all(), "TDM %d" % k
        assert (grids[k][:, rows:, :] == -7).all()               # nothing written outside the map rows
        assert (st_out == st).all()                               # generator states advanced exactly alike
    assert (st_in == states0).all()                               # the input buffer is not modified (double buffer)


def test_sampler_kernel_source_random_configurations(emu):
    """Fuzz: random map shapes, thread tiles, map counts, bin counts, segment counts, alphas and TDM counts."""
    rng = np.random.default_rng(2024)
    for case in range(10):
        B = int(rng.choice([2, 3, 4, 5, 8, 12, 13, 16, 20, 32]))
        nt = int(rng.integers(1, 3))
        tx, ty = int(rng.integers(1, 6)), int(rng.integers(1, 7))
        rows, cols = int(rng.integers(tx, 40)), int(rng.integers(ty, 44))
        M = int(rng.integers(1, 20))
        segs = int(rng.integers(1, 6))
        alpha = float(rng.choice([1.0, 0.9, 0.5, 0.13, 1.0]))
        bpad = (B + 3) // 4 * 4
        bin_values = np.linspace(0, 1, B)
        bounds = np.array([0.0, 1.0], dtype=np.float32)
        pmfs = [random_pmf(rng, B, rows, cols) for _ in range(nt)]
        grid_rows, pitch = rows + int(rng.integers(0, 4)), (cols + int(rng.integers(0, 9)) + 15) // 16 * 16
        states0 = X.create_states(tx * ty * M, int(rng.integers(1, 1000)))
        q = np.zeros(128, dtype=np.int8)
        q[:B] = TR.quantise_bin_values(bin_values, bounds)
        grids = [np.full((M, grid_rows, pitch), -7, dtype=np.int8) for _ in range(nt)]
        cums = [cumulative_table(p, bpad) for p in pmfs]
        st_in = np.ascontiguousarray(states0.copy())
        st_out = np.zeros_like(st_in)
        rc = emu.emu_sample_v2(nt, _ptr(grids[0]), _ptr(grids[nt - 1]), _ptr(cums[0]), _ptr(cums[nt - 1]), _ptr(st_in),
                               _ptr(st_out), _ptr(q), _ptr(q), bpad, rows, cols, grid_rows, pitch, tx, ty, M, segs, alpha, 100, None, None)
        assert rc == 0, case
        for k in range(nt):
            want = np.full((M, grid_rows, pitch), -7, dtype=np.int8)
            st = states0.copy()
            TR.sample_grids(want, pmfs[k], st, bin_values, bounds, alpha, (tx, ty), M)
            tag = "case %d: B=%d nt=%d t=(%d,%d) map=(%d,%d) M=%d segs=%d alpha=%g" % (case, B, nt, tx, ty, rows, cols, M, segs, alpha)
            assert (grids[k][:, :rows, :cols] == want[:, :rows, :cols]).all(), tag
            assert (st_out == st).all(), tag


def test_sampler_kernel_source_boxed_launch(emu):
    """Reach-box launches (solve() only): inside the box the maps are those of a whole-map walk, outside the box
    nothing is written, and advance_states_kernel leaves every generator exactly where the whole-map walk does --
    random boxes, tiles, segment counts, map counts (maps per CTA follow the number of active tile columns)."""
    rng = np.random.default_rng(77)
    skipped = 0
    for case in range(14):
        B = int(rng.choice([3, 5, 12, 12, 32]))
        nt = int(rng.integers(1, 3))
        tx, ty = int(rng.integers(1, 7)), int(rng.integers(1, 9))
        rows, cols = int(rng.integers(max(tx, 6), 60)), int(rng.integers(max(ty, 6), 70))
        M = int(rng.integers(1, 40))
        segs = int(rng.integers(1, 6))
        alpha = float(rng.choice([1.0, 0.7, 0.25]))
        r_lo = int(rng.integers(0, rows - 1)); r_hi = int(rng.integers(r_lo + 1, rows + 1))
        c_lo = int(rng.integers(0, cols - 1)); c_hi = int(rng.integers(c_lo + 1, cols + 1))
        box = np.array([r_lo, r_hi, c_lo, c_hi], dtype=np.int32)
        # every second case: the reach disc inscribed in the box (what solve() passes), centre at a fractional cell
        disc = None
        if case % 2:
            cy, cx = 0.5 * (r_lo + r_hi) + rng.uniform(-0.4, 0.4), 0.5 * (c_lo + c_hi) + rng.uniform(-0.4, 0.4)
            disc = np.array([cx, cy, 0.5 * max(r_hi - r_lo, c_hi - c_lo) + 0.5], dtype=np.float32)
        bpad = (B + 3) // 4 * 4
        bin_values = np.linspace(0, 1, B)
        bounds = np.array([0.0, 1.0], dtype=np.float32)
        pmfs = [random_pmf(rng, B, rows, cols) for _ in range(nt)]
        grid_rows, pitch = rows + int(rng.integers(0, 3)), (cols + int(rng.integers(0, 9)) + 15) // 16 * 16
        states0 = X.create_states(tx * ty * M, int(rng.integers(1, 1000)))
        q = np.zeros(128, dtype=np.int8)
        q[:B] = TR.quantise_bin_values(bin_values, bounds)
        grids = [np.full((M, grid_rows, pitch), -7, dtype=np.int8) for _ in range(nt)]
        cums = [cumulative_table(p, bpad) for p in pmfs]
        st_in = np.ascontiguousarray(states0.copy())
        st_out = np.zeros_like(st_in)
        rc = emu.emu_sample_v2(nt, _ptr(grids[0]), _ptr(grids[nt - 1]), _ptr(cums[0]), _ptr(cums[nt - 1]), _ptr(st_in),
                               _ptr(st_out), _ptr(q), _ptr(q), bpad, rows, cols, grid_rows, pitch, tx, ty, M, segs, alpha, 100,
                               _ptr(box), _ptr(disc) if disc is not None else None)
        tag = "case %d: B=%d nt=%d t=(%d,%d) map=(%d,%d) M=%d segs=%d alpha=%g box=%s" % (
            case, B, nt, tx, ty, rows, cols, M, segs, alpha, box.tolist())
        assert rc == 0, tag
        nrow, ncol = -(-rows // tx), -(-cols // ty)
        # what a boxed launch may touch: the box rows x the tile columns covering the box columns
        tc_lo, tc_hi = (c_lo // ncol) * ncol, min((((c_hi - 1) // ncol) + 1) * ncol, cols)
        for k in range(nt):
            want = np.full((M, grid_rows, pitch), -7, dtype=np.int8)
            st = states0.copy()
            TR.sample_grids(want, pmfs[k], st, bin_values, bounds, alpha, (tx, ty), M)
            inside = np.zeros((grid_rows, pitch), bool)
            inside[r_lo:r_hi, tc_lo:tc_hi] = True
            assert (grids[k][:, ~inside] == -7).all(), tag                    # nothing outside the box's tile columns
            if disc is None:
                assert (grids[k][:, inside] == want[:, inside]).all(), tag
            else:
                # every cell that holds a position within r of the centre is sampled (= the whole-map value); a cell
                # the launch did not sample is untouched
                yy, xx = np.mgrid[0:grid_rows, 0:pitch]
                dyc = np.maximum(np.maximum(yy - disc[1], disc[1] - (yy + 1)), 0)
                dxc = np.maximum(np.maximum(xx - disc[0], disc[0] - (xx + 1)), 0)
                need = inside & (dxc ** 2 + dyc ** 2 <= float(disc[2]) ** 2)
                got = grids[k]
                assert (got[:, need] == want[:, need]).all(), tag
                assert ((got == want) | (got == -7))[:, inside].all(), tag
                skipped += int(((got == -7) & inside[None]).sum())
            assert (st_out == st).all(), tag
        assert (st_in == states0).all()


def test_sampler_kernel_source_disc_parks_corner_tiles(emu):
    """A 64 x 64 map in 8 x 8 tiles, box = the interior, disc of radius 26 around the centre, 2-row segments: the
    segments near the top and the bottom of the box sample only the tile columns under the disc (the corner tiles
    stay untouched), every cell the disc needs equals the whole-map value, the generators advance as for whole maps."""
    rng = np.random.default_rng(5)
    B, nt, tx, ty, rows, cols, M, segs, alpha = 12, 2, 8, 8, 64, 64, 5, 4, 1.0
    box = np.array([4, 60, 4, 60], dtype=np.int32)
    disc = np.array([32.3, 31.6, 26.0], dtype=np.float32)
    bpad = 12
    bin_values = np.linspace(0, 1, B)
    bounds = np.array([0.0, 1.0], dtype=np.float32)
    pmfs = [random_pmf(rng, B, rows, cols) for _ in range(nt)]
    grid_rows, pitch = rows, 64
    states0 = X.create_states(tx * ty * M, 3)
    q = np.zeros(128, dtype=np.int8)
    q[:B] = TR.quantise_bin_values(bin_values, bounds)
    grids = [np.full((M, grid_rows, pitch), -7, dtype=np.int8) for _ in range(nt)]
    cums = [cumulative_table(p, bpad) for p in pmfs]
    st_in = np.ascontiguousarray(states0.copy())
    st_out = np.zeros_like(st_in)
    assert emu.emu_sample_v2(nt, _ptr(grids[0]), _ptr(grids[1]), _ptr(cums[0]), _ptr(cums[1]), _ptr(st_in), _ptr(st_out),
                             _ptr(q), _ptr(q), bpad, rows, cols, grid_rows, pitch, tx, ty, M, segs, alpha, 100, _ptr(box),
                             _ptr(disc)) == 0
    yy, xx = np.mgrid[0:rows, 0:cols]
    dyc = np.maximum(np.maximum(yy - disc[1], disc[1] - (yy + 1)), 0)
    dxc = np.maximum(np.maximum(xx - disc[0], disc[0] - (xx + 1)), 0)
    need = (dxc ** 2 + dyc ** 2 <= 26.0 ** 2) & (yy >= 4) & (yy < 60) & (xx >= 4) & (xx < 60)
    for k in range(nt):
        want = np.full((M, grid_rows, pitch), -7, dtype=np.int8)
        st = states0.copy()
        TR.sample_grids(want, pmfs[k], st, bin_values, bounds, alpha, (tx, ty), M)
        assert (grids[k][:, need] == want[:, need]).all()
        assert ((grids[k] == want) | (grids[k] == -7)).all()
        assert (grids[k][:, 4:8, 4:8] == -7).all() and (grids[k][:, 56:60, 56:60] == -7).all()     # corner tiles parked
        assert (st_out == st).all()
