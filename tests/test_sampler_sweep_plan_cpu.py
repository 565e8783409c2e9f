"""The GPU sampler sweep (tests/test_gpu_sampler_sweep.py) reaches every variant of the sampler's launch plan: the case
tables of tests/sampler_sweep_cases.py, run through the restated plan, cover each kernel instantiation and each
geometric edge, so an edit of a table cannot silently drop one.  The staged single-TDM cases also run through the
kernel's source on the host (tests/emu_sampler.py) against the oracle, so a GPU-only mismatch points at the hardware
build rather than at the test."""
import ctypes as C

import numpy as np
import pytest

from oracle import terrain_ref as TR
from oracle import xoroshiro as X
from tests import sampler_sweep_cases as S


@pytest.fixture(scope="module")
def libmod():
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def plans(libmod):
    """(name, alpha, plan) of every sampling call of the three tables."""
    out = []
    for row in S.CASES:
        c = S.case_dict(row)
        out += [(c["name"], a, p) for a, p in zip(c["alphas"], S.case_plans(c, libmod))]
    for row in S.PAIRS:
        p = S.pair_dict(row)
        out.append((p["name"], p["alpha"], S.pair_plan(p)))
    for row in S.BOXES:
        b = S.box_dict(row)
        out.append((b["name"], 1.0, S.box_plan(b)[0]))
    return out


def _covered(plans, what, pred):
    hits = sorted({name for name, _, p in plans if pred(p)})
    print("%-28s %s" % (what, ", ".join(hits)))
    assert hits, "no case of the sweep reaches: " + what


def test_every_variant_is_reached(plans):
    for nw in (1, 0, 3, 8):
        for nt in (1, 2):
            _covered(plans, "staged NT=%d NW=%d" % (nt, nw),
                     lambda p, nw=nw, nt=nt: p["kernel"] == "staged" and p["NW"] == nw and p["nt"] == nt)
    _covered(plans, "segs = 1", lambda p: p["kernel"] == "staged" and p["segs"] == 1)
    _covered(plans, "1 < segs < nrow", lambda p: p["kernel"] == "staged" and 1 < p["segs"] < p["nrow"])
    _covered(plans, "segs = nrow > 1", lambda p: p["kernel"] == "staged" and p["segs"] == p["nrow"] > 1)
    _covered(plans, "segs * seg_rows > nrow", lambda p: p["kernel"] == "staged" and p["segs_over"])
    _covered(plans, "segs = 33", lambda p: p["kernel"] == "staged" and p["segs"] == 33)
    _covered(plans, "ragged last tile column", lambda p: p["kernel"] == "staged" and p["ragged_col"])
    _covered(plans, "empty tile columns", lambda p: p["kernel"] == "staged" and p["empty_col"])
    _covered(plans, "ragged last tile row", lambda p: p["kernel"] == "staged" and p["ragged_row"])
    _covered(plans, "unaligned window start", lambda p: p["kernel"] == "staged" and p["cs0_unaligned"])
    _covered(plans, "partial last chunk", lambda p: p["kernel"] == "staged" and p["chunk_tail"])
    _covered(plans, "partial map group", lambda p: p["kernel"] == "staged" and p["partial_group"])
    _covered(plans, "gm cut by wide tiles", lambda p: p["kernel"] == "staged" and p["gm_cut"])
    _covered(plans, "boxed fused launch", lambda p: p["kernel"] == "staged" and p["boxed"] and p["nt"] == 2)


def test_generic_kernel_cases(libmod):
    """The generic kernel runs on well-formed PMFs (more than 32 bins, tiles too wide, alphas without a table) and on
    ill-formed ones (negative entries, running sums past 127: the int8 clamp of the cumulative table)."""
    kinds = set()
    for row in S.CASES:
        c = S.case_dict(row)
        ok, _ = S.pmf_valid(S.case_pmf(c))
        assert ok == (c["kind"] != "ill"), c["name"]
        for p in S.case_plans(c, libmod):
            if p["kernel"] == "generic":
                kinds.add(("well-formed" if ok else "ill-formed", "bpad>32" if p["bpad"] > 32 else
                           "no fit" if not S.fits(0, c["tile"][1], c["tile"][1], c["shape"][1], p["bpad"], p["bpad"],
                                                  p["gm"], 1) else "no table"))
    print(sorted(kinds))
    assert {("well-formed", "bpad>32"), ("well-formed", "no fit"), ("well-formed", "no table"),
            ("ill-formed", "bpad>32")} <= kinds
    ill = [S.case_pmf(S.case_dict(r)) for r in S.CASES if r[-1] == "ill"]
    acc = [np.cumsum(p.astype(np.int64), axis=0) for p in ill]
    assert any((a > 127).any() for a in acc) and any((a < -128).any() for a in acc)


def test_alphas_and_tables(libmod):
    """The alpha list: 1.0, 0.6, 1.27 with a table (column totals 127), the tight tables of 0.01 and 0.004, and
    refusals (q above every column total, q = 0 everywhere)."""
    seen = set()
    for row in S.CASES:
        c = S.case_dict(row)
        pmf = S.case_pmf(c)
        for a in c["alphas"]:
            seen.add((a, S.case_table_ok(libmod, pmf, a)))
    print(sorted(seen))
    assert {(1.0, True), (0.6, True), (1.27, True), (0.01, True), (0.004, True), (1.1, False), (0.0, False)} <= seen


def test_first_and_last_bin_columns():
    """Columns with all their mass on the first or the last bin, in every table-driven PMF kind."""
    for B in (2, 5, 32):
        for kind, total in (("sum100", 100), ("sum127", 127)):
            p = S.sweep_pmf(3, B, 6, 7, kind).astype(np.int64)
            assert (p.sum(0) == total).all()
            assert ((p[0] == total).any() and (p[-1] == total).any())


def test_box_plans():
    """Each boxed case leaves a box inside the map with the staged fused launch; the NW list of the boxed cases."""
    nws = set()
    for row in S.BOXES:
        b = S.box_dict(row)
        p, box, disc = S.box_plan(b)
        assert box is not None and p["kernel"] == "staged" and p["nt"] == 2, b["name"]
        assert 0 <= box[0] < box[1] <= b["shape"][0] and 0 <= box[2] < box[3] <= b["shape"][1]
        nws.add(p["NW"])
    assert nws == {1, 0, 3, 8}


@pytest.fixture(scope="module")
def emu(libmod, tmp_path_factory):
    from tests.emu_sampler import build
    return build(str(tmp_path_factory.mktemp("sweep_emu")))


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def test_staged_cases_through_the_emulated_kernel(libmod, emu):
    """Every staged single-TDM call of the whole-map table, small enough for the host, through the kernel source: the
    same maps (pitch padding included) and states as the oracle."""
    from tests.emu_sampler import cumulative_table
    ran = 0
    for row in S.CASES:
        c = S.case_dict(row)
        plans = S.case_plans(c, libmod)
        if any(p["kernel"] != "staged" for p in plans):
            continue
        tx, ty = c["tile"]
        rows, cols = c["shape"]
        ctas = plans[0]["segs"] * tx * -(-c["M"] // plans[0]["gm"])
        if ctas * plans[0]["threads"] > 40000:
            continue
        pmf, bv = S.case_pmf(c), S.bin_values(c["B"])
        bpad = plans[0]["bpad"]
        _, cap = S.pmf_valid(pmf)
        q = np.zeros(128, np.int8)
        q[:c["B"]] = TR.quantise_bin_values(bv, S.BOUNDS)
        grid_rows, pitch = c["maxdim"][0], -(-c["maxdim"][1] // 16) * 16
        grid = np.full((c["M"], grid_rows, pitch), S.SENTINEL, np.int8)
        want = grid.copy()
        cum = cumulative_table(pmf, bpad)
        st = np.ascontiguousarray(X.create_states(tx * ty * c["M"], c["seed"]))
        st_w = st.copy()
        for a, p in zip(c["alphas"], plans):
            out = np.zeros_like(st)
            rc = emu.emu_sample_v2(1, _ptr(grid), _ptr(grid), _ptr(cum), _ptr(cum), _ptr(st), _ptr(out), _ptr(q), _ptr(q),
                                   bpad, rows, cols, grid_rows, pitch, tx, ty, c["M"], p["segs"], float(a), min(cap, 127),
                                   None, None)
            assert rc == 0, c["name"]
            TR.sample_grids(want, pmf, st_w, bv, S.BOUNDS, a, c["tile"], c["M"])
            assert (grid == want).all(), (c["name"], a)
            assert (out == st_w).all(), (c["name"], a)
            st = out
        ran += 1
    print("%d cases emulated" % ran)
    assert ran >= 6
