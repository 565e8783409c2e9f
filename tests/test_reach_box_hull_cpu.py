"""The box of a TDM pair shared by several planners (reach_box_hull_add / reach_box_hull_close, csrc/kernels.h) and the
group-aware trial sampler that decides it on the device (sample_grids_v2_group_box_batch_kernel +
advance_states_group_batch_kernel, csrc/sample.cu), both compiled from their REAL source for the host:
- the hull against a Python restatement of its rules over a few thousand random member sets: one member is exactly its
  reach_box_decide result, disc included; the hull contains every member's box; a whole-map member gives whole maps;
  a hull whose sampler launch does not fit gives whole maps;
- the group kernel on one pair shared by three planners, all, one or none of them running, against the oracle's
  whole-map sampling (oracle/terrain_ref.py sample_grids): the hull's cells and every generator state byte for byte,
  the records of the group and of each running member, and nothing written when no member runs."""
import ctypes as C

import numpy as np
import pytest

from oracle import terrain_ref as TR
from oracle import xoroshiro as X
from tests import emu_core
from tests.emu_sampler import cumulative_table, kernels
from tests.scenarios import random_pmf

HARNESS = r'''
using namespace b200;
static ReachBoxConst rb_const(const int* g, const float* gf, const int* mi, const float* mf) {
  ReachBoxConst c{};
  c.rows = g[0]; c.cols = g[1]; c.nt = g[2]; c.tx = g[3]; c.ty = g[4]; c.num_maps = g[5]; c.bpad0 = g[6]; c.bpad1 = g[7];
  c.res = gf[0]; c.pxl = gf[1]; c.pyl = gf[2]; c.tr_abs_max = gf[3];
  c.mode = mi[0]; c.disc = mi[1]; c.T = mi[2];
  c.vr0 = mf[0]; c.vr1 = mf[1]; c.dt = mf[2];
  return c;
}
static void rb_out(const ReachBox& b, int ret, int* oi, float* of) {
  const int v[10] = {ret, b.geo, b.how, b.row_lo, b.row_hi, b.col_lo, b.col_hi, b.tiy_lo, b.nact, b.gm};
  for (int i = 0; i < 10; ++i) oi[i] = v[i];
  of[0] = b.cx; of[1] = b.cy; of[2] = b.r;
}
// n members of one pair: geometry g[8] (rows, cols, nt, tx, ty, num_maps, bpad0, bpad1), gf[4] (res, pxl, pyl,
// tr_abs_max); member j: mi[3j..] (mode, disc, T), mf[6j..] (vr0, vr1, dt, x, y, reach).  Each member's decision into
// oi[10j..] / of[3j..], the hull (sample_finish_group's order: decide, add, close) into oi[10n..] / of[3n..].
extern "C" int emu_hull(int n, const int* g, const float* gf, const int* mi, const float* mf, int* oi, float* of) {
  ReachBox h;
  ReachBoxConst c;
  for (int j = 0; j < n; ++j) {
    c = rb_const(g, gf, mi + 3 * j, mf + 6 * j);
    const float reach = mf[6 * j + 5];
    ReachBox m;
    const int how = reach_box_decide(c, mf[6 * j + 3], mf[6 * j + 4], c.mode == 2 ? &reach : nullptr, &m);
    rb_out(m, how, oi + 10 * j, of + 3 * j);
    reach_box_hull_add(&h, j, m);
  }
  const int how = reach_box_hull_close(c, n, &h);
  rb_out(h, how, oi + 10 * n, of + 3 * n);
  return how;
}

// ONE pair shared by K planners (one group, members 0 .. K-1), as run_stochastic_trials issues a step of a batch that
// shares it: the group-aware boxed sampler, then the group-aware state advance.  grid0 / grid1: (M, grid_rows, pitch);
// states: (ngen, 2) in; out0 / out1: (ngen, 2) out; rec: K x 5 member records; grec: 5.
extern "C" int emu_group_box_batch(int K, int8_t* grid0, int8_t* grid1, const int8_t* cum0, const int8_t* cum1,
                                   const uint64_t* states, uint64_t* out0, uint64_t* out1, const int8_t* qv0,
                                   const int8_t* qv1, int bpad, int rows, int cols, int grid_rows, int pitch, int tx,
                                   int ty, int M, int segs, double alpha, int q_cap, const int* ci, const float* cf,
                                   const float* x0, const float* reach, const int* active, int mrows, int ncact, int gm,
                                   int* rec, int* grec) {
  std::vector<uint64_t> T(SAMPLE_TABLE_WORDS);
  if (!build_sample_thresholds(alpha, q_cap, T.data())) return 1;
  int seg_rows;
  std::vector<uint64_t> J;
  emu::segment_jumps(rows, cols, tx, ty, segs, seg_rows, J);
  int64_t kt[4];
  sample_tile_draws(rows, cols, tx, ty, kt);
  std::vector<uint64_t> mats(4 * 256);
  build_jump_matrices(kt, 4, mats.data());
  const size_t ngen = (size_t)tx * ty * M;
  SampleGridsV2Args a{};
  a.t[0] = SampleTdm{grid0, cum0, states, out0, qv0, bpad};
  a.t[1] = SampleTdm{grid1, cum1, states, out1, qv1, bpad};
  a.thresholds = T.data(); a.jump = J.empty() ? nullptr : J.data();
  a.rows = rows; a.cols = cols; a.grid_rows = grid_rows; a.pitch = pitch; a.tx = tx; a.ty = ty; a.num_maps = M;
  a.segs = segs; a.seg_rows = seg_rows;
  sample_box_full(a);
  a.gm = gm; a.write_states = 0;
  std::vector<SampleBoxDesc> bx(K);
  std::vector<float> rs(2 * K);
  std::vector<int> members(K);
  for (int k = 0; k < K; ++k) {
    ReachBoxConst& c = bx[k].c;
    c.mode = ci[3 * k]; c.disc = ci[3 * k + 1]; c.T = ci[3 * k + 2]; c.rows = rows; c.cols = cols; c.nt = 2; c.tx = tx;
    c.ty = ty; c.num_maps = M; c.bpad0 = c.bpad1 = bpad;
    c.vr0 = cf[0]; c.vr1 = cf[1]; c.dt = cf[2]; c.tr_abs_max = cf[3]; c.res = cf[4]; c.pxl = cf[5]; c.pyl = cf[6];
    rs[2 * k] = 999.0f; rs[2 * k + 1] = reach[k];       // slot 1 is this step's
    bx[k].x0 = x0 + 2 * k; bx[k].reach = rs.data() + 2 * k; bx[k].slot = 1; bx[k].record = rec + 5 * k;
    bx[k].jump_tile = mats.data();
    members[k] = k;
  }
  const SampleGroupDesc grp{0, K, grec};
  const int threads = ((ncact * gm + 31) / 32) * 32;
  emu::sampler_nw(bpad, [&](auto NW) {
    emu::launch({(unsigned)(mrows * segs), (unsigned)((M + gm - 1) / gm), 1}, threads, [&] {
      sample_grids_v2_group_box_batch_kernel<decltype(NW)::value>(&a, bx.data(), &grp, members.data(), active, 0, mrows,
                                                                  ncact);
    });
  });
  emu::launch({(unsigned)((ngen + 127) / 128), 1, 1}, 128, [&] {
    advance_states_group_batch_kernel(&a, bx.data(), &grp, members.data(), active, rows, cols, tx, ty, M);
  });
  return 0;
}
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    import __graft_entry__
    __graft_entry__.build_engine()
    return emu_core.build(str(tmp_path_factory.mktemp("hull")), "hull", kernels(None, "sampler_box_batch"), HARNESS,
                          link_engine=True)


def _p(a):
    return C.c_void_p(a.ctypes.data)


# ----------------------------------------------------------------------------- restatement of the hull's rules
def smem(tiy_lo, nact, ty, cols, bpad, gm, nt):
    """sample_v2_smem_hd (csrc/kernels.h)."""
    ncol = -(-cols // ty)
    cfirst = min(tiy_lo * ncol, cols)
    cs1 = min((tiy_lo + nact) * ncol, cols)
    wcols = cs1 - (cfirst & ~15)
    row_bytes_al = (wcols * bpad + 15) & ~15
    stage = max(nt * gm * ((wcols + 15) & ~15), 2 * 128 * 16)
    return nt * row_bytes_al + stage + 256 * 8 + nt * 128


def fits(tiy_lo, nact, ty, cols, bpad0, bpad1, gm, nt):
    """sample_v2_fits_hd (csrc/kernels.h)."""
    return (1 <= gm <= 32 and nact >= 1 and tiy_lo >= 0 and tiy_lo + nact <= ty and (nact * gm + 31) // 32 * 32 <= 256
            and bpad0 <= 32 and smem(tiy_lo, nact, ty, cols, bpad0, gm, nt) <= 200 * 1024 and (nt == 1 or bpad0 == bpad1))


def hull_restated(g, boxes):
    """The contract of a shared pair's box from its members' decisions (ret, geo, how, row_lo, row_hi, col_lo, col_hi,
    tiy_lo, nact, gm) + disc (cx, cy, r): one member as decided; several: the rectangle hull, no disc, how the largest,
    whole maps if any member is whole or the hull's launch does not fit."""
    rows, cols, nt, tx, ty, M, bp0, bp1 = g
    if len(boxes) == 1:
        return boxes[0]
    whole = ([0, 0, 0, 0, rows, 0, cols, 0, ty, 0], [0.0, 0.0, 0.0])
    if any(b[0][2] == 0 for b in boxes):
        return whole
    r_lo, r_hi = min(b[0][3] for b in boxes), max(b[0][4] for b in boxes)
    c_lo, c_hi = min(b[0][5] for b in boxes), max(b[0][6] for b in boxes)
    ncol = -(-cols // ty)
    tiy_lo = c_lo // ncol
    nact = (c_hi - 1) // ncol - tiy_lo + 1
    gm = max(1, min(128 // nact, 32, M))
    if nt == 0 or not fits(tiy_lo, nact, ty, cols, bp0, bp1, gm, nt):
        return whole
    how = max(b[0][2] for b in boxes)
    return [how, 1, how, r_lo, r_hi, c_lo, c_hi, tiy_lo, nact, gm], [0.0, 0.0, 0.0]


def _random_case(rng, wide=False):
    ty = int(rng.choice([1, 3, 4, 8, 16])) if not wide else 300
    cols = int(rng.integers(20, 500)) if not wide else 600
    rows = int(rng.integers(20, 500))
    res = float(rng.choice([0.05, 0.1, 0.2, 1.0]))
    g = np.array([rows, cols, int(rng.choice([0, 1, 2, 2, 2])), int(rng.choice([1, 2, 4, 8])), ty,
                  int(rng.choice([1, 8, 24, 64])), *([int(rng.choice([4, 8, 12, 32]))] * 2)], dtype=np.int32)
    if rng.random() < 0.1:
        g[7] = 36                                                   # unfused pair of unequal bins: never fits at nt 2
    pxl, pyl = float(rng.uniform(-50, 50)), float(rng.uniform(-50, 50))
    gf = np.array([res, pxl, pyl, rng.uniform(0.5, 1.2)], dtype=np.float32)
    n = int(rng.integers(1, 6))
    mi = np.zeros((n, 3), dtype=np.int32)
    mf = np.zeros((n, 6), dtype=np.float32)
    for j in range(n):
        mi[j] = [rng.choice([0, 1, 2, 2, 2, 1]) if rng.random() < 0.95 else 0, rng.integers(0, 2), rng.integers(5, 40)]
        vmax = rng.uniform(0.2, 3.0)
        # a start anywhere on the map, mostly far enough inside for a box; sometimes near an edge or outside it
        fx, fy = (rng.uniform(0.02, 0.98, 2) if rng.random() < 0.3 else rng.uniform(0.25, 0.75, 2))
        if wide:
            fx = [0.03, 0.97][j % 2]
        mf[j] = [-vmax * rng.random(), vmax, rng.uniform(0.01, 0.15), pxl + fx * cols * res, pyl + fy * rows * res,
                 rng.uniform(0, 1.3) * vmax * mi[j, 2] if rng.random() < 0.9 else np.nan]
    return g, gf, mi, mf


def _run(lib, g, gf, mi, mf):
    n = len(mi)
    oi = np.zeros((n + 1, 10), dtype=np.int32)
    of = np.zeros((n + 1, 3), dtype=np.float32)
    ret = lib.emu_hull(n, _p(g), _p(gf), _p(np.ascontiguousarray(mi)), _p(np.ascontiguousarray(mf)), _p(oi), _p(of))
    assert ret == oi[n, 0]
    return [(list(oi[j]), list(of[j])) for j in range(n)], (list(oi[n]), list(of[n]))


def test_hull_matches_its_restatement(lib):
    rng = np.random.default_rng(2024)
    seen = dict(single=0, hull=0, whole_member=0, no_fit=0)
    for case in range(3000):
        g, gf, mi, mf = _random_case(rng, wide=(case % 10 == 9))
        members, hull = _run(lib, g, gf, mi, mf)
        tag = "case %d: g=%s members=%s" % (case, list(g), [m[0] for m in members])
        want = hull_restated(g, members)
        assert hull[0] == list(want[0]) and np.array_equal(np.float32(hull[1]), np.float32(want[1])), tag
        if len(members) == 1:                         # exactly the member's decision, disc included
            assert hull == members[0], tag
            seen["single"] += 1
            continue
        if any(m[0][2] == 0 for m in members):
            assert hull[0][2] == 0 and hull[0][1] == 0, tag
            seen["whole_member"] += 1
        elif hull[0][2] == 0:
            seen["no_fit"] += 1
        else:                                          # the hull contains every member's box, without a disc
            for m in members:
                assert hull[0][3] <= m[0][3] and hull[0][4] >= m[0][4] and hull[0][5] <= m[0][5] \
                    and hull[0][6] >= m[0][6], tag
            assert hull[1] == [0.0, 0.0, 0.0] and hull[0][2] == max(m[0][2] for m in members), tag
            seen["hull"] += 1
    assert min(seen.values()) >= 10, seen                    # every rule is exercised


# ----------------------------------------------------------------------------- the group-aware trial sampler
@pytest.mark.parametrize("running", ["all", "one", "none"])
def test_group_box_batch_against_whole_map_sampling(lib, running):
    rows, cols, tx, ty, M, B, segs, alpha = 61, 70, 4, 6, 5, 12, 3, 0.9       # ragged last tile row and column
    bpad = (B + 3) // 4 * 4
    rng = np.random.default_rng(17)
    pmfs = [random_pmf(rng, B, rows, cols) for _ in range(2)]
    cums = [cumulative_table(p, bpad) for p in pmfs]
    bin_values = np.linspace(0, 1, B)
    bounds = np.array([0.0, 1.0], dtype=np.float32)
    q = np.zeros(128, dtype=np.int8)
    q[:B] = TR.quantise_bin_values(bin_values, bounds)
    q_cap = min(int(min(int(np.cumsum(p.astype(np.int64), axis=0)[-1].min()) for p in pmfs)), 127)
    grid_rows, pitch = rows + 2, (cols + 15) // 16 * 16
    T_, vmax, dt, trm, res = 4, 1.0, 0.5, 1.0, 1.0
    # three planners on the pair: boxed from the reach statistic (with a disc), static, boxed from the reach statistic
    ci = np.array([[2, 1, T_], [1, 0, T_], [2, 1, T_]], dtype=np.int32)
    cf = np.array([-vmax, vmax, dt, trm, res, 0.0, 0.0], dtype=np.float32)
    x0 = np.array([[20.3, 22.7], [35.2, 30.1], [28.0, 40.0]], dtype=np.float32)
    reach = np.array([3.9, 2.1, 1.5], dtype=np.float32)
    active = np.array({"all": [1, 1, 1], "one": [0, 1, 0], "none": [0, 0, 0]}[running], dtype=np.int32)
    K = len(x0)
    u, w, h = 5.9605e-8, cols * res, rows * res               # run_stochastic_trials' launch size (static bound)
    D = (dt * trm * T_ * vmax * 1.0002 + T_ * u * (w + h)) / (1 - T_ * u)
    span = 2 * (D + u * (w + h + 2 * D)) / res + 8
    nrow, ncol = -(-rows // tx), -(-cols // ty)
    mrows, ncact = min(tx, int(span) // nrow + 2), min(ty, int(span) // ncol + 2)
    gm = max(1, min(128 // ncact, 32, M))
    ngen = tx * ty * M
    states = X.create_states(ngen, 41)
    g0 = np.full((M, grid_rows, pitch), -7, np.int8)
    g1 = np.full((M, grid_rows, pitch), -7, np.int8)
    o0, o1 = np.full((ngen, 2), 5, np.uint64), np.full((ngen, 2), 6, np.uint64)
    rec, grec = np.full((K, 5), -9, dtype=np.int32), np.full(5, -9, dtype=np.int32)
    assert lib.emu_group_box_batch(K, _p(g0), _p(g1), _p(cums[0]), _p(cums[1]), _p(states), _p(o0), _p(o1), _p(q),
                                   _p(q), bpad, rows, cols, grid_rows, pitch, tx, ty, M, segs, C.c_double(alpha), q_cap,
                                   _p(ci), _p(cf), _p(x0), _p(reach), _p(active), mrows, ncact, gm, _p(rec),
                                   _p(grec)) == 0
    if running == "none":                                     # no member runs: nothing written
        assert (g0 == -7).all() and (g1 == -7).all() and (o0 == 5).all() and (o1 == 6).all()
        assert (rec == -9).all() and (grec == -9).all()
        return
    g = np.array([rows, cols, 2, tx, ty, M, bpad, bpad], dtype=np.int32)
    gf = np.array([res, 0.0, 0.0, trm], dtype=np.float32)
    on = np.flatnonzero(active)
    mf = np.array([[-vmax, vmax, dt, x0[k, 0], x0[k, 1], reach[k]] for k in on], dtype=np.float32)
    members, hull = _run(lib, g, gf, ci[on], mf)
    how, r_lo, r_hi, c_lo, c_hi = hull[0][2], hull[0][3], hull[0][4], hull[0][5], hull[0][6]
    assert how != 0, "the case is meant to sample a box"
    if running == "one":
        assert hull == members[0]                             # the member's own decision (static box, no disc here)
    else:
        assert hull[1] == [0.0, 0.0, 0.0] and how == 2
        for m in members:
            assert r_lo <= m[0][3] and m[0][4] <= r_hi and c_lo <= m[0][5] and m[0][6] <= c_hi
    want_rec = [how, r_lo, r_hi, c_lo, c_hi]
    assert list(grec) == want_rec
    for k in range(K):
        assert list(rec[k]) == (want_rec if active[k] else [-9] * 5), "planner %d: record" % k
    for k, (grid, out) in enumerate(((g0, o0), (g1, o1))):
        want = np.full((M, grid_rows, pitch), -7, dtype=np.int8)
        st = states.copy()
        TR.sample_grids(want, pmfs[k], st, bin_values, bounds, alpha, (tx, ty), M)
        assert np.array_equal(grid[:, r_lo:r_hi, c_lo:c_hi], want[:, r_lo:r_hi, c_lo:c_hi]), "TDM %d: the hull" % k
        assert ((grid == want) | (grid == -7)).all(), "TDM %d: a cell outside whole-map sampling" % k
        assert np.array_equal(out, st), "TDM %d: generator states" % k
