"""The batched trial samplers over pairs whose maps differ in size (one launch class: the same bins, thread tile and
number of maps; rows, cols, pitch and row segments per pair), executed on the host from their REAL source
(csrc/sample.cu: sample_grids_v2_batch_kernel, sample_grids_v2_box_batch_kernel, sample_grids_v2_complete_batch_kernel,
advance_states_batch_kernel and their group variants).  One emulated launch, sized for the class's largest pair as
run_trials / run_stochastic_trials size it, holds three pairs: one larger than another in its columns only, one smaller
in both dimensions, with different row segmentations; the launch's class list names them in reverse order and leaves
out a fourth pair.
Each listed pair's maps and generator states equal the oracle's sampling of that pair alone (oracle/terrain_ref.py
sample_grids): inside its box for a boxed step, whole maps after the completion launch or for a box that leaves the map
(or for the whole-map sampler); the box record is the host's decision; the unlisted pair is left untouched byte for
byte."""
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
// P fused pairs of one class (bpad, tx, ty, M shared); pair p: geo[5p..] = rows, cols, grid_rows, pitch, segs (clamped
// as tdm_prepare_jump clamps it), its own cumulative tables, grids, generator states (in: st, out: o0 / o1), x0, reach
// and record.  The launches cover the n pairs pairs[0 .. n) (entry z samples pair pairs[z]), sized for the largest as
// the trial host code sizes them.  grouped: the group variants, each pair a group of one planner.
// mode 0: the whole-map sampler (one-map trials); 1: the boxed sampler and the state advance (stochastic trials), then,
// with map_end > 0, the completion of maps [0, map_end).
struct Pairs {
  std::vector<SampleGridsV2Args> d;
  std::vector<SampleBoxDesc> bx;
  std::vector<SampleGroupDesc> grp;
  std::vector<int> members;
  std::vector<std::vector<uint64_t>> J, mats;
  std::vector<uint64_t> T;
  std::vector<float> rs;
};

static int setup(Pairs& s, int P, const int* geo, int8_t* const* g0, int8_t* const* g1, const int8_t* const* c0,
                 const int8_t* const* c1, const uint64_t* const* st, uint64_t* const* o0, uint64_t* const* o1,
                 const int8_t* qv0, const int8_t* qv1, int bpad, int tx, int ty, int M, double alpha, int q_cap,
                 const int* ci, const float* cf, const float* x0, const float* reach, int* rec, int* grec) {
  s.T.resize(SAMPLE_TABLE_WORDS);
  if (!build_sample_thresholds(alpha, q_cap, s.T.data())) return 1;
  s.d.resize(P); s.bx.resize(P); s.grp.resize(P); s.members.resize(P); s.J.resize(P); s.mats.resize(P);
  s.rs.resize(2 * P);
  for (int p = 0; p < P; ++p) {
    const int rows = geo[5 * p], cols = geo[5 * p + 1];
    int segs = geo[5 * p + 4], seg_rows;
    emu::segment_jumps(rows, cols, tx, ty, segs, seg_rows, s.J[p]);
    int64_t kt[4];
    sample_tile_draws(rows, cols, tx, ty, kt);
    s.mats[p].resize(4 * 256);
    build_jump_matrices(kt, 4, s.mats[p].data());
    SampleGridsV2Args& a = s.d[p];
    a = SampleGridsV2Args{};
    a.t[0] = SampleTdm{g0[p], c0[p], st[p], o0[p], qv0, bpad};
    a.t[1] = SampleTdm{g1[p], c1[p], st[p], o1[p], qv1, bpad};
    a.thresholds = s.T.data(); a.jump = s.J[p].empty() ? nullptr : s.J[p].data();
    a.rows = rows; a.cols = cols; a.grid_rows = geo[5 * p + 2]; a.pitch = geo[5 * p + 3]; a.tx = tx; a.ty = ty;
    a.num_maps = M; a.segs = segs; a.seg_rows = seg_rows;
    sample_box_full(a);
    if (a.ty * a.gm > 256) a.gm = 256 / a.ty;                                   // fill_v2 (api.cu)
    ReachBoxConst& c = s.bx[p].c;
    c.mode = ci[3 * p]; c.disc = ci[3 * p + 1]; c.T = ci[3 * p + 2]; c.rows = rows; c.cols = cols; c.nt = 2; c.tx = tx;
    c.ty = ty; c.num_maps = M; c.bpad0 = c.bpad1 = bpad;
    c.vr0 = cf[0]; c.vr1 = cf[1]; c.dt = cf[2]; c.tr_abs_max = cf[3]; c.res = cf[4]; c.pxl = cf[5]; c.pyl = cf[6];
    s.rs[2 * p] = 999.0f; s.rs[2 * p + 1] = reach[p];                           // slot 1 is this step's
    s.bx[p].x0 = x0 + 2 * p; s.bx[p].reach = s.rs.data() + 2 * p; s.bx[p].slot = 1; s.bx[p].record = rec + 5 * p;
    s.bx[p].jump_tile = s.mats[p].data();
    s.grp[p] = SampleGroupDesc{p, 1, grec + 5 * p};
    s.members[p] = p;
  }
  return 0;
}

extern "C" int emu_class_batch(int P, int mode, int grouped, const int* geo, int8_t* const* g0, int8_t* const* g1,
                               const int8_t* const* c0, const int8_t* const* c1, const uint64_t* const* st,
                               uint64_t* const* o0, uint64_t* const* o1, const int8_t* qv0, const int8_t* qv1, int bpad,
                               int tx, int ty, int M, double alpha, int q_cap, const int* ci, const float* cf,
                               const float* x0, const float* reach, const int* pairs, int n, int mrows, int ncact,
                               int gm, int map_end, int* rec, int* grec) {
  Pairs s;
  int rc = setup(s, P, geo, g0, g1, c0, c1, st, o0, o1, qv0, qv1, bpad, tx, ty, M, alpha, q_cap, ci, cf, x0, reach, rec,
                 grec);
  if (rc) return rc;
  std::vector<int> active(P, 1);
  const SampleGridsV2Args* d = s.d.data();
  if (mode == 0) {                                      // onemap_trial_plans + launch_sample_grids_v2_batch
    std::vector<const SampleGridsV2Args*> mem;
    for (int z = 0; z < n; ++z) mem.push_back(&s.d[pairs[z]]);
    const SampleClassLaunch L = sample_class_launch(mem.data(), n);
    emu::sampler_nw(bpad, [&](auto NW) {
      emu::launch({(unsigned)L.gx, (unsigned)L.gy, (unsigned)n}, L.threads, [&] {
        if (grouped)
          sample_grids_v2_group_batch_kernel<2, decltype(NW)::value>(d, s.grp.data(), s.members.data(), active.data(),
                                                                     pairs);
        else
          sample_grids_v2_batch_kernel<2, decltype(NW)::value>(d, active.data(), pairs);
      });
    });
    return 0;
  }
  // stochastic_trial_plans: the boxed launch's maps per CTA over every pair; the launch sized for the largest
  std::vector<const SampleGridsV2Args*> mem;
  for (int p = 0; p < P; ++p) {
    s.d[p].gm = gm; s.d[p].write_states = 0;
    if (!sample_box_batch_fits(s.d[p], ncact)) return 4;
  }
  for (int z = 0; z < n; ++z) mem.push_back(&s.d[pairs[z]]);
  const SampleClassLaunch L = sample_box_class_launch(mem.data(), n, mrows, ncact);
  const SampleBoxDesc* bx = s.bx.data();
  emu::sampler_nw(bpad, [&](auto NW) {
    emu::launch({(unsigned)L.gx, (unsigned)L.gy, (unsigned)n}, L.threads, [&] {
      if (grouped)
        sample_grids_v2_group_box_batch_kernel<decltype(NW)::value>(d, s.bx.data(), s.grp.data(), s.members.data(),
                                                                    active.data(), 0, mrows, ncact, pairs);
      else
        sample_grids_v2_box_batch_kernel<decltype(NW)::value>(d, bx, active.data(), 0, mrows, ncact, pairs);
    });
  });
  const int64_t ngen = (int64_t)tx * ty * M;
  emu::launch({(unsigned)((ngen + 127) / 128), (unsigned)n, 1}, 128, [&] {
    if (grouped)
      advance_states_group_batch_kernel(d, bx, s.grp.data(), s.members.data(), active.data(), 0, 0, tx, ty, M, pairs);
    else
      advance_states_batch_kernel(d, bx, active.data(), 0, 0, tx, ty, M, pairs);
  });
  if (map_end > 0) {
    emu::sampler_nw(bpad, [&](auto NW) {
      emu::launch({(unsigned)L.gx, (unsigned)((map_end + L.gm - 1) / L.gm), (unsigned)n}, L.threads, [&] {
        if (grouped)
          sample_grids_v2_group_complete_batch_kernel<decltype(NW)::value>(d, s.grp.data(), s.members.data(),
                                                                           active.data(), map_end, mrows, ncact, pairs);
        else
          sample_grids_v2_complete_batch_kernel<decltype(NW)::value>(d, bx, active.data(), map_end, mrows, ncact,
                                                                     pairs);
      });
    });
  }
  return 0;
}

// reach_box_decide for one pair (the host's sample_finish): out = how, row_lo, row_hi, col_lo, col_hi
extern "C" int emu_decide(const int* ci, const float* cf, int rows, int cols, int tx, int ty, int M, int bpad, float x,
                          float y, float reach, int* out) {
  ReachBoxConst c{};
  c.mode = ci[0]; c.disc = ci[1]; c.T = ci[2]; c.rows = rows; c.cols = cols; c.nt = 2; c.tx = tx; c.ty = ty;
  c.num_maps = M; c.bpad0 = c.bpad1 = bpad;
  c.vr0 = cf[0]; c.vr1 = cf[1]; c.dt = cf[2]; c.tr_abs_max = cf[3]; c.res = cf[4]; c.pxl = cf[5]; c.pyl = cf[6];
  ReachBox b;
  const int how = reach_box_decide(c, x, y, c.mode == 2 ? &reach : nullptr, &b);
  out[0] = how; out[1] = how ? b.row_lo : 0; out[2] = how ? b.row_hi : rows; out[3] = how ? b.col_lo : 0;
  out[4] = how ? b.col_hi : cols;
  return how;
}
'''


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    import __graft_entry__
    __graft_entry__.build_engine()
    return emu_core.build(str(tmp_path_factory.mktemp("classbatch")), "classbatch",
                          kernels(None, "sampler_batch", "sampler_box_batch"), HARNESS, link_engine=True)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _pp(arrs):
    return (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])


TX, TY, M, B, ALPHA, FILL = 4, 6, 5, 12, 0.9, -7
BPAD = (B + 3) // 4 * 4
# rows, cols, requested row segments: pair 1 is pair 0 widened (columns only), pair 2 is smaller in both dimensions;
# pair 3 is not in the launch
GEO = [(61, 70, 3), (61, 100, 2), (37, 45, 1), (50, 50, 2)]
PAIRS = [2, 1, 0]
# starts (cells, res 1 m): boxes inside the map for pairs 0 and 1, a box leaving pair 2's map (whole maps)
X0 = [(30.3, 22.7), (80.2, 40.1), (1.5, 20.0), (25.0, 25.0)]
REACH = [3.9, 2.1, 1.0, 2.0]
T_, VMAX, DT, TRM, RES = 4, 1.0, 0.5, 1.0, 1.0


def _class_launch_size(geo):
    """stochastic_trial_plans (api.cu): per pair min(tx, span / nrow + 2) tile rows and min(ty, span / ncol + 2) tile
    columns of the static bound's span, the class's the largest; maps per CTA for that many tile columns."""
    mrows = ncact = 0
    for rows, cols, _ in (geo[p] for p in PAIRS):
        u, w, h = 5.9605e-8, cols * RES, rows * RES
        D = (DT * TRM * T_ * VMAX * 1.0002 + T_ * u * (w + h)) / (1 - T_ * u)
        span = 2 * (D + u * (w + h + 2 * D)) / RES + 8
        nrow, ncol = -(-rows // TX), -(-cols // TY)
        mrows, ncact = max(mrows, min(TX, int(span) // nrow + 2)), max(ncact, min(TY, int(span) // ncol + 2))
    return mrows, ncact, max(1, min(128 // ncact, 32, M))


@pytest.mark.parametrize("grouped", [False, True], ids=["plain", "group"])
@pytest.mark.parametrize("step", ["whole_map", "box", "box_completed"])
def test_class_launch_equals_each_pair_alone(lib, grouped, step):
    rng = np.random.default_rng(31)
    P = len(GEO)
    pmfs = [[random_pmf(rng, B, r, c) for _ in range(2)] for r, c, _ in GEO]
    cums = [[cumulative_table(p, BPAD) for p in pp] for pp in pmfs]
    bin_values = np.linspace(0, 1, B)
    bounds = np.array([0.0, 1.0], dtype=np.float32)
    q = np.zeros(128, dtype=np.int8)
    q[:B] = TR.quantise_bin_values(bin_values, bounds)
    q_cap = min(min(int(np.cumsum(p.astype(np.int64), axis=0)[-1].min()) for pp in pmfs for p in pp), 127)
    geo = np.array([[r, c, r + 2, (c + 15) // 16 * 16, s] for r, c, s in GEO], dtype=np.int32)
    ngen = TX * TY * M
    states = [X.create_states(ngen, 50 + p) for p in range(P)]
    grids = [[np.full((M, g[2], g[3]), FILL, np.int8) for _ in range(2)] for g in geo]
    outs = [[np.full((ngen, 2), 5 + k, np.uint64) for k in range(2)] for _ in range(P)]
    ci = np.array([[2, 0, T_]] * P, dtype=np.int32)                  # boxes from the reach statistic, no disc
    cf = np.array([-VMAX, VMAX, DT, TRM, RES, 0.0, 0.0], dtype=np.float32)
    x0 = np.array(X0, dtype=np.float32)
    reach = np.array(REACH, dtype=np.float32)
    rec, grec = np.full((P, 5), -9, np.int32), np.full((P, 5), -9, np.int32)
    pairs = np.array(PAIRS, dtype=np.int32)
    mrows, ncact, gm = _class_launch_size(GEO)
    mode = 0 if step == "whole_map" else 1
    map_end = M if step == "box_completed" else 0
    assert lib.emu_class_batch(P, mode, int(grouped), _p(geo), _pp([g[0] for g in grids]), _pp([g[1] for g in grids]),
                               _pp([c[0] for c in cums]), _pp([c[1] for c in cums]), _pp(states),
                               _pp([o[0] for o in outs]), _pp([o[1] for o in outs]), _p(q), _p(q), BPAD, TX, TY, M,
                               C.c_double(ALPHA), q_cap, _p(ci), _p(cf), _p(x0), _p(reach), _p(pairs), len(pairs),
                               mrows, ncact, gm, map_end, _p(rec), _p(grec)) == 0
    hows = {}
    for p in range(P):
        rows, cols = GEO[p][:2]
        if p not in pairs:                                            # untouched, byte for byte
            assert all((g == FILL).all() for g in grids[p]), "pair %d: maps" % p
            assert (outs[p][0] == 5).all() and (outs[p][1] == 6).all() and (rec[p] == -9).all() and (grec[p] == -9).all()
            continue
        want, after = [], []
        for k in range(2):                                            # the oracle's whole-map sampling of the pair alone
            want.append(np.full(grids[p][k].shape, FILL, np.int8))
            after.append(states[p].copy())
            TR.sample_grids(want[k], pmfs[p][k], after[k], bin_values, bounds, ALPHA, (TX, TY), M)
        st = after[0]
        assert np.array_equal(after[1], st)                           # one stream samples both TDMs
        for k in range(2):
            assert np.array_equal(outs[p][k], st), "pair %d TDM %d: generator states" % (p, k)
        if mode == 0:
            for k in range(2):
                assert np.array_equal(grids[p][k], want[k]), "pair %d TDM %d: whole maps" % (p, k)
            continue
        out = (C.c_int * 5)()
        how = lib.emu_decide(_p(ci[p]), _p(cf), rows, cols, TX, TY, M, BPAD, float(x0[p, 0]), float(x0[p, 1]),
                             float(reach[p]), out)
        hows[p] = how
        assert list(rec[p]) == list(out), "pair %d: record" % p
        if grouped:
            assert list(grec[p]) == list(out), "pair %d: group record" % p
        r_lo, r_hi, c_lo, c_hi = out[1], out[2], out[3], out[4]
        for k in range(2):
            g = grids[p][k]
            if how == 0 or map_end:                                   # whole maps, padding untouched
                assert np.array_equal(g, want[k]), "pair %d TDM %d (how %d): whole maps" % (p, k, how)
            else:
                assert np.array_equal(g[:, r_lo:r_hi, c_lo:c_hi], want[k][:, r_lo:r_hi, c_lo:c_hi]), \
                    "pair %d TDM %d: the box" % (p, k)
                assert ((g == want[k]) | (g == FILL)).all(), "pair %d TDM %d: a cell outside the sampling" % (p, k)
    if mode == 1:
        assert hows == {0: 2, 1: 2, 2: 0}, hows                             # a box, and one leaving the map
