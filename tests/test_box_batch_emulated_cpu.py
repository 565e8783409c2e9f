"""The batched boxed sampler of stochastic trials (sample_grids_v2_box_batch_kernel + advance_states_batch_kernel,
csrc/sample.cu), executed on the host from its REAL source, against per-pair boxed launches as solve() issues them
(tests/emu_sampler.py's emu_sample_v2 with the box and disc of reach_box_decide, or whole maps): the sampled maps and
every generator state bit for bit, the decision record, boxes at different positions in one launch, whole-map
fallbacks (map edge, reach beyond the speed limit, box off), ragged last tile rows and columns, the group loop of a box
larger than the launch, and a gated pair left untouched byte for byte."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import terrain_ref as TR
from oracle import xoroshiro as X
from tests.emu_sampler import CSRC, PRELUDE, ROOT, _region, build, cumulative_table
from tests.scenarios import random_pmf

HARNESS = r'''
bool build_sample_thresholds(double alpha, int q_cap, uint64_t* table);
void sample_tile_draws(int rows, int cols, int tx, int ty, int64_t ks[4]);
}  // namespace b200

// K fused pairs of one geometry (shared cum / qvals / thresholds; own maps, states, x0 and reach): ONE batched boxed
// launch (iteration 0: reach slot `slot`) and ONE batched advance, as run_stochastic_trials issues them.
// grid0 / grid1: K x (M, grid_rows, pitch); states: K x (ngen, 2) in; out0 / out1: K x (ngen, 2) out; rec: K x 5.
extern "C" int emu_box_batch(int K, int8_t* grid0, int8_t* grid1, const int8_t* cum0, const int8_t* cum1,
                             const uint64_t* states, uint64_t* out0, uint64_t* out1, const int8_t* qv0, const int8_t* qv1,
                             int bpad, int rows, int cols, int grid_rows, int pitch, int tx, int ty, int M, int segs,
                             double alpha, int q_cap, const int* ci, const float* cf, const float* x0, const float* reach,
                             const int* active, int mrows, int ncact, int gm, int* rec) {
  using namespace b200;
  std::vector<uint64_t> T(SAMPLE_TABLE_WORDS);
  if (!build_sample_thresholds(alpha, q_cap, T.data())) return 1;
  const int nrow = (rows + tx - 1) / tx, ncol = (cols + ty - 1) / ty;
  if (segs > nrow) segs = nrow;
  const int seg_rows = (nrow + segs - 1) / segs;
  std::vector<uint64_t> J;                          // tdm_prepare_jump's segment jumps
  if (segs > 1) {
    int last_w = cols - (ty - 1) * ncol;
    for (int iy = ty - 1; iy >= 0 && last_w <= 0; --iy) last_w = cols - iy * ncol;
    if (last_w > ncol) last_w = ncol;
    std::vector<int64_t> ks;
    for (int s = 1; s < segs; ++s) { ks.push_back((int64_t)s * seg_rows * ncol); ks.push_back((int64_t)s * seg_rows * last_w); }
    J.resize(ks.size() * 256);
    build_jump_matrices(ks.data(), (int)ks.size(), J.data());
  }
  int64_t kt[4];
  sample_tile_draws(rows, cols, tx, ty, kt);
  std::vector<uint64_t> mats(4 * 256);
  build_jump_matrices(kt, 4, mats.data());
  const size_t ngen = (size_t)tx * ty * M, gsz = (size_t)M * grid_rows * pitch;
  std::vector<SampleGridsV2Args> d(K);
  std::vector<SampleBoxDesc> bx(K);
  std::vector<float> rs(2 * K);
  for (int k = 0; k < K; ++k) {
    SampleGridsV2Args& a = d[k];
    a = SampleGridsV2Args{};
    a.t[0] = SampleTdm{grid0 + k * gsz, cum0, states + k * ngen * 2, out0 + k * ngen * 2, qv0, bpad};
    a.t[1] = SampleTdm{grid1 + k * gsz, cum1, states + k * ngen * 2, out1 + k * ngen * 2, qv1, bpad};
    a.thresholds = T.data(); a.jump = J.empty() ? nullptr : J.data();
    a.rows = rows; a.cols = cols; a.grid_rows = grid_rows; a.pitch = pitch; a.tx = tx; a.ty = ty; a.num_maps = M;
    a.segs = segs; a.seg_rows = seg_rows;
    sample_box_full(a);
    a.gm = gm; a.write_states = 0;
    ReachBoxConst& c = bx[k].c;
    c.mode = ci[0]; c.disc = ci[1]; c.T = ci[2]; c.rows = rows; c.cols = cols; c.nt = 2; c.tx = tx; c.ty = ty;
    c.num_maps = M; c.bpad0 = c.bpad1 = bpad;
    c.vr0 = cf[0]; c.vr1 = cf[1]; c.dt = cf[2]; c.tr_abs_max = cf[3]; c.res = cf[4]; c.pxl = cf[5]; c.pyl = cf[6];
    rs[2 * k] = 999.0f; rs[2 * k + 1] = reach[k];       // slot 1 is this step's
    bx[k].x0 = x0 + 2 * k; bx[k].reach = rs.data() + 2 * k; bx[k].slot = 1; bx[k].record = rec + 5 * k;
    bx[k].jump_tile = mats.data();
  }
  const int threads = ((ncact * gm + 31) / 32) * 32;
  const unsigned gx = (unsigned)(mrows * segs), gy = (unsigned)((M + gm - 1) / gm);
  for (unsigned z = 0; z < (unsigned)K; ++z)
    for (unsigned by = 0; by < gy; ++by)
      for (unsigned bxi = 0; bxi < gx; ++bxi) {
        std::barrier<> bar(threads);
        g_bar = &bar;
        std::vector<std::thread> th;
        for (int t = 0; t < threads; ++t)
          th.emplace_back([&, t] {
            threadIdx = {(unsigned)t, 0, 0}; blockIdx = {bxi, by, z}; blockDim = {(unsigned)threads, 1, 1};
            gridDim = {gx, gy, (unsigned)K};
            const int nw = bpad / 4;
            if (nw == 3) sample_grids_v2_box_batch_kernel<3>(d.data(), bx.data(), active, 0, mrows, ncact);
            else if (nw == 1) sample_grids_v2_box_batch_kernel<1>(d.data(), bx.data(), active, 0, mrows, ncact);
            else if (nw == 8) sample_grids_v2_box_batch_kernel<8>(d.data(), bx.data(), active, 0, mrows, ncact);
            else sample_grids_v2_box_batch_kernel<0>(d.data(), bx.data(), active, 0, mrows, ncact);
          });
        for (auto& x : th) x.join();
      }
  const unsigned nblk = (unsigned)((ngen + 127) / 128);
  for (unsigned y = 0; y < (unsigned)K; ++y)
    for (unsigned bxi = 0; bxi < nblk; ++bxi) {
      std::barrier<> bar(128);
      g_bar = &bar;
      std::vector<std::thread> th;
      for (int t = 0; t < 128; ++t)
        th.emplace_back([&, t] {
          threadIdx = {(unsigned)t, 0, 0}; blockIdx = {bxi, y, 0}; blockDim = {128, 1, 1}; gridDim = {nblk, (unsigned)K, 1};
          advance_states_batch_kernel(d.data(), bx.data(), active, rows, cols, tx, ty, M);
        });
      for (auto& x : th) x.join();
    }
  return 0;
}

// reach_box_decide for one pair (what the host's sample_finish decides): out = how, row_lo, row_hi, col_lo, col_hi;
// disc = cx, cy, r
extern "C" int emu_decide(const int* ci, const float* cf, int rows, int cols, int tx, int ty, int M, int bpad, float x,
                          float y, float reach, int* out, float* disc) {
  using namespace b200;
  ReachBoxConst c{};
  c.mode = ci[0]; c.disc = ci[1]; c.T = ci[2]; c.rows = rows; c.cols = cols; c.nt = 2; c.tx = tx; c.ty = ty;
  c.num_maps = M; c.bpad0 = c.bpad1 = bpad;
  c.vr0 = cf[0]; c.vr1 = cf[1]; c.dt = cf[2]; c.tr_abs_max = cf[3]; c.res = cf[4]; c.pxl = cf[5]; c.pyl = cf[6];
  ReachBox b;
  const int how = reach_box_decide(c, x, y, c.mode == 2 ? &reach : nullptr, &b);
  out[0] = how; out[1] = how ? b.row_lo : 0; out[2] = how ? b.row_hi : rows; out[3] = how ? b.col_lo : 0;
  out[4] = how ? b.col_hi : cols;
  disc[0] = b.cx; disc[1] = b.cy; disc[2] = b.r;
  return how;
}
'''


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    import __graft_entry__
    __graft_entry__.build_engine()
    d = tmp_path_factory.mktemp("boxbatch")
    kh, sc = os.path.join(CSRC, "kernels.h"), os.path.join(CSRC, "sample.cu")
    src = (PRELUDE + _region(kh, "sampler_args") + _region(kh, "box_desc") + _region(os.path.join(CSRC, "common.cuh"), "xoro") +
           _region(os.path.join(CSRC, "common.cuh"), "threshold") + _region(sc, "sampler_v2") +
           _region(sc, "sampler_box_batch") + HARNESS)
    cpp, so = d / "boxbatch.cpp", d / "libboxbatch.so"
    cpp.write_text(src)
    libdir = os.path.join(ROOT, "mppi_numba_b200")
    r = subprocess.run(["g++", "-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-Wno-unknown-pragmas",
                        "-ffp-contract=off", str(cpp), "-o", str(so), "-L" + libdir, "-l:libb200mppi.so",
                        "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    lib = C.CDLL(str(so))
    lib.emu_box_batch.restype = C.c_int
    lib.emu_decide.restype = C.c_int
    lib.emu_decide.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 6 + [C.c_float] * 3 + [C.c_void_p, C.c_void_p]
    return lib, build(str(d))


def _p(a):
    return C.c_void_p(a.ctypes.data)


@pytest.mark.parametrize("case", ["mixed", "disc_off", "box_off", "wide_box"])
def test_box_batch_equals_per_pair_boxed_launches(libs, case):
    lib, single = libs
    rows, cols, tx, ty, M, B, segs, alpha = 61, 70, 4, 6, 5, 12, 3, 0.9       # ragged last tile row and column
    bpad = (B + 3) // 4 * 4
    rng = np.random.default_rng(11)
    pmfs = [random_pmf(rng, B, rows, cols) for _ in range(2)]
    cums = [cumulative_table(p, bpad) for p in pmfs]
    q = np.zeros(128, dtype=np.int8)
    q[:B] = TR.quantise_bin_values(np.linspace(0, 1, B), np.array([0.0, 1.0], dtype=np.float32))
    q_cap = min(int(min(int(np.cumsum(p.astype(np.int64), axis=0)[-1].min()) for p in pmfs)), 127)
    grid_rows, pitch = rows + 2, (cols + 15) // 16 * 16
    T_, vmax, dt, trm, res = (4, 1.0, 0.5, 1.0, 1.0) if case != "wide_box" else (4, 1.0, 2.0, 1.0, 1.0)
    ci = np.array([0 if case == "box_off" else 2, 0 if case == "disc_off" else 1, T_], dtype=np.int32)
    cf = np.array([-vmax, vmax, dt, trm, res, 0.0, 0.0], dtype=np.float32)
    # x0: boxes at different positions, the map's edge, a reach beyond the speed limit (whole maps), a gated pair
    x0 = np.array([[10.3, 12.7], [55.2, 40.1], [1.5, 30.0], [33.0, 33.0], [20.0, 45.0], [40.4, 9.9]], dtype=np.float32)
    reach = np.array([3.9, 2.1, 1.0, 100.0, 0.0, 4.0], dtype=np.float32)
    active = np.array([1, 1, 1, 1, 1, 0], dtype=np.int32)
    K = len(x0)
    span = 2 * dt * trm * T_ * vmax * 1.0002 / res + 8
    nrow, ncol = -(-rows // tx), -(-cols // ty)
    mrows, ncact = min(tx, int(span) // nrow + 2), min(ty, int(span) // ncol + 2)
    if case == "wide_box":                     # a launch narrower than the box: the group loop covers it
        mrows, ncact = 1, 1
    gm = max(1, min(128 // ncact, 32, M))
    ngen = tx * ty * M
    states = np.stack([X.create_states(ngen, 40 + k) for k in range(K)])
    g0 = rng.integers(-100, 100, (K, M, grid_rows, pitch)).astype(np.int8)
    g1 = rng.integers(-100, 100, (K, M, grid_rows, pitch)).astype(np.int8)
    o0, o1 = np.full((K, ngen, 2), 5, np.uint64), np.full((K, ngen, 2), 6, np.uint64)
    rec = np.full((K, 5), -9, dtype=np.int32)
    before = [a.copy() for a in (g0, g1, o0, o1)]
    assert lib.emu_box_batch(K, _p(g0), _p(g1), _p(cums[0]), _p(cums[1]), _p(states), _p(o0), _p(o1), _p(q), _p(q), bpad,
                             rows, cols, grid_rows, pitch, tx, ty, M, segs, C.c_double(alpha), q_cap, _p(ci), _p(cf),
                             _p(x0), _p(reach), _p(active), mrows, ncact, gm, _p(rec)) == 0
    hows = []
    for k in range(K):
        if not active[k]:                       # gated: nothing written
            for a, b in zip((g0, g1, o0, o1), before):
                assert np.array_equal(a[k], b[k])
            assert (rec[k] == -9).all()
            continue
        out, disc = (C.c_int * 5)(), (C.c_float * 3)()
        how = lib.emu_decide(_p(ci), _p(cf), rows, cols, tx, ty, M, bpad, float(x0[k, 0]), float(x0[k, 1]),
                             float(reach[k]), out, disc)
        hows.append(how)
        assert list(rec[k]) == list(out), "pair %d: record" % k
        w0, w1 = before[0][k].copy(), before[1][k].copy()
        st_out = np.zeros((ngen, 2), np.uint64)
        box = (C.c_int * 4)(out[1], out[2], out[3], out[4]) if how else None
        rc = single.emu_sample_v2(2, _p(w0), _p(w1), _p(cums[0]), _p(cums[1]), _p(np.ascontiguousarray(states[k])),
                                  _p(st_out), _p(q), _p(q), bpad, rows, cols, grid_rows, pitch, tx, ty, M, segs,
                                  float(alpha), q_cap, box, disc if (how and ci[1]) else None)
        assert rc == 0
        assert np.array_equal(g0[k], w0) and np.array_equal(g1[k], w1), "pair %d (how %d): maps" % (k, how)
        assert np.array_equal(o0[k], st_out) and np.array_equal(o1[k], st_out), "pair %d: states" % k
    if case == "box_off":
        assert hows == [0] * 5
    else:
        assert hows.count(0) >= 2 and hows.count(2) >= 2, hows     # edge + over-limit reach whole, the others boxed
