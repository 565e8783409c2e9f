"""The batched visualisation rollouts and the map completion of recording stochastic trials, executed on the host from
their REAL source (tests/emu_vis_batch.py): state_rollout_batch_kernel against one state_rollout_kernel launch per
planner, byte for byte, for every mode; a planner gated out by ``active`` left untouched; records landing in their
(planner, record) slot.  sample_grids_v2_complete_batch_kernel against the whole-map sampler for maps [0, V): maps >= V,
every generator state and the pairs whose step sampled whole maps (or that are gated out) left untouched."""
import ctypes as C

import numpy as np
import pytest

from oracle import terrain_ref as TR
from oracle import xoroshiro as X
from tests import emu_vis_batch
from tests.emu_sampler import cumulative_table
from tests.scenarios import random_pmf

F32 = np.float32


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_vis_batch.build(str(tmp_path_factory.mktemp("visbatch")))


@pytest.fixture(scope="module")
def emu_complete(tmp_path_factory):
    import __graft_entry__
    __graft_entry__.build_engine()
    return emu_vis_batch.build_complete(str(tmp_path_factory.mktemp("complete")))


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _ptrs(arrays):
    return (C.c_void_p * len(arrays))(*[a.ctypes.data for a in arrays])


class Planners:
    """K planners of one mode with their own params, maps (M = V for mode 0, else 1), noise, u_cur and u_prev."""

    def __init__(self, mode, K, V=37, T=12, N=40, R=14, Cc=18, seed=5):
        rng = np.random.default_rng(seed + 10 * mode)
        self.mode, self.K, self.V, self.T = mode, K, V, T
        M = V + 2 if mode == 0 else 1
        pitch = (Cc + 15) // 16 * 16
        self.f, self.g, self.ratios = [], [], []
        self.lin, self.ang, self.noise, self.u_cur, self.u_prev = [], [], [], [], []
        for k in range(K):
            res, xlo, ylo = 0.5 + 0.1 * k, -1.0 - 0.2 * k, -0.5
            x0 = [xlo + 2.0 + 0.3 * k, ylo + 2.5, 0.2 * k - 0.3]
            lin_lo, ang_lo = 0.1 * k, -0.2
            self.f.append([res, xlo, ylo, 0.1 + 0.02 * k, *x0, 3.0, 2.0, 0.3, 0.01, 1.0, 1.0, 1.5, 0.0, 2.0 + 0.5 * k,
                           -np.pi, np.pi, 1e3, 10.0, 1.0, lin_lo, ang_lo])
            self.g.append([R, Cc, R, Cc, pitch, Cc, T, N, M])
            self.ratios.append([0.01 * np.float64(F32(F32(1.0) - F32(lin_lo))), 0.01 * np.float64(F32(F32(1.2) - F32(ang_lo)))])
            self.lin.append(rng.integers(0, 101, (M, R, pitch)).astype(np.int8))
            self.ang.append(rng.integers(0, 101, (M, R, pitch)).astype(np.int8))
            self.noise.append(rng.normal(0.0, 1.5, (N, T, 2)).astype(F32))
            self.u_cur.append(rng.uniform(-0.5, 2.5, (T, 2)).astype(F32))
            self.u_prev.append(rng.uniform(-0.5, 2.5, (T, 2)).astype(F32))
        self.f = np.ascontiguousarray(self.f, dtype=F32)
        self.g = np.ascontiguousarray(self.g, dtype=np.int32)
        self.ratios = np.ascontiguousarray(self.ratios, dtype=np.float64)
        self.modes = np.full(K, mode, dtype=np.int32)

    def launch(self, lib, batched, outs, active=None, out_off=0):
        lib.emu_vis(self.K, int(batched), _p(self.modes), self.V, _p(self.f), _p(self.g), _p(self.ratios),
                    _ptrs(self.lin), _ptrs(self.ang), _ptrs(self.noise), _ptrs(self.u_cur), _ptrs(self.u_prev),
                    _ptrs(outs), None if active is None else _p(active), out_off)

    def singles(self, lib):
        outs = [np.full((self.V, self.T + 1, 3), np.nan, F32) for _ in range(self.K)]
        self.launch(lib, False, outs)
        return np.stack(outs)


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_batched_equals_single_launches(emu, mode):
    """Modes 0 (u_cur over the first V maps), 1 / 2 (u_cur + V-1 clipped u_prev + noise) and 3 (no map)."""
    pl = Planners(mode, K=3)
    want = pl.singles(emu)
    assert not np.isnan(want).any()
    assert len({w.tobytes() for w in want}) == 3                     # the planners differ
    got = [np.full_like(want[0], 7.0) for _ in range(pl.K)]
    pl.launch(emu, True, got)
    assert np.stack(got).tobytes() == want.tobytes()


def test_inactive_planner_left_untouched(emu):
    pl = Planners(1, K=4)
    want = pl.singles(emu)
    got = [np.full_like(want[0], 7.0) for _ in range(pl.K)]
    pl.launch(emu, True, got, active=np.array([1, 0, 1, 0], dtype=np.int32))
    for k in range(pl.K):
        assert got[k].tobytes() == (want[k].tobytes() if k in (0, 2) else np.full_like(want[0], 7.0).tobytes()), k


def test_records_land_in_their_slot(emu):
    """Trial records: planner k's out is its (R, V, T+1, 3) slab, record r at out_off = r * V * (T+1) * 3 floats."""
    pl = Planners(0, K=3)
    want = pl.singles(emu)
    R = 4
    rec = np.full((pl.K, R, pl.V, pl.T + 1, 3), np.nan, F32)
    per = pl.V * (pl.T + 1) * 3
    for r in (2, 0):
        pl.launch(emu, True, [rec[k] for k in range(pl.K)], out_off=r * per)
    for k in range(pl.K):
        for r in range(R):
            if r in (0, 2):
                assert rec[k, r].tobytes() == want[k].tobytes(), (k, r)
            else:
                assert np.isnan(rec[k, r]).all(), (k, r)


def test_completion_equals_whole_map_sampling(emu_complete):
    """Maps [0, V) of every pair whose record says it sampled a box == the whole-map sampler from the same pre-call
    states; maps >= V, the states and the other buffers untouched; a pair whose step sampled whole maps and a gated
    pair untouched byte for byte."""
    lib = emu_complete
    rows, cols, tx, ty, M, B, segs, alpha = 61, 70, 4, 6, 5, 12, 3, 0.9       # ragged last tile row and column
    V, gm, mrows, ncact = 3, 2, 2, 4                  # gm 2: the launch's second map group holds map V, which it skips
    bpad = (B + 3) // 4 * 4
    rng = np.random.default_rng(17)
    pmfs = [random_pmf(rng, B, rows, cols) for _ in range(2)]
    cums = [cumulative_table(p, bpad) for p in pmfs]
    q = np.zeros(128, dtype=np.int8)
    q[:B] = TR.quantise_bin_values(np.linspace(0, 1, B), np.array([0.0, 1.0], dtype=np.float32))
    q_cap = min(int(min(int(np.cumsum(p.astype(np.int64), axis=0)[-1].min()) for p in pmfs)), 127)
    grid_rows, pitch = rows + 2, (cols + 15) // 16 * 16
    K, ngen = 4, tx * ty * M
    states = np.stack([X.create_states(ngen, 60 + k) for k in range(K)])
    # the whole-map sampling of every pair from its states (emu_sample_v2, tests/emu_sampler.py)
    whole = []
    for k in range(K):
        w0, w1 = np.zeros((M, grid_rows, pitch), np.int8), np.zeros((M, grid_rows, pitch), np.int8)
        assert lib.emu_sample_v2(2, _p(w0), _p(w1), _p(cums[0]), _p(cums[1]), _p(np.ascontiguousarray(states[k])),
                                 _p(np.zeros((ngen, 2), np.uint64)), _p(q), _p(q), bpad, rows, cols, grid_rows, pitch,
                                 tx, ty, M, segs, float(alpha), q_cap, None, None) == 0
        whole.append((w0, w1))
    # pair 0, 3: boxed steps (garbage outside the box); pair 1: a whole-map step (its maps already whole); pair 2 gated
    g0 = rng.integers(-100, 100, (K, M, grid_rows, pitch)).astype(np.int8)
    g1 = rng.integers(-100, 100, (K, M, grid_rows, pitch)).astype(np.int8)
    g0[1, :, :rows, :cols], g1[1, :, :rows, :cols] = whole[1][0][:, :rows, :cols], whole[1][1][:, :rows, :cols]
    rec = np.array([[2, 10, 20, 10, 20], [0, 0, rows, 0, cols], [1, 5, 9, 5, 9], [1, 30, 40, 30, 40]], dtype=np.int32)
    active = np.array([1, 1, 0, 1], dtype=np.int32)
    o0, o1 = np.full((K, ngen, 2), 5, np.uint64), np.full((K, ngen, 2), 6, np.uint64)
    before = [a.copy() for a in (g0, g1, o0, o1, states, rec)]
    assert lib.emu_complete(K, _p(g0), _p(g1), _p(cums[0]), _p(cums[1]), _p(states), _p(o0), _p(o1), _p(q), _p(q), bpad,
                            rows, cols, grid_rows, pitch, tx, ty, M, segs, C.c_double(alpha), q_cap, _p(rec),
                            _p(active), V, mrows, ncact, gm) == 0
    for a, b in zip((o0, o1, states, rec), before[2:]):
        assert a.tobytes() == b.tobytes()                       # no generator state, buffer or record written
    for k in range(K):
        if k in (0, 3):
            for got, w, b in zip((g0[k], g1[k]), whole[k], before[:2]):
                cells = np.zeros(got.shape, bool)
                cells[:V, :rows, :cols] = True
                assert got[cells].tobytes() == w[cells].tobytes(), "pair %d: maps [0, V)" % k
                assert got[~cells].tobytes() == b[k][~cells].tobytes(), "pair %d: maps >= V and padding" % k
        else:
            assert g0[k].tobytes() == before[0][k].tobytes() and g1[k].tobytes() == before[1][k].tobytes(), k
    assert (g0[1, :, :rows, :cols] == whole[1][0][:, :rows, :cols]).all()
    assert (g1[1, :, :rows, :cols] == whole[1][1][:, :rows, :cols]).all()
