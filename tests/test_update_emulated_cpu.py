"""The control-update kernels' real source (online softmax in two levels: CTA partials -> rank partial ->
combine), executed on the host by tests/emu_update.py, against a float64 reference of update_useq_numba
(mppi.py:1113-1191) within per-element bounds derived from the kernels' reduction structure (tests/reduce_bounds.py),
and against the reference's own result (ref_update.npz); N sharded over 'ranks' gives the one-rank update.  Shapes
cross the 64- and 8-row batches (rows_per_cta > 32 past N = 9472) and all four 256-column chunks (T up to 1024);
values include lambda from 1e-3 to 1e3, whole CTAs whose merge scale underflows, costs near 1e6, negative costs,
+inf costs (scattered, a whole CTA slab, a whole rank), u0 on the clip bounds and noise that cancels."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import mppi_ref as MR
from tests import reduce_bounds as RB
from tests.emu_update import build

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
VR, WR = np.array([0, 3], np.float32), np.array([-np.pi, np.pi], np.float32)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build(str(tmp_path_factory.mktemp("emu_update")))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _partial(emu, costs, noise, lam):
    N, T = noise.shape[:2]
    ctas = emu.emu_update_num_ctas(N)
    w_raw = np.zeros(N, np.float32)
    parts = np.zeros((ctas, 2 * T + 2), np.float32)
    rank = np.zeros(2 * T + 2, np.float32)
    emu.emu_update_partial(_p(costs), _p(noise), _p(w_raw), _p(parts), _p(rank), N, T, np.float32(lam))
    return w_raw, parts, rank


def _finish(emu, gathered, w_raw, parts, u0, N, T, lam):
    u = u0.copy()
    w = np.zeros(N, np.float32)
    g = np.ascontiguousarray(gathered, dtype=np.float32)
    emu.emu_update_finish(_p(g), g.shape[0], _p(w_raw), _p(parts), _p(u), _p(w), N, T, np.float32(lam), _p(VR), _p(WR))
    return u, w


def _one_rank(emu, costs, noise, u0, lam):
    """The one-launch update (UPD_TAIL_APPLY): (u, weights, rank partial)."""
    N, T = noise.shape[:2]
    ctas = emu.emu_update_num_ctas(N)
    w_raw, parts, rank = np.zeros(N, np.float32), np.zeros((ctas, 2 * T + 2), np.float32), np.zeros(2 * T + 2, np.float32)
    u, w = u0.copy(), np.zeros(N, np.float32)
    assert emu.emu_update_one_rank(_p(costs), _p(noise), _p(w_raw), _p(parts), _p(rank), _p(u), _p(w), N, T,
                                   np.float32(lam), _p(VR), _p(WR)) == 0
    return u, w, rank


@pytest.mark.parametrize("lam", [1.0, 0.3])
def test_update_kernels_match_reference_golden(emu, lam):
    g = np.load(os.path.join(GOLDEN, "ref_update.npz"))
    costs, noise, u0 = (np.ascontiguousarray(g[k], dtype=np.float32) for k in ("costs", "noise", "u0"))
    N, T = noise.shape[:2]
    w_raw, parts, rank = _partial(emu, costs, noise, lam)
    u, w = _finish(emu, rank[None, :], w_raw, parts, u0, N, T, lam)
    key = "lam%02d" % int(lam * 10)
    np.testing.assert_allclose(u, g["u_" + key], rtol=1e-5, atol=2e-6)     # the reference's own float32 result
    np.testing.assert_allclose(w, g["w_" + key], rtol=1e-4, atol=1e-12)
    RB.check_update(u, w, costs, noise, u0, lam, VR, WR, label="golden lam %g" % lam)


SHAPES = [(1000, 50), (300, 300), (37, 3), (9600, 8),
          (1, 1024), (2, 513), (31, 512), (32, 511), (33, 257), (9472, 256), (9473, 255), (16384, 1), (15000, 64),
          (16384, 1024)]
VALUES = [(k, lam) for k in ("mild", "underflow", "far", "signed", "inf", "clip", "cancel")
          for lam in (1e-3, 0.3, 1.0, 1e3)]


@pytest.mark.parametrize("N,T,kind,lam", [pytest.param(N, T, "mild", 1.0, id="%d-%d" % (N, T)) for N, T in SHAPES] +
                         [(N, T, k, lam) for N, T in ((1000, 50), (9473, 33)) for k, lam in VALUES
                          if N == 1000 or lam in (1e-3, 1e3)])
def test_update_kernels_match_oracle(emu, N, T, kind, lam):
    costs, noise, u0 = RB.update_inputs(kind, N, T, seed=N + T, lam=lam)
    w_raw, parts, rank = _partial(emu, costs, noise, lam)
    u, w = _finish(emu, rank[None, :], w_raw, parts, u0, N, T, lam)
    label = "N%d T%d %s lam %g" % (N, T, kind, lam)
    RB.check_update(u, w, costs, noise, u0, lam, VR, WR, label=label)
    # the numpy oracle (float32 weights, float32 normalisation, another order) stays within the same bounds
    want_u, want_w = MR.update_useq(lam, costs, noise, VR, WR, u0)
    RB.check_update(want_u, want_w, costs, noise, u0, lam, VR, WR, label=label + " (numpy oracle)")
    assert abs(float(w.sum(dtype=np.float64)) - 1.0) < 1e-5


def _sharded_inputs(kind, N, T, ws):
    if kind == "inf_rank":            # rank 1's rollouts all cost +inf
        costs, noise, u0 = RB.update_inputs("mild", N, T, seed=3)
        costs[N // ws: 2 * N // ws] = np.inf
        return costs, noise, u0, 1.0
    costs, noise, u0 = RB.update_inputs(kind, N, T, seed=3)
    return costs, noise, u0, 1.0


def test_sharded_update_equals_single_rank(emu):
    """4 'ranks' own N/4 control sequences each; their (2T+2)-float partials, gathered, give every rank the one-rank u
    (every rank's u within the bound of the float64 reference, and all ranks identical)."""
    _sharded_update(emu, "mild")


@pytest.mark.parametrize("kind", ["inf_rank", "underflow"])
def test_sharded_update_with_an_all_inf_rank_or_underflowing_ctas(emu, kind):
    """The sharded update when one rank's rollouts all cost +inf (its partial must not poison the other ranks' u) and
    when whole CTAs' merge scales underflow: every rank's u and the weights within the bound, all ranks identical."""
    _sharded_update(emu, kind)


def _sharded_update(emu, kind):
    N, T, ws = 2048, 64, 4
    costs, noise, u0, lam = _sharded_inputs(kind, N, T, ws)
    w_raw, parts, rank = _partial(emu, costs, noise, lam)
    u1, w1 = _finish(emu, rank[None, :], w_raw, parts, u0, N, T, lam)
    RB.check_update(u1, w1, costs, noise, u0, lam, VR, WR, label="one rank " + kind)
    shards = []
    for r in range(ws):
        sl = slice(N * r // ws, N * (r + 1) // ws)
        shards.append(_partial(emu, np.ascontiguousarray(costs[sl]), np.ascontiguousarray(noise[sl]), lam))
    gathered = np.stack([s[2] for s in shards])
    ws_w, us = [], []
    for r in range(ws):
        u, w = _finish(emu, gathered, shards[r][0], shards[r][1], u0, N // ws, T, lam)
        us.append(u)
        ws_w.append(w)
    assert all((x == us[0]).all() for x in us)
    RB.check_update(us[0], np.concatenate(ws_w), costs, noise, u0, lam, VR, WR, N=N // ws, merges=ws,
                    label="sharded " + kind)


@pytest.mark.parametrize("N,T", [(1000, 50), (8192, 128), (37, 3), (9473, 513), (16384, 1024)])
def test_one_launch_update_equals_partial_plus_finish(emu, N, T):
    """One rank: the last CTA of update_partial_kernel applies the update itself (UPD_TAIL_APPLY) -- bit-identical to
    the two-step path (rank partial, then update_apply_kernel on that single partial), and within the bound."""
    rng = np.random.default_rng(N * 7 + T)
    costs = rng.uniform(900, 930, N).astype(np.float32)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(np.float32)
    u0 = np.stack([rng.uniform(0, 2.9, T), rng.uniform(-3, 3, T)], 1).astype(np.float32)
    w_raw, parts, rank = _partial(emu, costs, noise, 1.0)
    u2, w2 = _finish(emu, rank[None, :], w_raw, parts, u0, N, T, 1.0)
    u1, w1, rank1 = _one_rank(emu, costs, noise, u0, 1.0)
    assert (u1 == u2).all() and (w1 == w2).all() and (rank1 == rank).all()
    RB.check_update(u1, w1, costs, noise, u0, 1.0, VR, WR, label="N%d T%d" % (N, T))


@pytest.mark.parametrize("N", [1000, 9473])
def test_update_with_an_all_inf_cta_slab(emu, N):
    """One CTA slab of +inf costs: its baseline is +inf, and c - beta = inf - inf must not turn its weights, S and V
    into NaN (which the clip would turn into u = the upper bounds).  Its rollouts get weight exactly 0 and u equals the
    float64 reference, whose beta is the global minimum (exp(-inf) = 0), within the bound -- in the one-launch update
    and in the two-step path."""
    T = 4 if N == 1000 else 64
    costs = RB.inf_slab_costs(N)
    rng = np.random.default_rng(N)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(np.float32)
    u0 = np.stack([rng.uniform(0, 2.9, T), rng.uniform(-3, 3, T)], 1).astype(np.float32)
    u1, w1, _ = _one_rank(emu, costs, noise, u0, 1.0)
    RB.check_update(u1, w1, costs, noise, u0, 1.0, VR, WR, label="one launch, N %d" % N)
    w_raw, parts, rank = _partial(emu, costs, noise, 1.0)
    assert (w_raw[np.isinf(costs)] == 0).all()
    u2, w2 = _finish(emu, rank[None, :], w_raw, parts, u0, N, T, 1.0)
    assert (u1 == u2).all() and (w1 == w2).all()


@pytest.mark.parametrize("N,T", [(37, 3), (1000, 4), (9473, 64)])
def test_update_with_every_cost_inf(emu, N, T):
    """Every cost +inf (a barebone planner whose penalties overflow float32): every partial has scale 0, so W = 0.  The
    update is a zero step -- u = clip(u0), with u0 outside the bounds in places -- and every weight is 0, in the
    one-launch update, the two-step path and the sharded combine of 4 ranks; 0 / 0 would make u NaN, which the clip
    turns into the upper bounds."""
    rng = np.random.default_rng(N + T)
    costs = np.full(N, np.inf, np.float32)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(np.float32)
    u0 = np.stack([rng.uniform(-1, 4, T), rng.uniform(-4, 4, T)], 1).astype(np.float32)
    u1, w1, _ = _one_rank(emu, costs, noise, u0, 1.0)
    RB.check_update(u1, w1, costs, noise, u0, 1.0, VR, WR, label="one launch, N %d" % N)
    w_raw, parts, rank = _partial(emu, costs, noise, 1.0)
    u2, w2 = _finish(emu, rank[None, :], w_raw, parts, u0, N, T, 1.0)
    RB.check_update(u2, w2, costs, noise, u0, 1.0, VR, WR, label="two steps, N %d" % N)
    ws = 4
    shards = [_partial(emu, np.ascontiguousarray(costs[N * r // ws: N * (r + 1) // ws]),
                       np.ascontiguousarray(noise[N * r // ws: N * (r + 1) // ws]), 1.0) for r in range(ws)]
    gathered = np.stack([s[2] for s in shards])
    for r in range(ws):
        n = N * (r + 1) // ws - N * r // ws
        u, w = _finish(emu, gathered, shards[r][0], shards[r][1], u0, n, T, 1.0)
        RB.check_update(u, None, costs, noise, u0, 1.0, VR, WR, label="sharded, rank %d" % r)
        assert (w == 0).all()


def test_update_tail_broadcasts_the_rank_partial_to_every_peer(emu):
    """UPD_TAIL_BCAST (peer-memory exchange): 3 'ranks', each stores its partial into slot `rank` of all three
    gather buffers and raises its own epoch flag in every peer -- the gather buffers end up identical and equal to
    the stacked rank partials; combining them gives the one-rank update."""
    N, T, ws = 1536, 32, 3
    rng = np.random.default_rng(11)
    costs = rng.uniform(900, 930, N).astype(np.float32)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(np.float32)
    u0 = rng.uniform(0, 1, (T, 2)).astype(np.float32)
    gather = np.zeros((ws, ws, 2 * T + 2), np.float32)
    flags = np.zeros((ws, ws), np.uint32)
    shards = []
    for r in range(ws):
        sl = slice(N * r // ws, N * (r + 1) // ws)
        n = N // ws
        ctas = emu.emu_update_num_ctas(n)
        w_raw, parts, rank = np.zeros(n, np.float32), np.zeros((ctas, 2 * T + 2), np.float32), np.zeros(2 * T + 2, np.float32)
        assert emu.emu_update_bcast(_p(np.ascontiguousarray(costs[sl])), _p(np.ascontiguousarray(noise[sl])), _p(w_raw),
                                    _p(parts), _p(rank), n, T, np.float32(1.0), ws, r, _p(gather), _p(flags), 5) == 0
        shards.append((w_raw, parts, rank))
    assert (flags == 5).all()
    for q in range(ws):
        assert (gather[q] == np.stack([s[2] for s in shards])).all()
    u, _ = _finish(emu, gather[0], shards[0][0], shards[0][1], u0, N // ws, T, 1.0)
    RB.check_update(u, None, costs, noise, u0, 1.0, VR, WR, N=N // ws, merges=ws, label="broadcast")
