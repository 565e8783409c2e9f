"""The batched one-map kernels compiled for the host (tests/emu_batch.py): ONE batched launch over K = 3 heterogeneous
planners (seeds, start poses, goals, lambda, u_std, map contents, rollout geometry) equals three single launches of
the same kernel text, bit for bit -- noise and RNG states, per-rollout costs (modes 1, 2, 3), the update's u, u_prev,
weights and the contiguous (K, T, 2) output, and the fused lin + ang sampler's maps and RNG states."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_batch
from tests.emu_sampler import cumulative_table

K = 3


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("emu_batch"))
    return dict(noise=emu_batch.build_noise(d), rollout=emu_batch.build_rollout(d), update=emu_batch.build_update(d),
                sampler=emu_batch.build_sampler(d))


def ptrs(arrays):
    return (C.c_void_p * len(arrays))(*[(a.ctypes.data if a is not None else None) for a in arrays])


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_noise_batched_equals_single(libs):
    N, T = 70, 9
    rng = np.random.default_rng(0)
    states0 = [rng.integers(1, 2 ** 63, (N * T, 2), dtype=np.uint64) for _ in range(K)]
    std = np.array([[2.0, 3.0], [0.5, 1.5], [1.0, 0.25]], dtype=np.float32)
    out = {}
    for batched in (0, 1):
        st = [s.copy() for s in states0]
        nz = [np.zeros((N, T, 2), np.float32) for _ in range(K)]
        libs["noise"].emu_noise(K, batched, ptrs(st), ptrs(nz), p(std), N * T)
        out[batched] = (st, nz)
    for i in range(K):
        assert np.array_equal(out[0][0][i], out[1][0][i]) and np.array_equal(out[0][1][i], out[1][1][i])
        assert not np.array_equal(out[1][0][i], states0[i])                          # the generators advanced
    assert not np.array_equal(out[1][1][0] / std[0], out[1][1][1] / std[1])             # each planner its own stream


def rollout_inputs(mode, seed, N, T):
    rng = np.random.default_rng(seed)
    rows, cols = 20 + 3 * seed, 24 + 2 * seed                   # geometry differs per planner
    grid_rows, grid_cols = rows + 2, cols + 5
    pitch, mpitch = (grid_cols + 15) // 16 * 16, (cols + 15) // 16 * 16
    res = 0.25 + 0.05 * seed
    f = np.zeros(23, np.float32)
    L = rows * res
    f[:23] = [res, 0.0, 0.0, 0.1, L / 2 + 0.1 * seed, L / 2 - 0.2 * seed, 0.3 * seed, L * 0.8, L * 0.3 + seed,
              0.4, 0.01, [1.0, 0.5, 2.0][seed % 3], 2.0 + seed * 0.3, 3.0 - seed * 0.5, 0.0, 3.0, -np.pi, np.pi,
              1e5 if mode != 3 else 1e3, 1e2, [1.0, 10.0, 0.5][seed % 3], 0.0, 0.0]
    g = np.array([rows, cols, grid_rows, grid_cols, pitch, mpitch, T, N, 1], np.int32)
    ratios = np.array([0.01, 0.01], np.float64)
    lin = rng.integers(0, 101, (grid_rows, pitch)).astype(np.int8)
    ang = rng.integers(0, 101, (grid_rows, pitch)).astype(np.int8)
    obs = (rng.random((rows, mpitch)) < 0.05).astype(np.int8)
    unk = (rng.random((rows, mpitch)) < 0.05).astype(np.int8)
    risk = rng.integers(0, 101, (rows, mpitch)).astype(np.int8)
    noise = (rng.standard_normal((N, T, 2)) * [2.0, 3.0]).astype(np.float32)
    u = np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(np.float32)
    ob = np.concatenate([rng.uniform(0, L, (2 + seed, 2)), rng.uniform(0.2, 1.0, (2 + seed, 1))], 1).astype(np.float32)
    return dict(f=f, g=g, ratios=ratios, lin=lin, ang=ang, obs=obs, unk=unk, risk=risk if mode == 2 else None,
                noise=noise, u=u, ob=ob if mode == 3 else np.zeros((1, 3), np.float32), nob=len(ob) if mode == 3 else 0)


@pytest.mark.parametrize("mode", [1, 2, 3])
def test_rollout_batched_equals_single(libs, mode):
    N, T = 150, 12
    ins = [rollout_inputs(mode, s, N, T) for s in range(K)]
    f = np.concatenate([x["f"] for x in ins])
    g = np.concatenate([x["g"] for x in ins])
    r = np.concatenate([x["ratios"] for x in ins])
    costs = {}
    for batched in (0, 1):
        c = [np.full(N, np.nan, np.float32) for _ in range(K)]
        libs["rollout"].emu_rollout(K, batched, mode, p(f), p(g), p(r), *[ptrs([x[k] for x in ins]) for k in (
            "lin", "ang", "obs", "unk", "risk", "noise", "u")], ptrs(c), ptrs([x["ob"] for x in ins]),
            p(np.array([x["nob"] for x in ins], np.int32)))
        costs[batched] = c
    for i in range(K):
        assert np.isfinite(costs[1][i]).all()
        assert np.array_equal(costs[0][i], costs[1][i]), "planner %d" % i
    assert not np.array_equal(costs[1][0], costs[1][1])


def test_update_batched_equals_single(libs):
    N, T = 300, 10                                                    # 10 CTAs per planner
    rng = np.random.default_rng(5)
    costs0 = [rng.uniform(0, 50, N).astype(np.float32) for _ in range(K)]
    noise0 = [rng.standard_normal((N, T, 2)).astype(np.float32) for _ in range(K)]
    u0 = [np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(np.float32) for _ in range(K)]
    lam = np.array([1.0, 0.3, 4.0], np.float32)
    vr = np.array([0, 3, 0, 2, 0.5, 2.5], np.float32)
    wr = np.array([-3, 3, -1, 1, -2, 2], np.float32)
    res = {}
    for batched in (0, 1):
        w_raw = [np.zeros(N, np.float32) for _ in range(K)]
        parts = [np.zeros((10, 2 * T + 2), np.float32) for _ in range(K)]
        rank = [np.zeros(2 * T + 2, np.float32) for _ in range(K)]
        u = [x.copy() for x in u0]
        w = [np.zeros(N, np.float32) for _ in range(K)]
        u_prev = [np.zeros((T, 2), np.float32) for _ in range(K)]
        u_out = np.zeros((K, T, 2), np.float32)
        left = libs["update"].emu_update(K, batched, ptrs(costs0), ptrs(noise0), ptrs(w_raw), ptrs(parts), ptrs(rank),
                                         ptrs(u), ptrs(w), ptrs(u_prev), ptrs([u_out[i] for i in range(K)]), N, T,
                                         p(lam), p(vr), p(wr))
        assert left == 0                                              # every ticket counter reset for the next launch
        res[batched] = dict(w_raw=w_raw, parts=parts, rank=rank, u=u, w=w, u_prev=u_prev, u_out=u_out)
    for i in range(K):
        for k in ("w_raw", "parts", "rank", "u", "w"):
            assert np.array_equal(res[0][k][i], res[1][k][i]), (i, k)
        # the batched tail stores u_prev (single path: after_u_update's copy) and the contiguous output
        assert np.array_equal(res[1]["u_prev"][i], res[0]["u"][i])
        assert np.array_equal(res[1]["u_out"][i], res[0]["u"][i])
        assert not np.array_equal(res[0]["u"][i], u0[i])
        assert abs(float(res[1]["w"][i].sum(dtype=np.float64)) - 1.0) < 1e-5
    assert not res[0]["u_prev"][0].any()                              # the single launch leaves u_prev / u_out alone


def test_sampler_batched_equals_single(libs):
    B, bpad, rows, cols, tx, ty, segs = 6, 8, 37, 45, 4, 4, 3
    grid_rows, pitch = 40, 48
    rng = np.random.default_rng(9)

    def pmf():
        cuts = np.sort(rng.integers(0, 101, (B - 1, rows, cols)), axis=0)
        out = np.empty((B, rows, cols), np.int64)
        out[0] = cuts[0]
        out[1:B - 1] = cuts[1:] - cuts[:-1]
        out[B - 1] = 100 - cuts[B - 2]
        return out.astype(np.int8)
    cum = [[cumulative_table(pmf(), bpad) for _ in range(2)] for _ in range(K)]
    q = [[np.zeros(128, np.int8) for _ in range(2)] for _ in range(K)]
    for i in range(K):
        for t in range(2):
            q[i][t][:B] = np.sort(rng.integers(0, 100, B)).astype(np.int8)
    st = [rng.integers(1, 2 ** 63, (tx * ty, 2), dtype=np.uint64) for _ in range(K)]
    out = {}
    for batched in (0, 1):
        g0 = [np.full((grid_rows, pitch), -1, np.int8) for _ in range(K)]
        g1 = [np.full((grid_rows, pitch), -1, np.int8) for _ in range(K)]
        so0 = [np.zeros_like(s) for s in st]
        so1 = [np.zeros_like(s) for s in st]
        rc = libs["sampler"].emu_sampler(K, batched, ptrs(g0), ptrs(g1), ptrs([c[0] for c in cum]),
                                         ptrs([c[1] for c in cum]), ptrs(st), ptrs(so0), ptrs(so1),
                                         ptrs([x[0] for x in q]), ptrs([x[1] for x in q]), bpad, rows, cols, grid_rows,
                                         pitch, tx, ty, segs, 1.0, 100)
        assert rc == 0
        out[batched] = (g0, g1, so0, so1)
    for i in range(K):
        for k in range(4):
            assert np.array_equal(out[0][k][i], out[1][k][i]), (i, k)
        assert (out[1][0][i][:rows, :cols] >= 0).all()                 # every map cell sampled
        assert np.array_equal(out[1][2][i], out[1][3][i])              # both TDMs advance alike
    assert not np.array_equal(out[1][0][0], out[1][0][1])
