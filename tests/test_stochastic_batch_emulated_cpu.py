"""The batched stochastic kernels' real source executed on the host (tests/emu_stochastic_batch.py) against the
single-planner kernels they stand in for, bit for bit: the batched noise + prepare launch, the batched windowed
rollout (planners differing in goal, start, dt, penalties and traction ratios; windows clamped at the map edge and
rollouts leaving them; a ragged last chunk; 0/1 and 0..3 masks; shares of 1-7 CTAs crossing planner boundaries in each
share regime) and the batched CVaR."""
import numpy as np
import pytest

from tests.emu_stochastic_batch import build
from tests.test_rollout_emulated_cpu import _c, _fparams, _p, _ratios

F32 = np.float32


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build(str(tmp_path_factory.mktemp("emu_sto_batch")))


@pytest.mark.parametrize("iteration", [0, 1])
def test_batched_noise_prepare_equals_single_launches(emu, iteration):
    win, _ = emu
    K, N, T = 3, 45, 37                                   # N not a multiple of 8 or 32, T over one 32-step tile
    rng = np.random.default_rng(3 + iteration)
    states = _c(rng.integers(0, 2 ** 63, (K, N * T, 2), dtype=np.uint64), np.uint64)
    u = _c(rng.uniform(-1, 2, (K, T, 2)), F32)
    fp = _c([[2.0 + k, 3.0 - 0.5 * k, 0.5 + k, -0.1 * k, 2.5 + k, -3.0, 3.0 - k] for k in range(K)], F32)
    slots = _c([0, 1, 0], np.int32)
    assert win.emu_noise_prepare_batch(K, _p(states), _p(u), N, T, _p(fp), _p(slots), iteration) == 0


def planners(K, N, T, M, H, W, seed, mixed_masks):
    rng = np.random.default_rng(seed)
    R, Cc = H + 3, W + 5                                   # sample buffers larger than the map
    pitch = (Cc + 15) // 16 * 16
    mpitch = (W + 15) // 16 * 16
    lin = rng.integers(-128, 128, (K, M, R, pitch)).astype(np.int8)
    ang = rng.integers(-128, 128, (K, M, R, pitch)).astype(np.int8)
    obs = np.zeros((K, H, mpitch), np.int8)
    unk = np.zeros((K, H, mpitch), np.int8)
    m01 = []
    for k in range(K):
        hi = 4 if (mixed_masks and k == 1) else 2
        obs[k, :, :W] = rng.integers(0, hi, (H, W)) * (rng.random((H, W)) < 0.1)
        unk[k, :, :W] = rng.integers(0, hi, (H, W)) * (rng.random((H, W)) < 0.1)
        m01.append(int(hi == 2))
    res = 0.2
    fs, ratios = [], []
    for k in range(K):
        x0 = [W * res * (0.5 + 0.1 * k), H * res * (0.45 - 0.1 * k), 0.3 * k]
        if k == 2:
            x0 = [0.3, H * res - 0.3, 1.0]                     # at a map corner: rollouts leave the map
        goal = [x0[0] + 3.0 - k, x0[1] + 1.0 + k]
        fs.append(_fparams(res, -0.6, -0.4, [0.1, 0.08, 0.13][k % 3], x0, goal, 0.3 + 0.1 * k, 0.01 + 0.01 * k,
                           1.0 + 0.5 * k, [1.5 + 0.2 * k, 2.0], [0.0, 3.0], [-np.pi, np.pi], 1e3 * (k + 1), 50.0 + k,
                           1.0 + 0.3 * k, -0.2 * k, -0.1))
        ratios.append(_ratios([-0.2 * k, 1.0 + 0.1 * k], [-0.1, 0.9 + 0.2 * k]))
    geo = _c([H, W, R, Cc, pitch, mpitch, T, N, M], np.int32)
    noise = _c(rng.normal(0, 1.5, (K, N, T, 2)), F32)
    u = _c(rng.uniform(-0.5, 2.0, (K, T, 2)), F32)
    return (_c(np.concatenate(fs), F32), geo, _c(np.concatenate(ratios), np.float64), _c(lin, np.int8), _c(ang, np.int8),
            _c(obs, np.int8), _c(unk, np.int8), noise, u, _c(m01, np.int32))


@pytest.mark.parametrize("ctas,unit", [(1, 32), (5, 32), (3, 1), (7, 1), (6, 0), (7, 0)])
def test_batched_windowed_rollout_equals_single_launches(emu, ctas, unit):
    win, _ = emu
    K, N, T, M = 3, 40, 14, 2                              # ragged last chunk: 40 = 32 + 8
    args = planners(K, N, T, M, H=60, W=70, seed=ctas * 10 + unit, mixed_masks=(ctas % 2 == 1))
    out_b = np.full((K, N, M), np.nan, F32)
    out_s = np.full((K, N, M), np.nan, F32)
    assert win.emu_win_batch(K, *[_p(a) for a in args[:9]], ctas, unit, _p(args[9]), _p(out_b), _p(out_s)) == 0
    assert np.isfinite(out_s).all()
    assert out_b.tobytes() == out_s.tobytes()


def test_batched_cvar_equals_single_launches(emu):
    _, cv = emu
    rng = np.random.default_rng(5)
    for N, M in ((70, 24), (33, 200)):
        K = 3
        costs = _c(rng.normal(10, 3, (K, M, N)), F32)
        numel = _c([max(1, int(np.ceil(M * a))) for a in (0.5, 0.1, 1.0)], np.int32)
        ob, os_ = np.zeros((K, N), F32), np.full((K, N), np.nan, F32)
        assert cv.emu_cvar_batch(K, _p(costs), N, M, _p(numel), _p(ob), _p(os_)) == 0
        assert ob.tobytes() == os_.tobytes()
