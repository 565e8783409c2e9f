"""Active-planner gating of the batched kernels, emulated on the host (tests/emu_batch.py's sources with a harness that
passes ``active``): an inactive planner's buffers -- its generator states, noise, CTA partials, weights, u and the update's
ticket counter -- are byte-identical to before the launch, and an active planner's are byte-identical to the ungated
launch."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_batch

NOISE = r'''
extern "C" void emu_noise_gated(int K, const int* active, uint64_t** states, float** noise, const float* std, long long count) {
  std::vector<NoiseDesc> d(K);
  for (int i = 0; i < K; ++i) d[i] = NoiseDesc{states[i], noise[i], std[2 * i], std[2 * i + 1]};
  emu::launch_serial({(unsigned)((count + 255) / 256), (unsigned)K, 1}, 256, [&] { sample_noise_batch_kernel(d.data(), count, active); });
}
'''

UPDATE = r'''
extern "C" void emu_update_gated(int K, const int* active, const float** costs, const float** noise, float** w_raw,
                                 float** parts, float** rank_partial, float** u_cur, float** weights, float** u_prev,
                                 float** u_out, unsigned* counters, int N, int T) {
  std::vector<UpdateBatchDesc> d(K);
  int ctas, rows_per_cta;
  emu::update_geometry(N, ctas, rows_per_cta);
  for (int i = 0; i < K; ++i) {
    UpdateArgs a{};
    a.costs = costs[i]; a.noise = noise[i]; a.w_raw = w_raw[i]; a.cta_partials = parts[i]; a.rank_partial = rank_partial[i];
    a.u_cur = u_cur[i]; a.weights = weights[i]; a.N = N; a.T = T; a.num_ctas = ctas; a.rows_per_cta = rows_per_cta;
    a.lambda = 1.0f + i; a.vrange[0] = 0.0f; a.vrange[1] = 3.0f; a.wrange[0] = -3.0f; a.wrange[1] = 3.0f;
    UpdateTail tl{};
    tl.counter = &counters[i]; tl.mode = UPD_TAIL_APPLY; tl.u_prev = u_prev[i]; tl.u_out = u_out[i];
    d[i] = UpdateBatchDesc{a, tl};
  }
  emu::launch({(unsigned)ctas, (unsigned)K, 1}, UPD_THREADS, [&] { update_partial_batch_kernel(d.data(), active); });
}
'''


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("gating"))
    return emu_batch.build_noise(out, extra=NOISE), emu_batch.build_update(out, extra=UPDATE)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def ptrs(arrs):
    return (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])


def test_noise_gating(libs):
    noise_lib = libs[0]
    K, N, T = 3, 40, 7
    rng = np.random.default_rng(0)
    states0 = [rng.integers(1, 2 ** 63, (N * T, 2), dtype=np.uint64) for _ in range(K)]
    std = np.array([1.0, 2.0, 1.5, 0.5, 3.0, 1.0], np.float32)
    runs = []
    for active in ([1, 1, 1], [1, 0, 1]):
        st = [s.copy() for s in states0]
        nz = [np.full((N, T, 2), 9.0, np.float32) for _ in range(K)]
        act = np.array(active, np.int32)
        noise_lib.emu_noise_gated(K, _p(act), ptrs(st), ptrs(nz), _p(std), N * T)
        runs.append((st, nz))
    (s_all, n_all), (s_g, n_g) = runs
    assert np.array_equal(s_g[1], states0[1]) and (n_g[1] == 9.0).all()
    for k in (0, 2):
        assert np.array_equal(s_g[k], s_all[k]) and np.array_equal(n_g[k], n_all[k])
        assert not np.array_equal(s_all[k], states0[k])


def test_update_gating_leaves_the_ticket_counter(libs):
    update_lib = libs[1]
    K, N, T = 3, 100, 6
    rng = np.random.default_rng(1)
    costs = [rng.uniform(0, 10, N).astype(np.float32) for _ in range(K)]
    noise = [rng.normal(size=(N, T, 2)).astype(np.float32) for _ in range(K)]
    u0 = [rng.uniform(-1, 1, (T, 2)).astype(np.float32) for _ in range(K)]
    ctas = (N + 31) // 32
    runs = []
    for active in ([1, 1, 1], [0, 1, 1]):
        bufs = dict(w=[np.full(N, 5.0, np.float32) for _ in range(K)],
                    parts=[np.full((ctas, 2 * T + 2), 5.0, np.float32) for _ in range(K)],
                    rank=[np.full(2 * T + 2, 5.0, np.float32) for _ in range(K)], u=[u.copy() for u in u0],
                    weights=[np.full(N, 5.0, np.float32) for _ in range(K)],
                    prev=[np.full((T, 2), 5.0, np.float32) for _ in range(K)],
                    out=[np.full((T, 2), 5.0, np.float32) for _ in range(K)])
        counters = np.array([7, 0, 0], np.uint32) if active[0] == 0 else np.zeros(K, np.uint32)
        act = np.array(active, np.int32)
        update_lib.emu_update_gated(K, _p(act), ptrs(costs), ptrs(noise), ptrs(bufs["w"]), ptrs(bufs["parts"]),
                                    ptrs(bufs["rank"]), ptrs(bufs["u"]), ptrs(bufs["weights"]), ptrs(bufs["prev"]),
                                    ptrs(bufs["out"]), _p(counters), N, T)
        runs.append((bufs, counters))
    (b_all, c_all), (b_g, c_g) = runs
    assert c_g.tolist() == [7, 0, 0] and c_all.tolist() == [0, 0, 0]
    for name in b_all:
        assert np.array_equal(b_g[name][0], np.full_like(b_g[name][0], 5.0) if name != "u" else u0[0]), name
        for k in (1, 2):
            assert np.array_equal(b_g[name][k], b_all[name][k]), (name, k)
