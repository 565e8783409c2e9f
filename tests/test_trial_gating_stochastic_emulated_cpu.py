"""Gating of the batched stochastic kernels for closed-loop trials, from their REAL source on the host (the harnesses
of tests/emu_stochastic_batch.py): noise_prepare_batch_kernel with an `active` array and cvar_batch_kernel with
CvarDesc::active -- running planners equal an ungated launch bit for bit, stopped planners are left byte for byte as
they were (states, noise, transposed controls, control costs, both reach slots; CVaR costs)."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_stochastic_batch as ESB

NOISE = r'''
// K planners, one gated and one ungated batched launch (iteration `iter`) on copies of the same buffers; returns
// 0 when the running planners agree and the stopped ones are untouched
extern "C" int emu_noise_gated(int K, const uint64_t* states_in, const float* u_cur, int N, int T, const float* fp,
                               int iter, const int* active) {
  const int npad = (N + 31) / 32 * 32;
  const size_t ns = (size_t)N * T * 2, nT = (size_t)(T + 1) * npad;
  struct Bufs {
    std::vector<uint64_t> st; std::vector<float> noise, ctrl, reach; std::vector<double2> noiseT; std::vector<NoisePrepDesc> d;
  } b[3];
  for (auto& x : b) {
    x.st.assign(states_in, states_in + K * ns);
    x.noise.assign(K * ns, 3.0f); x.ctrl.assign(K * npad, 4.0f); x.reach.assign(2 * K, 7.0f);
    x.noiseT.assign(K * nT, double2{5, 6});
    x.d.resize(K);
    for (int k = 0; k < K; ++k) {
      const float* q = fp + 7 * k;
      x.d[k] = NoisePrepDesc{x.st.data() + k * ns, x.noise.data() + k * ns, u_cur + (size_t)k * T * 2,
                             reinterpret_cast<float*>(x.noiseT.data() + k * nT), x.ctrl.data() + k * npad,
                             x.reach.data() + 2 * k, k & 1, q[0], q[1], q[2], q[0] * q[0], q[1] * q[1], q[3], q[4], q[5], q[6]};
      x.reach[2 * k + ((k & 1) ^ (iter & 1))] = 0.0f;
    }
  }
  const EmuDim3 grid{(unsigned)(npad / NP_NB), (unsigned)K, 1};
  emu::launch(grid, 256, [&] { noise_prepare_batch_kernel(b[0].d.data(), N, T, npad, iter, active); });
  emu::launch(grid, 256, [&] { noise_prepare_batch_kernel(b[1].d.data(), N, T, npad, iter); });
  for (int k = 0; k < K; ++k) {
    const Bufs& want = active[k] ? b[1] : b[2];        // b[2]: never launched
    if (std::memcmp(b[0].st.data() + k * ns, want.st.data() + k * ns, ns * 8)) return 1;
    if (std::memcmp(b[0].noise.data() + k * ns, want.noise.data() + k * ns, ns * 4)) return 2;
    if (std::memcmp(b[0].noiseT.data() + k * nT, want.noiseT.data() + k * nT, nT * 16)) return 3;
    if (std::memcmp(b[0].ctrl.data() + k * npad, want.ctrl.data() + k * npad, npad * 4)) return 4;
    if (std::memcmp(b[0].reach.data() + 2 * k, want.reach.data() + 2 * k, 8)) return 5;
  }
  return 0;
}
'''

CVAR = r'''
extern "C" int emu_cvar_gated(int K, const float* costs_mn, int N, int M, const int* numel, const int* active) {
  std::vector<float> gated(K * N, -3.0f), full(K * N, -3.0f);
  std::vector<CvarDesc> dg(K), df(K);
  for (int k = 0; k < K; ++k) {
    dg[k] = CvarDesc{costs_mn + (size_t)k * M * N, gated.data() + (size_t)k * N, N, N, M, numel[k], active + k};
    df[k] = CvarDesc{costs_mn + (size_t)k * M * N, full.data() + (size_t)k * N, N, N, M, numel[k]};
  }
  const int nb = cvar_block_n(M);
  const EmuDim3 grid{(unsigned)((N + nb - 1) / nb), (unsigned)K, 1};
  emu::cvar_per(M, [&](auto P) {
    emu::launch(grid, CVAR_THREADS, [&] { cvar_batch_kernel<decltype(P)::value>(dg.data()); });
    emu::launch(grid, CVAR_THREADS, [&] { cvar_batch_kernel<decltype(P)::value>(df.data()); });
  });
  for (int k = 0; k < K; ++k)
    for (int n = 0; n < N; ++n) {
      const float want = active[k] ? full[(size_t)k * N + n] : -3.0f;
      if (std::memcmp(&gated[(size_t)k * N + n], &want, 4)) return 1 + k;
    }
  return 0;
}
'''


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    return ESB.build(str(tmp_path_factory.mktemp("gating")), extra=NOISE, cvar_extra=CVAR)


def _p(a):
    return C.c_void_p(a.ctypes.data)


@pytest.mark.parametrize("iteration", [0, 3])
def test_gated_noise_prepare(libs, iteration):
    from oracle import xoroshiro as X
    lib, _ = libs
    K, N, T = 4, 45, 6
    rng = np.random.default_rng(9)
    states = np.concatenate([X.create_states(N * T * 2, 3 + k) for k in range(K)])
    u = rng.uniform(-1, 1, (K, T, 2)).astype(np.float32)
    fp = np.tile(np.array([0.5, 0.7, 1.0, -1.0, 2.0, -1.5, 1.5], np.float32), K)
    active = np.array([1, 0, 1, 0], np.int32)
    assert lib.emu_noise_gated(K, _p(states), _p(u), N, T, _p(fp), iteration, _p(active)) == 0


def test_gated_cvar(libs):
    _, cvl = libs
    K, N, M = 3, 70, 40
    rng = np.random.default_rng(4)
    costs = rng.uniform(0, 10, (K, M, N)).astype(np.float32)
    numel = np.array([4, 20, 40], np.int32)
    active = np.array([0, 1, 0], np.int32)
    assert cvl.emu_cvar_gated(K, _p(costs), N, M, _p(numel), _p(active)) == 0
