"""Host emulation of the batched stochastic kernels (TEST INFRASTRUCTURE; tests/emu_core.py): noise_prepare_batch_kernel
and rollout_win_batch_kernel (csrc/rollout_win.cu) next to their single-planner kernels, with the harness of
tests/emu_rollout_win.py (emu_rollout_win included) compiled in as the single-planner reference; cvar_batch_kernel
(csrc/rollout.cu) next to launch_cvar's single kernels, with the harness of tests/emu_cvar.py."""
from tests import emu_cvar, emu_rollout_win
from tests.emu_core import build as _build

HARNESS = r'''
// K planners of equal N, T: one batched noise + prepare launch (iteration `iter`) against one single launch per planner
extern "C" int emu_noise_prepare_batch(int K, const uint64_t* states_in, const float* u_cur, int N, int T, const float* fp,
                                       const int* slots, int iter) {
  const int npad = (N + 31) / 32 * 32;
  const size_t ns = (size_t)N * T * 2, nT = (size_t)(T + 1) * npad;
  std::vector<uint64_t> st(states_in, states_in + K * ns), st2 = st;
  std::vector<float> noise(K * ns, 0.0f), noise2 = noise, ctrl(K * npad, 0.0f), ctrl2 = ctrl;
  std::vector<double2> noiseT(K * nT, double2{0, 0}), noiseT2 = noiseT;
  std::vector<float> reach(2 * K, 7.0f), reach2 = reach;
  std::vector<NoisePrepDesc> d(K);
  for (int k = 0; k < K; ++k) {
    const float* q = fp + 7 * k;                            // std_v, std_w, lambda, v_lo, v_hi, w_lo, w_hi
    d[k] = NoisePrepDesc{st.data() + k * ns, noise.data() + k * ns, u_cur + (size_t)k * T * 2,
                         reinterpret_cast<float*>(noiseT.data() + k * nT), ctrl.data() + k * npad, reach.data() + 2 * k,
                         slots[k], q[0], q[1], q[2], q[0] * q[0], q[1] * q[1], q[3], q[4], q[5], q[6]};
    reach[2 * k + (slots[k] ^ (iter & 1))] = 0.0f;         // the slot this launch reduces into starts cleared
    reach2[2 * k + (slots[k] ^ (iter & 1))] = 0.0f;
  }
  emu::launch({(unsigned)(npad / NP_NB), (unsigned)K, 1}, 256, [&] { noise_prepare_batch_kernel(d.data(), N, T, npad, iter); });
  for (int k = 0; k < K; ++k) {
    const float* q = fp + 7 * k;
    emu::launch({(unsigned)(npad / NP_NB), 1, 1}, 256, [&] {
      noise_prepare_kernel(st2.data() + k * ns, reinterpret_cast<float2*>(noise2.data() + k * ns), u_cur + (size_t)k * T * 2,
                           noiseT2.data() + k * nT, ctrl2.data() + k * npad, reach2.data() + 2 * k, slots[k] ^ (iter & 1),
                           N, T, npad, q[0], q[1], q[2], q[0] * q[0], q[1] * q[1], q[3], q[4], q[5], q[6]);
    });
  }
  if (std::memcmp(st.data(), st2.data(), st.size() * 8)) return 1;
  if (std::memcmp(noise.data(), noise2.data(), noise.size() * 4)) return 2;
  if (std::memcmp(noiseT.data(), noiseT2.data(), noiseT.size() * 16)) return 3;
  if (std::memcmp(ctrl.data(), ctrl2.data(), ctrl.size() * 4)) return 4;
  if (std::memcmp(reach.data(), reach2.data(), reach.size() * 4)) return 5;
  for (int k = 0; k < K; ++k)
    if (reach[2 * k + (slots[k] ^ (iter & 1) ^ 1)] != 0.0f) return 6;   // the other slot cleared for the next launch
  return 0;
}

// K planners of equal N, T, M (their own params, maps, masks, noise, u): one batched windowed launch on `ctas` CTAs with
// share unit `unit` (0: by unit, needs ctas >= K*M; 1; 32) -> out_batch (K, N, M); each planner's single launch
// (emu_rollout_win, the launcher's own CTA count) -> out_single (K, N, M)
extern "C" int emu_win_batch(int K, const float* f, const int* g, const double* ratios, const int8_t* lin, const int8_t* ang,
                             const int8_t* obs, const int8_t* unk, const float* noise, const float* u_cur, int ctas, int unit,
                             const int* masks01, float* out_batch, float* out_single) {
  const int T = g[6], N = g[7], M = g[8], rows = g[0], grid_rows = g[2], grid_cols = g[3], pitch = g[4], mpitch = g[5];
  const int npad = (N + 31) / 32 * 32;
  const size_t gs = (size_t)M * grid_rows * pitch, ms = (size_t)rows * mpitch;
  std::vector<std::vector<double2>> noiseT(K, std::vector<double2>((size_t)(T + 1) * npad, double2{0, 0}));
  std::vector<std::vector<float>> ctrl(K, std::vector<float>(npad, 0.0f));
  std::vector<std::vector<float>> dst(K, std::vector<float>((size_t)M * N, -1.0f));
  std::vector<RolloutWinArgs> d(K);
  std::vector<CUtensorMap> tm(4 * K);
  bool all01 = true;
  const int WW = WIN_WW, WH = (win_smem_layout(WIN_WW, 232, T).total + (int)sizeof(RolloutWinArgs) <= 232448) ? 232 : 224;
  if (WH != 232) return 1;
  for (int k = 0; k < K; ++k) {
    RolloutWinArgs& w = d[k];
    w = RolloutWinArgs{};
    emu::params(w.p, f + 23 * k, g, ratios + 2 * k, M);
    const RolloutParams& p = w.p;
    const float* nk = noise + (size_t)k * N * T * 2;
    const float* uk = u_cur + (size_t)k * T * 2;
    emu::launch({(unsigned)(npad / 32), 1, 1}, 256, [&] {
      prepare_rollout_kernel(reinterpret_cast<const float2*>(nk), uk, noiseT[k].data(), ctrl[k].data(), nullptr, N, T, npad,
                             p.lambda, p.u_std[0] * p.u_std[0], p.u_std[1] * p.u_std[1], p.vrange[0], p.vrange[1],
                             p.wrange[0], p.wrange[1]);
    });
    emu::win_place(w, WW, WH);
    w.npad = npad; w.masks01 = masks01[k];
    all01 = all01 && masks01[k];
    w.lin_grid = lin + k * gs; w.ang_grid = ang + k * gs; w.obstacle = obs + k * ms; w.unknown = unk + k * ms;
    w.noiseT = reinterpret_cast<const float*>(noiseT[k].data()); w.ctrl = ctrl[k].data(); w.u_cur = uk;
    w.dst.base[0] = dst[k].data(); w.dst.n_per = N; w.dst.ld = N; w.dst.row0 = 0;
    tm[4 * k + 0] = CUtensorMap{(const unsigned char*)w.lin_grid, grid_cols, grid_rows, M, pitch, WW, WH};
    tm[4 * k + 1] = CUtensorMap{(const unsigned char*)w.ang_grid, grid_cols, grid_rows, M, pitch, WW, WH};
    tm[4 * k + 2] = CUtensorMap{(const unsigned char*)w.obstacle, p.g.cols, p.g.rows, 1, mpitch, WW, WH};
    tm[4 * k + 3] = CUtensorMap{(const unsigned char*)w.unknown, p.g.cols, p.g.rows, 1, mpitch, WW, WH};
  }
  RolloutWinArgs ga = d[0];                                  // launch_rollout_win_batch: the launch-wide fields
  ga.unit = unit; ga.sync_passes = 0; ga.stagger = 0; ga.rotate = 0; ga.dbg = nullptr; ga.sig = CostSignal{};
  if (unit == 0 && ctas < K * M) return 2;
  if (all01) emu::launch({(unsigned)ctas, 1, 1}, 1024, [&] { rollout_win_batch_kernel<1024, 232, true>(ga, d.data(), tm.data(), K); });
  else emu::launch({(unsigned)ctas, 1, 1}, 1024, [&] { rollout_win_batch_kernel<1024, 232, false>(ga, d.data(), tm.data(), K); });
  for (int k = 0; k < K; ++k) {
    for (int n = 0; n < N; ++n)
      for (int m = 0; m < M; ++m) out_batch[((size_t)k * N + n) * M + m] = dst[k][(size_t)m * N + n];
    const int rc = emu_rollout_win(f + 23 * k, g, ratios + 2 * k, lin + k * gs, ang + k * gs, obs + k * ms, unk + k * ms,
                                   noise + (size_t)k * N * T * 2, u_cur + (size_t)k * T * 2, out_single + (size_t)k * N * M,
                                   0, 0, nullptr, nullptr, 0, 1, 0, 0, masks01[k]);
    if (rc) return 10 + rc;
  }
  return 0;
}
'''

CVAR_HARNESS = r'''
// K planners of equal N and M, each with its own numel: one batched launch against launch_cvar per planner
extern "C" int emu_cvar_batch(int K, const float* costs_mn, int N, int M, const int* numel, float* out_batch, float* out_single) {
  if (M > 32 * CVAR_MAX_PER_LANE) return 1;
  std::vector<CvarDesc> d(K);
  for (int k = 0; k < K; ++k) d[k] = CvarDesc{costs_mn + (size_t)k * M * N, out_batch + (size_t)k * N, N, N, M, numel[k]};
  const int nb = cvar_block_n(M);
  const unsigned blocks = (unsigned)((N + nb - 1) / nb);
  emu::cvar_per(M, [&](auto P) {
    for (int k = 0; k < K; ++k)
      emu::launch({blocks, 1, 1}, CVAR_THREADS, [&] {
        cvar_kernel<decltype(P)::value>(costs_mn + (size_t)k * M * N, out_single + (size_t)k * N, N, N, M, numel[k], FlagWait{});
      });
    emu::launch({blocks, (unsigned)K, 1}, CVAR_THREADS, [&] { cvar_batch_kernel<decltype(P)::value>(d.data()); });
  });
  return 0;
}
'''


def build(out_dir, extra="", cvar_extra=""):
    """(windowed-kernel library, CVaR library); ``extra`` / ``cvar_extra``: more harness text for either."""
    lib = _build(out_dir, "stochastic_batch_emu", emu_rollout_win.kernels(prep=("noise_prepare_batch",), win=("win_batch",)),
                 emu_rollout_win.HARNESS + HARNESS + extra)
    cvl = _build(out_dir, "cvar_batch_emu", emu_cvar.kernels("cvar_batch"), emu_cvar.HARNESS + CVAR_HARNESS + cvar_extra)
    return lib, cvl
