"""Host emulation of the batched stochastic kernels (TEST INFRASTRUCTURE): noise_prepare_batch_kernel and
rollout_win_batch_kernel (csrc/rollout_win.cu) next to their single-planner kernels, with the technique and the
hardware stand-ins of tests/emu_rollout_win.py (whose harness, emu_rollout_win included, is compiled in as the
single-planner reference); cvar_batch_kernel (csrc/rollout.cu) with those of tests/emu_cvar.py."""
import ctypes as C
import os
import re
import subprocess

from tests import emu_cvar, emu_rollout_win
from tests.emu_rollout import PRELUDE as ROLLOUT_PRELUDE
from tests.emu_rollout import _region

CSRC = emu_rollout_win.CSRC

HARNESS = r'''
// K planners of equal N, T: one batched noise + prepare launch (iteration `iter`) against one single launch per planner
extern "C" int emu_noise_prepare_batch(int K, const uint64_t* states_in, const float* u_cur, int N, int T, const float* fp,
                                       const int* slots, int iter) {
  using namespace b200;
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
  run([&] { noise_prepare_batch_kernel(d.data(), N, T, npad, iter); }, 256, (unsigned)(npad / NP_NB), (unsigned)K);
  for (int k = 0; k < K; ++k) {
    const float* q = fp + 7 * k;
    run([&] { noise_prepare_kernel(st2.data() + k * ns, reinterpret_cast<float2*>(noise2.data() + k * ns), u_cur + (size_t)k * T * 2,
                                   noiseT2.data() + k * nT, ctrl2.data() + k * npad, reach2.data() + 2 * k, slots[k] ^ (iter & 1),
                                   N, T, npad, q[0], q[1], q[2], q[0] * q[0], q[1] * q[1], q[3], q[4], q[5], q[6]); },
        256, (unsigned)(npad / NP_NB), 1);
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
  using namespace b200;
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
    w.p = params(f + 23 * k, g, ratios + 2 * k);
    const RolloutParams& p = w.p;
    const float* nk = noise + (size_t)k * N * T * 2;
    const float* uk = u_cur + (size_t)k * T * 2;
    run([&] { prepare_rollout_kernel(reinterpret_cast<const float2*>(nk), uk, noiseT[k].data(), ctrl[k].data(), nullptr, N, T, npad,
                                     p.lambda, p.u_std[0] * p.u_std[0], p.u_std[1] * p.u_std[1], p.vrange[0], p.vrange[1],
                                     p.wrange[0], p.wrange[1]); }, 256, (unsigned)(npad / 32), 1);
    // fill_win_args (api.cu)
    const int xi0 = (int)std::floor(((double)p.x0[0] - (double)p.g.xlo) / (double)p.g.res);
    const int yi0 = (int)std::floor(((double)p.x0[1] - (double)p.g.ylo) / (double)p.g.res);
    int cx = xi0 - WW / 2, cy = yi0 - WH / 2;
    cx = std::max(0, std::min(cx, p.g.cols - WW));
    cy = std::max(0, std::min(cy, p.g.rows - WH));
    w.WW = WW; w.WH = WH; w.wx0 = cx & ~15; w.wy0 = cy;
    w.ww = std::min(WW, p.g.cols - w.wx0); w.wh = std::min(WH, p.g.rows - w.wy0);
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
  if (all01) run([&] { rollout_win_batch_kernel<1024, 232, true>(ga, d.data(), tm.data(), K); }, 1024, (unsigned)ctas, 1);
  else run([&] { rollout_win_batch_kernel<1024, 232, false>(ga, d.data(), tm.data(), K); }, 1024, (unsigned)ctas, 1);
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
  using namespace b200;
  if (M > 32 * CVAR_MAX_PER_LANE) return 1;
  std::vector<CvarDesc> d(K);
  for (int k = 0; k < K; ++k) d[k] = CvarDesc{costs_mn + (size_t)k * M * N, out_batch + (size_t)k * N, N, N, M, numel[k]};
  const int nb = cvar_block_n(M), per = (M + 31) / 32;
  const unsigned blocks = (unsigned)((N + nb - 1) / nb);
  for (int k = 0; k < K; ++k) {
    auto single = [&](auto kern) {
      run([&] { kern(costs_mn + (size_t)k * M * N, out_single + (size_t)k * N, N, N, M, numel[k], FlagWait{}); }, CVAR_THREADS, blocks);
    };
    if (per <= 1) single(cvar_kernel<1>); else if (per <= 2) single(cvar_kernel<2>); else if (per <= 4) single(cvar_kernel<4>);
    else if (per <= 8) single(cvar_kernel<8>); else if (per <= 16) single(cvar_kernel<16>); else single(cvar_kernel<32>);
  }
  // the batched grid (blocks, K): planner = blockIdx.y
  auto batched = [&](auto kern) {
    for (int k = 0; k < K; ++k)
      run([&] { blockIdx.y = (unsigned)k; kern(d.data()); }, CVAR_THREADS, blocks);
  };
  if (per <= 1) batched(cvar_batch_kernel<1>); else if (per <= 2) batched(cvar_batch_kernel<2>);
  else if (per <= 4) batched(cvar_batch_kernel<4>); else if (per <= 8) batched(cvar_batch_kernel<8>);
  else if (per <= 16) batched(cvar_batch_kernel<16>); else batched(cvar_batch_kernel<32>);
  return 0;
}
'''


def _compile(src, out_dir, name, extra=()):
    cpp = os.path.join(out_dir, name + ".cpp")
    so = os.path.join(out_dir, "lib%s.so" % name)
    open(cpp, "w").write(src)
    r = subprocess.run(["g++", "-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-Wno-unknown-pragmas"] + list(extra) +
                       [cpp, "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-6000:]
    return C.CDLL(so)


def build(out_dir):
    cell = _region(os.path.join(CSRC, "common.cuh"), "cell_index")
    cell, n = re.subn(r'int k; asm\("cvt\.rzi\.ftz\.s32\.f32[^;]*;[^;]*;', "int k = (int)res;   /* cvt.rzi */", cell)
    assert n == 1
    win = os.path.join(CSRC, "rollout_win.cu")
    prep = (_region(os.path.join(CSRC, "common.cuh"), "xoro") + _region(os.path.join(CSRC, "common.cuh"), "normal") +
            _region(win, "prepare") + _region(win, "noise_prepare") + _region(win, "noise_prepare_batch"))
    prep = re.sub(r"(?m)^(\s*)__shared__ ", r"\1static ", prep)
    kern = _region(win, "win_kernel") + _region(win, "win_batch")
    kern, n = re.subn(r'(?m)^\s*asm volatile\("fence\.[^;]*;[^;]*;\n', "", kern)            # mbarrier / proxy fences
    assert n == 2, n
    kern, n = re.subn(r'asm volatile \("fence\.proxy\.tensormap[^;]*;[^;]*;', ";", kern)     # tensor-map acquire
    assert n == 1, n
    kern = kern.replace("extern __shared__ __align__(128) unsigned char smem[];", "")
    kh = os.path.join(CSRC, "kernels.h")
    src = (ROLLOUT_PRELUDE.replace("float s_u[4096];", "") + emu_rollout_win.EXTRA +
           _region(os.path.join(CSRC, "common.cuh"), "params") + cell + _region(kh, "cost_dst") + _region(kh, "win_args") +
           _region(kh, "noise_prep_desc") + prep + kern + emu_rollout_win.HARNESS + HARNESS)
    lib = _compile(src, out_dir, "stochastic_batch_emu", ["-ffp-contract=off"])
    P, I = C.c_void_p, C.c_int
    lib.emu_noise_prepare_batch.restype = I
    lib.emu_noise_prepare_batch.argtypes = [I, P, P, I, I, P, P, I]
    lib.emu_win_batch.restype = I
    lib.emu_win_batch.argtypes = [I, P, P, P, P, P, P, P, P, P, I, I, P, P, P]
    rollout = os.path.join(CSRC, "rollout.cu")
    cv = _region(rollout, "cvar") + _region(rollout, "cvar_batch")
    cv = re.sub(r"(?m)^(\s*)__shared__ ", r"\1static ", cv)
    cv_src = (emu_cvar.PRELUDE + _region(kh, "cvar_desc") + _region(os.path.join(CSRC, "common.cuh"), "warp_sum") + cv +
              emu_cvar.HARNESS + CVAR_HARNESS)
    cvl = _compile(cv_src, out_dir, "cvar_batch_emu")
    cvl.emu_cvar_batch.restype = I
    cvl.emu_cvar_batch.argtypes = [I, P, I, I, P, P, P]
    return lib, cvl
