"""Host emulation of the batched one-map kernels (TEST INFRASTRUCTURE; technique of tests/emu_sampler.py).  The kernel
text of the noise, rollout, update and sampler regions of csrc/*.cu -- the single-planner kernels AND their batched
wrappers (``[emu:... *_batch]``) -- is compiled with g++ against the preludes of the existing emulators, with a launch
loop over blockIdx.y / blockIdx.z.  Each library runs either K single launches or ONE batched launch of the same
emulated code, so the CPU suite checks the descriptor plumbing and the grid-coordinate indexing of the batched
kernels bit for bit."""
import ctypes as C
import os
import re
import subprocess

from tests import emu_noise, emu_rollout, emu_sampler, emu_update
from tests.emu_rollout import _region

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mppi_numba_b200", "csrc")


def _src(name, region):
    return _region(os.path.join(CSRC, name), region)


def _compile(out_dir, stem, src, std="c++20", extra=()):
    cpp, so = os.path.join(out_dir, stem + ".cpp"), os.path.join(out_dir, "lib" + stem + ".so")
    open(cpp, "w").write(src)
    cmd = ["g++", "-O1", "-std=" + std, "-pthread", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-ffp-contract=off",
           cpp, "-o", so] + list(extra)
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return C.CDLL(so)


# ----------------------------------------------------------------------------- noise
NOISE_HARNESS = r'''
}  // namespace b200
// K planners: batched != 0 -> ONE launch over blockIdx.y, else K single launches of sample_noise_kernel
extern "C" void emu_noise(int K, int batched, uint64_t** states, float** noise, const float* std, long long count) {
  using namespace b200;
  std::vector<NoiseDesc> d(K);
  for (int i = 0; i < K; ++i) d[i] = NoiseDesc{states[i], noise[i], std[2 * i], std[2 * i + 1]};
  blockDim = {256, 1, 1};
  const long long padded = (count + 255) / 256 * 256;
  for (int i = 0; i < K; ++i)
    for (long long g = 0; g < padded; ++g) {
      blockIdx = {(unsigned)(g / 256), batched ? (unsigned)i : 0u, 0}; threadIdx = {(unsigned)(g % 256), 0, 0};
      if (batched) sample_noise_batch_kernel(d.data(), count);
      else sample_noise_kernel(states[i], reinterpret_cast<float2*>(noise[i]), count, std[2 * i], std[2 * i + 1], nullptr);
    }
}
'''


def build_noise(out_dir):
    src = ("#include <vector>\n" + emu_noise.PRELUDE + _src("common.cuh", "xoro") + _src("common.cuh", "normal") + _src("reduce.cu", "noise") +
           _src("kernels.h", "noise_desc") + _src("reduce.cu", "noise_batch") + NOISE_HARNESS)
    lib = _compile(out_dir, "noise_batch_emu", src, std="c++17")
    P = C.c_void_p
    lib.emu_noise.restype = None
    lib.emu_noise.argtypes = [C.c_int, C.c_int, P, P, P, C.c_longlong]
    return lib


# ----------------------------------------------------------------------------- rollout (modes 1, 2, 3)
ROLLOUT_HARNESS = r'''
template <class K>
static void run(K kernel, int threads, unsigned gx, unsigned gy) {
  for (unsigned by = 0; by < gy; ++by)
    for (unsigned bx = 0; bx < gx; ++bx) {
      std::barrier<> bar(threads);
      g_bar = &bar;
      std::vector<std::thread> th;
      for (int t = 0; t < threads; ++t)
        th.emplace_back([&, t] {
          threadIdx = {(unsigned)t, 0, 0}; blockIdx = {bx, by, 0}; blockDim = {(unsigned)threads, 1, 1}; gridDim = {gx, gy, 1};
          kernel();
        });
      for (auto& x : th) x.join();
    }
}
static RolloutParams params(const float* f, const int* g, const double* ratios) {
  RolloutParams p{};
  p.g.res = f[0]; p.g.inv_res = 1.0f / f[0]; p.g.xlo = f[1]; p.g.ylo = f[2];
  p.g.rows = g[0]; p.g.cols = g[1]; p.g.grid_rows = g[2]; p.g.grid_cols = g[3]; p.g.grid_pitch = g[4]; p.g.mask_pitch = g[5];
  p.dt = f[3]; p.x0[0] = f[4]; p.x0[1] = f[5]; p.x0[2] = f[6]; p.xgoal[0] = f[7]; p.xgoal[1] = f[8];
  p.tol2 = f[9] * f[9]; p.v_post = f[10]; p.lambda = f[11]; p.u_std[0] = f[12]; p.u_std[1] = f[13];
  p.vrange[0] = f[14]; p.vrange[1] = f[15]; p.wrange[0] = f[16]; p.wrange[1] = f[17];
  p.obs_cost = f[18]; p.unk_cost = f[19]; p.dist_weight = f[20]; p.lin_lo = f[21]; p.ang_lo = f[22];
  p.lin_ratio = ratios[0]; p.ang_ratio = ratios[1];
  p.T = g[6]; p.N = g[7]; p.M = 1;
  return p;
}
}  // namespace b200

// planner i: f[23 i ..], g[9 i ..] as tests/emu_rollout.py, ratios[2 i ..]; per-planner buffers as pointer arrays
extern "C" void emu_rollout(int K, int batched, int mode, const float* f, const int* g, const double* ratios,
                            const int8_t** lin, const int8_t** ang, const int8_t** obs, const int8_t** unk,
                            const int8_t** risk, const float** noise, const float** u_cur, float** costs,
                            const float** obstacles, const int* num_obstacles) {
  using namespace b200;
  std::vector<RolloutArgs> d(K);
  for (int i = 0; i < K; ++i) {
    RolloutArgs a{};
    a.p = params(f + 23 * i, g + 9 * i, ratios + 2 * i);
    a.mode = mode; a.lin_grid = lin[i]; a.ang_grid = ang[i]; a.obstacle = obs[i]; a.unknown = unk[i]; a.risk = risk[i];
    a.noise = noise[i]; a.u_cur = u_cur[i]; a.costs = costs[i]; a.obstacles = obstacles[i];
    a.num_obstacles = num_obstacles[i];
    d[i] = a;
  }
  const int threads = 128;
  const unsigned gx = (unsigned)((d[0].p.N + threads - 1) / threads);
  if (batched) {
    if (mode == 1) run([&] { rollout_batch_kernel<1>(d.data()); }, threads, gx, (unsigned)K);
    else if (mode == 2) run([&] { rollout_batch_kernel<2>(d.data()); }, threads, gx, (unsigned)K);
    else run([&] { rollout_batch_kernel<3>(d.data()); }, threads, gx, (unsigned)K);
    return;
  }
  for (int i = 0; i < K; ++i) {
    const RolloutArgs a = d[i];
    if (mode == 1) run([&] { rollout_kernel<1>(a); }, threads, gx, 1);
    else if (mode == 2) run([&] { rollout_kernel<2>(a); }, threads, gx, 1);
    else run([&] { rollout_barebone_kernel(a); }, threads, gx, 1);
  }
}
'''


def build_rollout(out_dir):
    cell = _src("common.cuh", "cell_index")
    cell, n = re.subn(r'int k; asm\("cvt\.rzi\.ftz\.s32\.f32[^;]*;[^;]*;', "int k = (int)res;   /* cvt.rzi */", cell)
    assert n == 1
    kernels = (_src("rollout.cu", "rollout") + _src("rollout.cu", "rollout_batch")).replace(
        "extern __shared__ float s_u[];", "")
    src = (emu_rollout.PRELUDE + _src("common.cuh", "params") + cell + _src("kernels.h", "cost_dst") +
           _src("kernels.h", "rollout_args") + kernels + ROLLOUT_HARNESS)
    lib = _compile(out_dir, "rollout_batch_emu", src)
    P, I = C.c_void_p, C.c_int
    lib.emu_rollout.restype = None
    lib.emu_rollout.argtypes = [I, I, I, P, P, P] + [P] * 10
    return lib


# ----------------------------------------------------------------------------- update (UPD_TAIL_APPLY)
UPDATE_HARNESS = r'''
template <class K>
static void run(K kernel, int threads, unsigned gx, unsigned gy) {
  for (unsigned by = 0; by < gy; ++by)
    for (unsigned bx = 0; bx < gx; ++bx) {
      std::barrier<> bar(threads);
      g_bar = &bar;
      std::vector<std::unique_ptr<EmuWarp>> warps;
      for (int w = 0; w < threads / 32; ++w) warps.emplace_back(new EmuWarp());
      std::vector<std::thread> th;
      for (int t = 0; t < threads; ++t)
        th.emplace_back([&, t] {
          threadIdx = {(unsigned)t, 0, 0}; blockIdx = {bx, by, 0}; blockDim = {(unsigned)threads, 1, 1}; gridDim = {gx, gy, 1};
          g_warp = warps[t / 32].get();
          kernel();
        });
      for (auto& x : th) x.join();
    }
}
}  // namespace b200

// planner i: costs / noise / w_raw / cta_partials / rank_partial / u_cur / weights / u_prev / u_out buffers, lambda[i],
// ranges vr[2 i], wr[2 i]; batched: ONE launch over blockIdx.y, else K single launches (u_prev / u_out unset: the
// single-planner path's tail, whose u_prev the caller then copies as after_u_update does).  Returns the sum of the
// ticket counters left behind (0: every planner's counter is reset for the next launch).
extern "C" int emu_update(int K, int batched, const float** costs, const float** noise, float** w_raw, float** parts,
                          float** rank_partial, float** u_cur, float** weights, float** u_prev, float** u_out, int N,
                          int T, const float* lambda, const float* vr, const float* wr) {
  using namespace b200;
  std::vector<UpdateBatchDesc> d(K);
  std::vector<unsigned> counters(K, 0);
  int ctas = (N + 31) / 32;                       // update_num_ctas + the planner's rows_per_cta rule (api.cu)
  if (ctas > 296) ctas = 296;
  if (ctas < 1) ctas = 1;
  const int rows_per_cta = (N + ctas - 1) / ctas;
  ctas = (N + rows_per_cta - 1) / rows_per_cta;
  for (int i = 0; i < K; ++i) {
    UpdateArgs a{};
    a.costs = costs[i]; a.noise = noise[i]; a.w_raw = w_raw[i]; a.cta_partials = parts[i]; a.rank_partial = rank_partial[i];
    a.u_cur = u_cur[i]; a.weights = weights[i]; a.N = N; a.T = T; a.num_ctas = ctas; a.rows_per_cta = rows_per_cta;
    a.lambda = lambda[i]; a.vrange[0] = vr[2 * i]; a.vrange[1] = vr[2 * i + 1]; a.wrange[0] = wr[2 * i]; a.wrange[1] = wr[2 * i + 1];
    UpdateTail tl{};
    tl.counter = &counters[i]; tl.mode = UPD_TAIL_APPLY;
    if (batched) { tl.u_prev = u_prev[i]; tl.u_out = u_out[i]; }
    d[i] = UpdateBatchDesc{a, tl};
  }
  if (batched) {
    run([&] { update_partial_batch_kernel(d.data()); }, UPD_THREADS, (unsigned)ctas, (unsigned)K);
  } else {
    for (int i = 0; i < K; ++i) {
      const UpdateArgs a = d[i].a;
      const UpdateTail tl = d[i].tl;
      run([&] { update_partial_kernel(a, tl); }, UPD_THREADS, (unsigned)ctas, 1);
    }
  }
  int left = 0;
  for (unsigned c : counters) left += (int)c;
  return left;
}
'''


def build_update(out_dir):
    kernels = _src("reduce.cu", "update") + _src("reduce.cu", "update_batch")
    kernels = re.sub(r"(?m)^(\s*)__shared__ ", r"\1static ", kernels)      # block-shared arrays: one instance
    kernels = kernels.replace("int update_num_ctas(int N) {", "static int update_num_ctas_unused(int N) {")
    src = (emu_update.PRELUDE + "constexpr int P2P_MAX_PEERS = 16;\n" + _src("kernels.h", "update_args") +
           _src("kernels.h", "update_tail") + _src("kernels.h", "update_desc") + _src("common.cuh", "warp_min") +
           _src("common.cuh", "warp_sum") + kernels + UPDATE_HARNESS)
    lib = _compile(out_dir, "update_batch_emu", src)
    P, I = C.c_void_p, C.c_int
    lib.emu_update.restype = I
    lib.emu_update.argtypes = [I, I] + [P] * 9 + [I, I, P, P, P]
    return lib


# ----------------------------------------------------------------------------- sampler (fused lin + ang, whole maps)
SAMPLER_HARNESS = r'''
bool build_sample_thresholds(double alpha, int q_cap, uint64_t* table);

template <class Kern>
static void run(Kern kernel, int threads, unsigned gx, unsigned gy, unsigned gz) {
  for (unsigned bz = 0; bz < gz; ++bz)
    for (unsigned by = 0; by < gy; ++by)
      for (unsigned bx = 0; bx < gx; ++bx) {
        std::barrier<> bar(threads);
        g_bar = &bar;
        std::vector<std::thread> th;
        for (int t = 0; t < threads; ++t)
          th.emplace_back([&, t] {
            threadIdx = {(unsigned)t, 0, 0}; blockIdx = {bx, by, bz}; blockDim = {(unsigned)threads, 1, 1};
            gridDim = {gx, gy, gz};
            kernel();
          });
        for (auto& x : th) x.join();
      }
}
template <int NW>
static void go(int K, int batched, const std::vector<SampleGridsV2Args>& d, int threads, unsigned gx, unsigned gy) {
  if (batched) { run([&] { sample_grids_v2_batch_kernel<2, NW>(d.data()); }, threads, gx, gy, (unsigned)K); return; }
  for (int i = 0; i < K; ++i) {
    const SampleGridsV2Args a = d[i];
    run([&] { sample_grids_v2_kernel<2, NW>(a); }, threads, gx, gy, 1);
  }
}
}  // namespace b200

// pair i: grids g0[i] / g1[i] (grid_rows, pitch), cumulative tables c0[i] / c1[i], ONE set of generator states st[i]
// (fused: both TDMs hold the same states) -> so0[i] / so1[i], value tables q0[i] / q1[i]; one geometry for all pairs
extern "C" int emu_sampler(int K, int batched, int8_t** g0, int8_t** g1, const int8_t** c0, const int8_t** c1,
                           const uint64_t** st, uint64_t** so0, uint64_t** so1, const int8_t** q0, const int8_t** q1,
                           int bpad, int rows, int cols, int grid_rows, int pitch, int tx, int ty, int segs, double alpha,
                           int q_cap) {
  using namespace b200;
  std::vector<uint64_t> T(SAMPLE_TABLE_WORDS);
  if (!build_sample_thresholds(alpha, q_cap, T.data())) return 1;
  const int nrow = (rows + tx - 1) / tx, ncol = (cols + ty - 1) / ty;
  if (segs > nrow) segs = nrow;
  if (segs < 1) segs = 1;
  const int seg_rows = (nrow + segs - 1) / segs;
  std::vector<uint64_t> J(256);
  if (segs > 1) {                      // as tdm_prepare_jump (api.cu)
    int last_w = cols - (ty - 1) * ncol;
    for (int iy = ty - 1; iy >= 0 && last_w <= 0; --iy) last_w = cols - iy * ncol;
    if (last_w > ncol) last_w = ncol;
    if (last_w < 0) last_w = 0;
    std::vector<int64_t> ks;
    for (int s = 1; s < segs; ++s) { ks.push_back((int64_t)s * seg_rows * ncol); ks.push_back((int64_t)s * seg_rows * last_w); }
    J.resize(ks.size() * 256);
    build_jump_matrices(ks.data(), (int)ks.size(), J.data());
  }
  std::vector<SampleGridsV2Args> d(K);
  for (int i = 0; i < K; ++i) {
    SampleGridsV2Args a{};
    a.t[0] = SampleTdm{g0[i], c0[i], st[i], so0[i], q0[i], bpad};
    a.t[1] = SampleTdm{g1[i], c1[i], st[i], so1[i], q1[i], bpad};
    a.thresholds = T.data(); a.jump = J.data();
    a.rows = rows; a.cols = cols; a.grid_rows = grid_rows; a.pitch = pitch; a.tx = tx; a.ty = ty; a.num_maps = 1;
    a.segs = segs; a.seg_rows = seg_rows;
    sample_box_full(a);
    if (a.ty * a.gm > 256) a.gm = 256 / a.ty;
    d[i] = a;
  }
  const int threads = ((d[0].nact * d[0].gm + 31) / 32) * 32;
  if (threads > 256 || d[0].gm < 1) return 3;
  const int tix_hi = std::min(tx - 1, (rows - 1) / nrow);               // launch_v2_nt (sample.cu)
  const unsigned gx = (unsigned)((tix_hi + 1) * segs), gy = (unsigned)((1 + d[0].gm - 1) / d[0].gm);
  const int nw = bpad / 4;
  if (nw == 3) go<3>(K, batched, d, threads, gx, gy);
  else if (nw == 8) go<8>(K, batched, d, threads, gx, gy);
  else if (nw == 1) go<1>(K, batched, d, threads, gx, gy);
  else go<0>(K, batched, d, threads, gx, gy);
  return 0;
}
'''


def build_sampler(out_dir):
    src = (emu_sampler.PRELUDE + _src("kernels.h", "sampler_args") + _src("common.cuh", "xoro") +
           _src("common.cuh", "threshold") + _src("sample.cu", "sampler_v2") + _src("sample.cu", "sampler_batch") +
           SAMPLER_HARNESS)
    libdir = os.path.join(ROOT, "mppi_numba_b200")
    lib = _compile(out_dir, "sampler_batch_emu", src,
                   extra=["-L" + libdir, "-l:libb200mppi.so", "-Wl,-rpath," + libdir])
    P, I = C.c_void_p, C.c_int
    lib.emu_sampler.restype = I
    lib.emu_sampler.argtypes = [I, I] + [P] * 9 + [I] * 8 + [C.c_double, I]
    return lib
