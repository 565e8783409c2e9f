"""Host emulation of the windowed (TMA-staged) stochastic rollout kernel and its prepare kernel (TEST
INFRASTRUCTURE; technique of tests/emu_sampler.py).  The kernels' text is lifted from csrc/rollout_win.cu between
the ``[emu:... prepare]`` / ``[emu:... win_kernel]`` markers.  What stands in for the hardware: a CUtensorMap is a
plain descriptor (base, dims, pitch, box) and ``tma_load_2d/3d`` copy the box with zero fill outside the tensor
(what CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE does for integer types); mbarrier calls are no-ops (the copy is done when
the call returns); shared-space addresses are offsets into one static buffer; ``__fadd_rd`` is a round-down add
derived from the rounded sum and its exact error (TwoSum); 1024 std::threads stand for the CTA.  Arithmetic helpers as in
tests/emu_rollout.py (IEEE meaning; libm for the MUFU approximations)."""
import ctypes as C
import os
import re
import subprocess

from tests.emu_rollout import PRELUDE as ROLLOUT_PRELUDE
from tests.emu_rollout import _region

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mppi_numba_b200", "csrc")

EXTRA = r'''
struct CUtensorMap { const unsigned char* base; int cols, rows, maps, pitch, WW, WH; };
struct double2 { double x, y; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline int __double2loint(double d) { uint64_t u; std::memcpy(&u, &d, 8); return (int)(uint32_t)u; }
static inline int __double2hiint(double d) { uint64_t u; std::memcpy(&u, &d, 8); return (int)(uint32_t)(u >> 32); }
static inline double __hiloint2double(int hi, int lo) {
  const uint64_t u = ((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo; double d; std::memcpy(&d, &u, 8); return d;
}
static inline float __fadd_rd(float a, float b) {           // add.rm.f32 from the round-to-nearest sum + its exact error
  volatile float s = a + b;                                 // (TwoSum; volatile: no re-association, no excess precision)
  volatile float bb = s - a;
  volatile float e1 = a - (s - bb), e2 = b - bb;
  const float err = e1 + e2;                                // exact: a + b == s + err
  return (err < 0.0f) ? std::nextafterf(s, -INFINITY) : (float)s;
}
static inline float __fadd_ru(float a, float b) {           // add.rp.f32, same construction
  volatile float s = a + b;
  volatile float bb = s - a;
  volatile float e1 = a - (s - bb), e2 = b - bb;
  const float err = e1 + e2;
  return (err > 0.0f) ? std::nextafterf(s, INFINITY) : (float)s;
}
static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
static inline unsigned atomicMax(unsigned* p, unsigned v) { const unsigned o = *p; if (v > o) *p = v; return o; }   // blocks run one by one
struct EmuWarp { std::barrier<> bar{32}; float fbuf[32]; int ibuf[32]; };     // warp collectives: exchange between two warp barriers
static EmuWarp g_warps[32];
static inline float __shfl_xor_sync(unsigned, float v, int o) {
  EmuWarp& w = g_warps[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  w.fbuf[lane] = v;
  w.bar.arrive_and_wait();
  const float r = w.fbuf[lane ^ o];
  w.bar.arrive_and_wait();
  return r;
}
static inline int __shfl_sync(unsigned, int v, int src) {
  EmuWarp& w = g_warps[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  w.ibuf[lane] = v;
  w.bar.arrive_and_wait();
  const int r = w.ibuf[src];
  w.bar.arrive_and_wait();
  return r;
}
static inline int __reduce_max_sync(unsigned, int v) {
  EmuWarp& w = g_warps[threadIdx.x >> 5];
  w.ibuf[threadIdx.x & 31] = v;
  w.bar.arrive_and_wait();
  int r = w.ibuf[0];
  for (int i = 1; i < 32; ++i) r = w.ibuf[i] > r ? w.ibuf[i] : r;
  w.bar.arrive_and_wait();
  return r;
}
static inline long long clock64() { return 0; }
static inline unsigned long long globaltimer_ns() { return 0; }
static inline unsigned sm_id() { return 0; }
static inline void keep_in_registers(float&, float&) {}
#define VELTKAMP_C 536870913.0
static inline unsigned __activemask() { return 0xffffffffu; }
static inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T __ldcg(const T* p) { return *p; }
static inline void __threadfence_system() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void st_flag_sys(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
struct ulonglong2 { unsigned long long x, y; };
static inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { return ulonglong2{x, y}; }
static inline float xoro_unit_f32(uint64_t x) { return (float)((double)(x >> 11) * (1.0 / 9007199254740992.0)); }
#define __grid_constant__
#define __align__(n)
#undef __launch_bounds__
#define __launch_bounds__(...)
alignas(128) unsigned char smem[1 << 18];
static inline uint32_t smem_u32(const void* p) { return (uint32_t)((const unsigned char*)p - smem); }
static inline void mbar_init(uint64_t*, int) {}
static inline void mbar_expect_tx(uint64_t*, uint32_t) {}
static inline void mbar_wait(uint64_t*, uint32_t) {}
static inline void tma_box(unsigned char* dst, const CUtensorMap* tm, int c0, int c1, int c2) {
  for (int y = 0; y < tm->WH; ++y)
    for (int x = 0; x < tm->WW; ++x) {
      const int gx = c0 + x, gy = c1 + y;
      const bool in = gx >= 0 && gx < tm->cols && gy >= 0 && gy < tm->rows && c2 >= 0 && c2 < tm->maps;
      dst[y * tm->WW + x] = in ? tm->base[((size_t)c2 * tm->rows + gy) * tm->pitch + gx] : 0;
    }
}
static inline void tma_load_3d(void* dst, const CUtensorMap* tm, uint64_t*, int c0, int c1, int c2) { tma_box((unsigned char*)dst, tm, c0, c1, c2); }
static inline void tma_load_2d(void* dst, const CUtensorMap* tm, uint64_t*, int c0, int c1) { tma_box((unsigned char*)dst, tm, c0, c1, 0); }
static inline int lds_s8(uint32_t addr, int imm_plane) { return (int)(int8_t)smem[addr + (uint32_t)imm_plane]; }
static inline double lds_f64(uint32_t addr) { double v; std::memcpy(&v, smem + addr, 8); return v; }
static inline double widen(float a) { return (double)a; }
static inline float narrow(double a) { return (float)a; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }

'''

HARNESS = r'''
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
  p.T = g[6]; p.N = g[7]; p.M = g[8];
  return p;
}
}  // namespace b200

// stage_rollout of csrc/api.cu for MODE_TDM: prepare kernel, window origin, launch geometry of launch_rollout_win.
// shift_x / shift_y move the window away from the robot (cells) to force the global-memory path.
// The fused noise + controls kernel (launch_noise_prepare) next to the two kernels it replaces (sample_noise_kernel
// is restated here as its one-line body: generator g -> (std_v * normal, std_w * normal), tests/emu_noise.py runs the
// real one): states, noise, transposed controls, control costs and the reach statistic must agree bit for bit.
extern "C" int emu_noise_prepare(const uint64_t* states_in, const float* u_cur, int N, int T, float std_v, float std_w,
                                 float lambda, const float* vr, const float* wr, uint64_t* states_out, float* noise_out,
                                 double* noiseT_out, float* ctrl_out, float* reach_out) {
  using namespace b200;
  const int npad = (N + 31) / 32 * 32;
  std::vector<uint64_t> st((size_t)N * T * 2);
  std::memcpy(st.data(), states_in, st.size() * 8);
  std::vector<float> noise((size_t)N * T * 2, 0.0f), ctrl(npad, 0.0f);
  std::vector<double2> noiseT((size_t)T * npad, double2{0, 0});
  float reach[2] = {0.0f, 123.0f};
  run([&] { noise_prepare_kernel(st.data(), reinterpret_cast<float2*>(noise.data()), u_cur, noiseT.data(), ctrl.data(), reach, 0,
                                 N, T, npad, std_v, std_w, lambda, std_v * std_v, std_w * std_w, vr[0], vr[1], wr[0], wr[1]); },
      256, (unsigned)(npad / NP_NB), 1);
  if (reach[1] != 0.0f) return 1;                                  // the other slot is cleared for the next launch
  // the two separate kernels
  std::vector<uint64_t> st2((size_t)N * T * 2);
  std::memcpy(st2.data(), states_in, st2.size() * 8);
  std::vector<float> noise2((size_t)N * T * 2, 0.0f), ctrl2(npad, 0.0f);
  std::vector<double2> noiseT2((size_t)T * npad, double2{0, 0});
  for (size_t g = 0; g < (size_t)N * T; ++g) {
    Xoro s{st2[2 * g], st2[2 * g + 1]};
    noise2[2 * g] = fmul(std_v, xoro_normal(s));
    noise2[2 * g + 1] = fmul(std_w, xoro_normal(s));
    st2[2 * g] = s.s0; st2[2 * g + 1] = s.s1;
  }
  float reach2 = 0.0f;
  run([&] { prepare_rollout_kernel(reinterpret_cast<const float2*>(noise2.data()), u_cur, noiseT2.data(), ctrl2.data(), &reach2,
                                   N, T, npad, lambda, std_v * std_v, std_w * std_w, vr[0], vr[1], wr[0], wr[1]); },
      256, (unsigned)(npad / 32), 1);
  if (std::memcmp(st.data(), st2.data(), st.size() * 8)) return 2;
  if (std::memcmp(noise.data(), noise2.data(), noise.size() * 4)) return 3;
  if (std::memcmp(noiseT.data(), noiseT2.data(), noiseT.size() * 16)) return 4;
  if (std::memcmp(ctrl.data(), ctrl2.data(), ctrl.size() * 4)) return 5;
  if (reach[0] != reach2) return 6;
  std::memcpy(states_out, st.data(), st.size() * 8);
  std::memcpy(noise_out, noise.data(), noise.size() * 4);
  std::memcpy(noiseT_out, noiseT.data(), noiseT.size() * 16);
  std::memcpy(ctrl_out, ctrl.data(), ctrl.size() * 4);
  *reach_out = reach[0];
  return 0;
}

// cell_from_interval (the division-free decision of the rare path) against the reference's exact sequence:
// out_new[i] = the kernel's result for a[i] (magic-number floors of the interval's ends, then cell_from_interval),
// out_ref[i] = cell_index_exact(a[i], res); differ[i] = 1 when the floors differed (the decision ran)
extern "C" void emu_cell_between(const float* a, int n, float res, int* out_new, int* out_ref, int* differ) {
  using namespace b200;
  const float inv_res = 1.0f / res;
  const float inv_lo = inv_res * (1.0f - 2.4e-7f), inv_hi = inv_res * (1.0f + 2.4e-7f);
  const float MAGIC = 12582912.0f;
  for (int i = 0; i < n; ++i) {
    const float k = __fadd_rd(fmaf(a[i], inv_lo, -1e-30f), MAGIC), k2 = __fadd_rd(fmaf(a[i], inv_hi, 1e-30f), MAGIC);
    differ[i] = __float_as_int(k) != __float_as_int(k2);
    out_new[i] = cell_from_interval(a[i], res, k, k2);
    out_ref[i] = cell_index_exact(a[i], res);
  }
}

// ctas: number of persistent CTAs (0: launch_rollout_win's own rule for a 132-SM device, an H100 SXM).
// dst_blocks: 1 = one map-major (M, N) destination; ws > 1 = the sharded layout, ws separate (ws*M, N/ws) "receive
// buffers" written at the rows of "rank" 1 (fill_cost_dst with direct = true) plus the epoch flags of CostSignal --
// checked here; costs_nm always comes back as the logical (N, M) array.
extern "C" int emu_rollout_win(const float* f, const int* g, const double* ratios, const int8_t* lin, const int8_t* ang,
                               const int8_t* obs, const int8_t* unk, const float* noise, const float* u_cur,
                               float* costs_nm, int shift_x, int shift_y, int* origin_out, float* reach_out, int ctas,
                               int dst_blocks, int unit_override, int sync_passes, int masks01) {
  using namespace b200;
  RolloutWinArgs w{};
  w.p = params(f, g, ratios);
  const RolloutParams& p = w.p;
  const int npad = (p.N + 31) / 32 * 32;
  std::vector<double2> noiseT((size_t)(p.T + 1) * npad, double2{0, 0});      // + 1 row: the kernel prefetches unguarded
  std::vector<float> ctrl(npad, 0.0f);
  float reach = 0.0f;
  run([&] { prepare_rollout_kernel(reinterpret_cast<const float2*>(noise), u_cur, noiseT.data(), ctrl.data(), &reach, p.N, p.T, npad,
                                   p.lambda, p.u_std[0] * p.u_std[0], p.u_std[1] * p.u_std[1], p.vrange[0], p.vrange[1],
                                   p.wrange[0], p.wrange[1]); }, 256, (unsigned)(npad / 32), 1);
  const int WW = WIN_WW, WH = (win_smem_layout(WIN_WW, 232, p.T).total <= 232448) ? 232 : 224;
  if (WH != 232) return 1;
  const int xi0 = (int)std::floor(((double)p.x0[0] - (double)p.g.xlo) / (double)p.g.res);
  const int yi0 = (int)std::floor(((double)p.x0[1] - (double)p.g.ylo) / (double)p.g.res);
  int cx = xi0 - WW / 2 + shift_x, cy = yi0 - WH / 2 + shift_y;
  cx = std::max(0, std::min(cx, p.g.cols - WW));              // stage_rollout (api.cu): the window stays inside the map
  cy = std::max(0, std::min(cy, p.g.rows - WH));
  w.WW = WW; w.WH = WH;
  w.wx0 = cx & ~15;
  w.wy0 = cy;
  w.ww = std::min(WW, p.g.cols - w.wx0);
  w.wh = std::min(WH, p.g.rows - w.wy0);
  w.npad = npad;
  w.lin_grid = lin; w.ang_grid = ang; w.obstacle = obs; w.unknown = unk;
  w.noiseT = reinterpret_cast<const float*>(noiseT.data()); w.ctrl = ctrl.data(); w.u_cur = u_cur;
  const int ws = dst_blocks < 1 ? 1 : dst_blocks;
  if (p.N % ws) return 4;
  const int n_per = p.N / ws, rank = ws > 1 ? 1 : 0;
  std::vector<std::vector<float>> recv(ws, std::vector<float>((size_t)ws * p.M * n_per, -1.0f));
  std::vector<std::vector<uint32_t>> flags(ws, std::vector<uint32_t>(ws, 0u));
  unsigned counter = 0;
  w.dst.n_per = n_per; w.dst.ld = n_per; w.dst.row0 = rank * p.M;
  for (int d = 0; d < ws; ++d) { w.dst.base[d] = recv[d].data(); w.sig.peer_flags[d] = flags[d].data(); }
  w.sig.ws = ws > 1 ? ws : 0; w.sig.rank = rank; w.sig.counter = &counter; w.sig.epoch = 7u;
  if (origin_out) { origin_out[0] = w.wx0; origin_out[1] = w.wy0; }
  if (reach_out) *reach_out = reach;
  const CUtensorMap t_lin{(const unsigned char*)lin, p.g.grid_cols, p.g.grid_rows, p.M, p.g.grid_pitch, WW, WH};
  const CUtensorMap t_ang{(const unsigned char*)ang, p.g.grid_cols, p.g.grid_rows, p.M, p.g.grid_pitch, WW, WH};
  const CUtensorMap t_obs{(const unsigned char*)obs, p.g.cols, p.g.rows, 1, p.g.mask_pitch, WW, WH};
  const CUtensorMap t_unk{(const unsigned char*)unk, p.g.cols, p.g.rows, 1, p.g.mask_pitch, WW, WH};
  if (ctas <= 0) {                                            // launch_rollout_win (rollout_win.cu)
    const long long total = (long long)p.M * (npad / 32);
    ctas = (int)std::min<long long>(std::max<long long>(total / 8, 1), 132);
  }
  w.unit = ((long long)p.M * (npad / 32) / (32LL * ctas) >= 1) ? 32 : 1;     // launch_rollout_win
  if (unit_override > 0) w.unit = unit_override;
  if (unit_override < 0) w.unit = 0;                         // shares by map (needs ctas >= M)
  w.sync_passes = sync_passes;
  w.masks01 = masks01;
  if (masks01) run([&] { rollout_win_kernel<1024, 232, true>(w, t_lin, t_ang, t_obs, t_unk); }, 1024, (unsigned)ctas, 1);
  else run([&] { rollout_win_kernel<1024, 232, false>(w, t_lin, t_ang, t_obs, t_unk); }, 1024, (unsigned)ctas, 1);
  for (int n = 0; n < p.N; ++n)
    for (int m = 0; m < p.M; ++m)
      costs_nm[(size_t)n * p.M + m] = recv[n / n_per][((size_t)rank * p.M + m) * n_per + n % n_per];
  if (ws > 1) {
    if (counter != 0) return 5;
    for (int d = 0; d < ws; ++d)
      for (int r = 0; r < ws; ++r)
        if (flags[d][r] != (r == rank ? 7u : 0u)) return 6;           // exactly this rank's flag, in every peer
    for (int d = 0; d < ws; ++d)                                      // rows of the other "ranks" untouched
      for (int r = 0; r < ws; ++r)
        if (r != rank)
          for (size_t i = 0; i < (size_t)p.M * n_per; ++i)
            if (recv[d][(size_t)r * p.M * n_per + i] != -1.0f) return 7;
  }
  return 0;
}
'''


def build(out_dir):
    cell = _region(os.path.join(CSRC, "common.cuh"), "cell_index")
    cell, n = re.subn(r'int k; asm\("cvt\.rzi\.ftz\.s32\.f32[^;]*;[^;]*;', "int k = (int)res;   /* cvt.rzi */", cell)
    assert n == 1
    prep = (_region(os.path.join(CSRC, "common.cuh"), "xoro") + _region(os.path.join(CSRC, "common.cuh"), "normal") +
            _region(os.path.join(CSRC, "rollout_win.cu"), "prepare") + _region(os.path.join(CSRC, "rollout_win.cu"), "noise_prepare"))
    prep = re.sub(r"(?m)^(\s*)__shared__ ", r"\1static ", prep)
    kern = _region(os.path.join(CSRC, "rollout_win.cu"), "win_kernel")
    kern, n = re.subn(r'(?m)^\s*asm volatile\("fence\.[^;]*;[^;]*;\n', "", kern)        # mbarrier / proxy fences
    assert n == 2, n
    kern = kern.replace("extern __shared__ __align__(128) unsigned char smem[];", "")
    prelude = ROLLOUT_PRELUDE.replace("float s_u[4096];", "")
    src = (prelude + EXTRA + _region(os.path.join(CSRC, "common.cuh"), "params") + cell +
           _region(os.path.join(CSRC, "kernels.h"), "cost_dst") + _region(os.path.join(CSRC, "kernels.h"), "win_args") +
           prep + kern + HARNESS)
    cpp = os.path.join(out_dir, "rollout_win_emu.cpp")
    so = os.path.join(out_dir, "librollout_win_emu.so")
    open(cpp, "w").write(src)
    r = subprocess.run(["g++", "-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-Wno-unknown-pragmas",
                        "-ffp-contract=off", cpp, "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-6000:]
    lib = C.CDLL(so)
    P, I = C.c_void_p, C.c_int
    lib.emu_noise_prepare.restype = I
    lib.emu_noise_prepare.argtypes = [P, P, I, I, C.c_float, C.c_float, C.c_float, P, P, P, P, P, P, P]
    lib.emu_rollout_win.restype = I
    lib.emu_cell_between.argtypes = [P, I, C.c_float, P, P, P]
    lib.emu_cell_between.restype = None
    lib.emu_rollout_win.argtypes = [P, P, P, P, P, P, P, P, P, P, I, I, P, P, I, I, I, I, I]
    return lib
