// Host stand-ins for the CUDA the kernels use, and the launcher that runs a kernel's blocks on host threads (TEST
// INFRASTRUCTURE).  tests/emu_core.py compiles every kernel emulator as: this header, then the kernel text lifted from
// csrc/ inside namespace b200, then the emulator's extern "C" harness.  Each stand-in is defined once, here; a kernel
// that needs one more intrinsic gets it here.
//
// The arithmetic helpers of common.cuh (inline PTX on the GPU) have their IEEE meaning: add / sub / mul / fma rounded
// to nearest, floor, float <-> double conversions; the MUFU approximations (sin, cos, sqrt) and the approximate
// divisions are libm's correctly rounded functions.  Flush-to-zero is not emulated.
#pragma once
#include <algorithm>
#include <barrier>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <memory>
#include <thread>
#include <type_traits>
#include <vector>

// ------------------------------------------------------------------------------------------------------ language
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __launch_bounds__(...)
#define __grid_constant__
#define __align__(n)
#define __shared__          // function-scope __shared__ arrays become `static` (emu_core.shared_static)
using std::max;
using std::min;

// ------------------------------------------------------------------------------------------ vector types
struct EmuDim3 { unsigned x, y, z; };
struct float2 { float x, y; };
struct double2 { double x, y; };
struct ulonglong2 { unsigned long long x, y; };
struct uint4 { unsigned x, y, z, w; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { return ulonglong2{x, y}; }

// ------------------------------------------------------------------------------ block state of the launcher
namespace emu {
// the warp collectives exchange through a buffer between two barriers of the warp's threads
struct Warp {
  std::barrier<> bar;
  int ibuf[32];
  float fbuf[32];
  explicit Warp(int lanes) : bar(lanes) {}
};
inline std::barrier<>* block_bar = nullptr;   // blocks run one after another: one block barrier at a time
inline int block_count = 0;                     // __syncthreads_count's sum (zero between calls)
inline thread_local Warp* warp = nullptr;
// the block's shared memory: every `extern __shared__` array is a view of it (emu_core.extern_shared)
alignas(128) inline unsigned char smem[1 << 20];
}  // namespace emu

// ------------------------------------------------------------------------------------ indices and barriers
static thread_local EmuDim3 threadIdx, blockIdx, blockDim, gridDim;
static inline void __syncthreads() { emu::block_bar->arrive_and_wait(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { emu::warp->bar.arrive_and_wait(); }
// the block barrier plus the number of threads whose predicate is non-zero: counted between two barriers, cleared
// behind a third (no thread of the next call counts before every thread has read this one's sum)
static inline int __syncthreads_count(int pred) {
  if (pred) __atomic_fetch_add(&emu::block_count, 1, __ATOMIC_SEQ_CST);
  emu::block_bar->arrive_and_wait();
  const int r = __atomic_load_n(&emu::block_count, __ATOMIC_SEQ_CST);
  emu::block_bar->arrive_and_wait();
  if (threadIdx.x == 0) __atomic_store_n(&emu::block_count, 0, __ATOMIC_SEQ_CST);
  emu::block_bar->arrive_and_wait();
  return r;
}

// ---------------------------------------------------------------------------------------- warp collectives
static inline unsigned __activemask() { return 0xffffffffu; }
static inline float __shfl_xor_sync(unsigned, float v, int o) {
  emu::Warp& w = *emu::warp;
  const int lane = threadIdx.x & 31;
  w.fbuf[lane] = v;
  w.bar.arrive_and_wait();
  const float r = w.fbuf[lane ^ o];
  w.bar.arrive_and_wait();
  return r;
}
static inline int __shfl_sync(unsigned, int v, int src) {
  emu::Warp& w = *emu::warp;
  w.ibuf[threadIdx.x & 31] = v;
  w.bar.arrive_and_wait();
  const int r = w.ibuf[src];
  w.bar.arrive_and_wait();
  return r;
}
static inline int __reduce_add_sync(unsigned, int v) {
  emu::Warp& w = *emu::warp;
  w.ibuf[threadIdx.x & 31] = v;
  w.bar.arrive_and_wait();
  int s = 0;
  for (int i = 0; i < 32; ++i) s += w.ibuf[i];
  w.bar.arrive_and_wait();
  return s;
}
static inline int __reduce_max_sync(unsigned, int v) {
  emu::Warp& w = *emu::warp;
  w.ibuf[threadIdx.x & 31] = v;
  w.bar.arrive_and_wait();
  int r = w.ibuf[0];
  for (int i = 1; i < 32; ++i) r = w.ibuf[i] > r ? w.ibuf[i] : r;
  w.bar.arrive_and_wait();
  return r;
}

// ---------------------------------------------------------------------------------------- memory operations
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) {
  return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST);
}
static inline int atomicSub(int* p, int v) { return __atomic_fetch_sub(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicMax(unsigned* p, unsigned v) {
  unsigned o = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (o < v && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return o;
}
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void __threadfence_system() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline long long clock64() { return 0; }

// ------------------------------------------------------------------------------ bit and rounding intrinsics
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline int __double2loint(double d) { uint64_t u; std::memcpy(&u, &d, 8); return (int)(uint32_t)u; }
static inline int __double2hiint(double d) { uint64_t u; std::memcpy(&u, &d, 8); return (int)(uint32_t)(u >> 32); }
static inline double __hiloint2double(int hi, int lo) {
  const uint64_t u = ((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo; double d; std::memcpy(&d, &u, 8); return d;
}
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned s) {        // default mode, no msb replication
  const unsigned long long src = ((unsigned long long)b << 32) | a;
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) r |= (unsigned)((src >> (8 * ((s >> (4 * i)) & 7))) & 0xffu) << (8 * i);
  return r;
}
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __dsqrt_rn(double a) { return std::sqrt(a); }
static inline float __double2float_rn(double a) { return (float)a; }
// add.rm / add.rp.f32: the round-to-nearest sum moved one ulp towards the sign of its exact error (TwoSum; volatile:
// no re-association, no excess precision)
static inline float __fadd_rd(float a, float b) {
  volatile float s = a + b;
  volatile float bb = s - a;
  volatile float e1 = a - (s - bb), e2 = b - bb;
  const float err = e1 + e2;                                // exact: a + b == s + err
  return (err < 0.0f) ? std::nextafterf(s, -INFINITY) : (float)s;
}
static inline float __fadd_ru(float a, float b) {
  volatile float s = a + b;
  volatile float bb = s - a;
  volatile float e1 = a - (s - bb), e2 = b - bb;
  const float err = e1 + e2;
  return (err > 0.0f) ? std::nextafterf(s, INFINITY) : (float)s;
}

// -------------------------------------------------------------- the TMA descriptor of the windowed kernel
// a plain descriptor: base, dims, pitch, box; tma_load_* copy the box with zero fill outside the tensor (what
// CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE does for integer types)
struct CUtensorMap { const unsigned char* base; int cols, rows, maps, pitch, WW, WH; };

namespace b200 {
// ---------------------------------------------------------------------------------- helpers of common.cuh
static inline float sin_approx(float x) { return sinf(x); }
static inline float cos_approx(float x) { return cosf(x); }
static inline float sqrt_approx(float x) { return sqrtf(x); }
static inline float div_approx(float a, float b) { return a / b; }
static inline float div_full(float a, float b) { return a / b; }
static inline float div_rn(float a, float b) { return a / b; }
static inline float fadd(float a, float b) { return a + b; }
static inline float fsub(float a, float b) { return a - b; }
static inline float fmul(float a, float b) { return a * b; }
static inline float ffma(float a, float b, float c) { return fmaf(a, b, c); }
static inline float ffloor(float a) { return floorf(a); }
static inline double f2d(float a) { return (double)a; }
static inline float d2f(double a) { return (float)a; }
static inline float xoro_unit_f32(uint64_t x) { return (float)((double)(x >> 11) * (1.0 / 9007199254740992.0)); }
static inline unsigned sm_id() { return 0; }
static inline unsigned long long globaltimer_ns() { return 0; }
static inline void st_flag_sys(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
struct FlagWait { const uint32_t* flags; int ws; uint32_t epoch; unsigned long long timeout_ns; int* status; };
static inline void flag_wait(const FlagWait&) {}          // blocks run one after another: nothing to wait for

// ------------------------------------------------------------------- helpers of the windowed kernel (rollout_win.cu)
// mbarriers are no-ops (a copy is done when its call returns); shared-space addresses are offsets into emu::smem
static inline uint32_t smem_u32(const void* p) { return (uint32_t)((const unsigned char*)p - emu::smem); }
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
static inline void tma_load_3d(void* dst, const CUtensorMap* tm, uint64_t*, int c0, int c1, int c2) {
  tma_box((unsigned char*)dst, tm, c0, c1, c2);
}
static inline void tma_load_2d(void* dst, const CUtensorMap* tm, uint64_t*, int c0, int c1) {
  tma_box((unsigned char*)dst, tm, c0, c1, 0);
}
static inline int lds_s8(uint32_t addr, int imm_plane) { return (int)(int8_t)emu::smem[addr + (uint32_t)imm_plane]; }
static inline double lds_f64(uint32_t addr) { double v; std::memcpy(&v, emu::smem + addr, 8); return v; }
static inline double widen(float a) { return (double)a; }
static inline float narrow(double a) { return (float)a; }
static inline void keep_in_registers(float&, float&) {}
#define VELTKAMP_C 536870913.0

int update_num_ctas(int N);                                                      // reduce.cu
// the sampler's host-side table builders (sample.cu): linked from libb200mppi.so
void build_jump_matrices(const int64_t* ks, int count, uint64_t* out);
bool build_sample_thresholds(double alpha, int q_cap, uint64_t* table);
void sample_tile_draws(int rows, int cols, int tx, int ty, int64_t ks[4]);
}  // namespace b200

namespace emu {
// ------------------------------------------------------------------------------------------------ the launcher
// Blocks run one after another in x, then y, then z order, each with one std::thread per CUDA thread, one block
// barrier (__syncthreads) and one emu::Warp per 32 threads (__syncwarp and the warp collectives).
template <class F> static void launch(EmuDim3 grid, int threads, F&& kernel) {
  for (unsigned z = 0; z < grid.z; ++z)
    for (unsigned y = 0; y < grid.y; ++y)
      for (unsigned x = 0; x < grid.x; ++x) {
        std::barrier<> bar(threads);
        block_bar = &bar;
        std::vector<std::unique_ptr<Warp>> warps;
        for (int w = 0; w < (threads + 31) / 32; ++w) warps.emplace_back(new Warp(std::min(32, threads - 32 * w)));
        std::vector<std::thread> th;
        for (int t = 0; t < threads; ++t)
          th.emplace_back([&, t] {
            threadIdx = {(unsigned)t, 0, 0}; blockIdx = {x, y, z}; blockDim = {(unsigned)threads, 1, 1}; gridDim = grid;
            warp = warps[t / 32].get();
            kernel();
          });
        for (auto& t : th) t.join();
      }
}
// The kernels without barriers (noise, setters): every thread of every block in turn on the calling thread.
template <class F> static void launch_serial(EmuDim3 grid, int threads, F&& kernel) {
  blockDim = {(unsigned)threads, 1, 1}; gridDim = grid;
  for (unsigned z = 0; z < grid.z; ++z)
    for (unsigned y = 0; y < grid.y; ++y)
      for (unsigned x = 0; x < grid.x; ++x)
        for (int t = 0; t < threads; ++t) {
          blockIdx = {x, y, z}; threadIdx = {(unsigned)t, 0, 0};
          kernel();
        }
}

// ------------------------------------------------------------- launch rules of the host code, stated once
// The rollout harnesses' parameter block -> RolloutParams (b200mppi_planner_set_params), M given by the caller:
// f: res, xlo, ylo, dt, x0[3], xgoal[2], goal_tol, v_post, lambda, u_std[2], vrange[2], wrange[2], obs, unk, dist_w,
//    lin_lo, ang_lo (23 floats);  g: rows, cols, grid_rows, grid_cols, grid_pitch, mask_pitch, T, N (then M);
// ratios: lin_ratio, ang_ratio
template <class P> static void params(P& p, const float* f, const int* g, const double* ratios, int M) {
  p = P{};
  p.g.res = f[0]; p.g.inv_res = 1.0f / f[0]; p.g.xlo = f[1]; p.g.ylo = f[2];
  p.g.rows = g[0]; p.g.cols = g[1]; p.g.grid_rows = g[2]; p.g.grid_cols = g[3]; p.g.grid_pitch = g[4]; p.g.mask_pitch = g[5];
  p.dt = f[3]; p.x0[0] = f[4]; p.x0[1] = f[5]; p.x0[2] = f[6]; p.xgoal[0] = f[7]; p.xgoal[1] = f[8];
  p.tol2 = f[9] * f[9]; p.v_post = f[10]; p.lambda = f[11]; p.u_std[0] = f[12]; p.u_std[1] = f[13];
  p.vrange[0] = f[14]; p.vrange[1] = f[15]; p.wrange[0] = f[16]; p.wrange[1] = f[17];
  p.obs_cost = f[18]; p.unk_cost = f[19]; p.dist_weight = f[20]; p.lin_lo = f[21]; p.ang_lo = f[22];
  p.lin_ratio = ratios[0]; p.ang_ratio = ratios[1];
  p.T = g[6]; p.N = g[7]; p.M = M;
}

// launch_cvar (rollout.cu): the warp kernel's values per lane for M maps, passed to f as a std::integral_constant
template <class F> static void cvar_per(int M, F&& f) {
  const int per = (M + 31) / 32;
  if (per <= 1) f(std::integral_constant<int, 1>{});
  else if (per <= 2) f(std::integral_constant<int, 2>{});
  else if (per <= 4) f(std::integral_constant<int, 4>{});
  else if (per <= 8) f(std::integral_constant<int, 8>{});
  else if (per <= 16) f(std::integral_constant<int, 16>{});
  else f(std::integral_constant<int, 32>{});
}

// launch_v2_nt (sample.cu): the sampler kernel's 32-bit words per cumulative-table cell, as a std::integral_constant
template <class F> static void sampler_nw(int bpad, F&& f) {
  const int nw = bpad / 4;
  if (nw == 3) f(std::integral_constant<int, 3>{});
  else if (nw == 8) f(std::integral_constant<int, 8>{});
  else if (nw == 1) f(std::integral_constant<int, 1>{});
  else f(std::integral_constant<int, 0>{});
}

// The update's CTAs for N rollouts: update_num_ctas (reduce.cu), then the planner's rule (api.cu) of whole slabs of
// rows_per_cta rows
static inline void update_geometry(int N, int& num_ctas, int& rows_per_cta) {
  const int ctas = b200::update_num_ctas(N);
  rows_per_cta = (N + ctas - 1) / ctas;
  num_ctas = (N + rows_per_cta - 1) / rows_per_cta;
}

// tdm_prepare_jump (api.cu): the sampler's row segments (at most one per tile row) and, for more than one, the jump
// matrices of each segment start in both width classes (full tile columns, the last column); J stays empty for one
static inline void segment_jumps(int rows, int cols, int tx, int ty, int& segs, int& seg_rows, std::vector<uint64_t>& J) {
  const int nrow = (rows + tx - 1) / tx, ncol = (cols + ty - 1) / ty;
  if (segs > nrow) segs = nrow;
  if (segs < 1) segs = 1;
  seg_rows = (nrow + segs - 1) / segs;
  J.clear();
  if (segs == 1) return;
  int last_w = cols - (ty - 1) * ncol;
  for (int iy = ty - 1; iy >= 0 && last_w <= 0; --iy) last_w = cols - iy * ncol;
  if (last_w > ncol) last_w = ncol;
  if (last_w < 0) last_w = 0;
  std::vector<int64_t> ks;
  for (int s = 1; s < segs; ++s) { ks.push_back((int64_t)s * seg_rows * ncol); ks.push_back((int64_t)s * seg_rows * last_w); }
  J.resize(ks.size() * 256);
  b200::build_jump_matrices(ks.data(), (int)ks.size(), J.data());
}

// fill_win_args / stage_rollout (api.cu): the window around the robot's cell, moved by (shift_x, shift_y) cells, kept
// inside the map, its x aligned down to 16 cells
template <class W> static void win_place(W& w, int WW, int WH, int shift_x = 0, int shift_y = 0) {
  const auto& p = w.p;
  const int xi0 = (int)std::floor(((double)p.x0[0] - (double)p.g.xlo) / (double)p.g.res);
  const int yi0 = (int)std::floor(((double)p.x0[1] - (double)p.g.ylo) / (double)p.g.res);
  int cx = xi0 - WW / 2 + shift_x, cy = yi0 - WH / 2 + shift_y;
  cx = std::max(0, std::min(cx, p.g.cols - WW));
  cy = std::max(0, std::min(cy, p.g.rows - WH));
  w.WW = WW; w.WH = WH;
  w.wx0 = cx & ~15;
  w.wy0 = cy;
  w.ww = std::min(WW, p.g.cols - w.wx0);
  w.wh = std::min(WH, p.g.rows - w.wy0);
}
}  // namespace emu
