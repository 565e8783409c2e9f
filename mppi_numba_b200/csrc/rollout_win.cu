// rollout_win.cu -- the stochastic ("CVaR-cost") rollout kernel as it is meant to run on an H100 (sm_90a):
// a persistent CTA per SM works on ONE sampled traction map at a time; the window of that map around the robot
// (linear and angular traction planes of map m, plus the obstacle / unknown planes shared by all maps) is staged
// into shared memory with four TMA tensor loads (cp.async.bulk.tensor), after which every per-step lookup of the
// CTA's rollouts on that map is a shared-memory byte load.
// Lanes of a warp share the map and differ in the control sequence n -- the opposite of the
// reference (mppi_numba/mppi.py:613-755: block = n, thread = m, i.e. 32 different maps per warp-load).
//
// Arithmetic: identical to rollout.cu / the reference (float64 FMA state update rounded once to
// float32, approximate sin/cos/sqrt, the reference's FMA contractions).  What differs from the
// generic kernel is only HOW the same numbers are obtained:
//   * lo + ratio*q and its product with dt (two float64 ops per step in the reference) come from a
//     256-entry float64 table per map type built with the same two operations;
//   * the cell index uses round-down magic-number arithmetic on the FP32 pipe (no FRND / F2I on the
//     XU pipe) and falls back to the exact reference sequence near cell edges;
//   * obstacle / unknown penalties without an integer-to-float conversion (masks of 0 / 1: cost + bits(c)*mask);
//   * the control-cost sum over T, identical for all M maps of a control sequence, is computed once
//     per n by the prepare kernel (rounding differs from the reference's running sum by ~1 ulp).
// A rollout that leaves the window reads the maps from global memory instead (same values); the window never
// extends beyond the map, so out-of-map indices always take that path and wrap / clamp exactly like the generic
// kernel (rollout.cu: wrap_clamp).
#include <cuda.h>

#include <algorithm>
#include <cstdlib>

#include "kernels.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// prepare: noise (N,T,2) -> transposed CLIPPED NOISY CONTROLS ctlT [T][npad] double2
//   (v, w) = (clip(u_v[t] + e_v, vrange), clip(u_w[t] + e_w, wrange))           (mppi.py:686-689)
// -- identical for all M maps of a control sequence, so computed once here (coalesced per-step loads
// for lanes = consecutive n) -- and the per-n control cost sum_t lambda*(u_v/s_v^2*e_v + u_w/s_w^2*e_w)
// (mppi.py:708-710), accumulated in the reference's order t = 0..T-1.
// noiseT has T + 1 rows of npad double2 (the rollout kernel prefetches one row ahead without a guard; row T is never
// used and never written).
// [emu:begin prepare]
__global__ void __launch_bounds__(256) prepare_rollout_kernel(const float2* __restrict__ noise,
                                                              const float* __restrict__ u_cur,
                                                              double2* __restrict__ noiseT,
                                                              float* __restrict__ ctrl, float* __restrict__ reach,
                                                              int N, int T, int npad,
                                                              float lambda, float sv2, float sw2, float v_lo,
                                                              float v_hi, float w_lo, float w_hi) {
  __shared__ float2 tile[32][33];
  const int n0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8
  float acc = 0.0f, vsum = 0.0f;
  for (int t0 = 0; t0 < T; t0 += 32) {
    for (int r = ty; r < 32; r += 8) {                         // rows = n, cols = t  (coalesced along t)
      const int n = n0 + r, t = t0 + tx;
      tile[r][tx] = (n < N && t < T) ? noise[(size_t)n * T + t] : make_float2(0.f, 0.f);
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {                         // rows = t, cols = n  (coalesced along n)
      const int t = t0 + r;
      if (t < T) {
        const float2 e = tile[tx][r];
        // stored already widened to float64 (exact): the rollout kernel's per-step f2d(v), f2d(w) are
        // XU-pipe conversions, and these values are shared by all M maps of the control sequence
        double2 c;
        c.x = f2d(fmaxf(v_lo, fminf(v_hi, fadd(u_cur[2 * t], e.x))));
        c.y = f2d(fmaxf(w_lo, fminf(w_hi, fadd(u_cur[2 * t + 1], e.y))));
        noiseT[(size_t)t * npad + n0 + tx] = c;
      }
    }
    if (ty == 0) {                                             // lane tx owns rollout n0+tx
      const int tend = min(32, T - t0);
      for (int j = 0; j < tend; ++j) {
        const float2 e = tile[tx][j];
        const float a = div_approx(u_cur[2 * (t0 + j)], sv2);
        const float b = div_approx(u_cur[2 * (t0 + j) + 1], sw2);
        acc = ffma(ffma(a, e.x, fmul(b, e.y)), lambda, acc);
        // reach statistic: sum_t |v| of the clipped speed command (rounded up: it is used as an upper bound)
        vsum = __fadd_ru(vsum, fabsf(fmaxf(v_lo, fminf(v_hi, fadd(u_cur[2 * (t0 + j)], e.x)))));
      }
    }
    __syncthreads();
  }
  if (ty == 0) {
    if (n0 + tx < N) ctrl[n0 + tx] = acc; else vsum = 0.0f;
    if (reach) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) vsum = fmaxf(vsum, __shfl_xor_sync(0xffffffffu, vsum, o));
      // non-negative floats order like their bit patterns; a NaN (sign clear) compares above every number and
      // makes the host fall back to the static bound
      if (tx == 0) atomicMax(reinterpret_cast<unsigned int*>(reach), __float_as_uint(vsum));
    }
  }
}

// [emu:end prepare]

// ---------------------------------------------------------------------------------------------
// noise + prepare in ONE launch (what solve() runs): the control noise of sample_noise_numba (mppi.py:1354-1370;
// generator n*T + t, Box-Muller, states advanced in place) is written once in the reference's (N, T, 2) layout for the
// update kernel and the public noise_samples_d -- and, from the same registers, through the shared-memory transpose
// of the prepare kernel above, as the clipped float64 controls [T][npad] the rollout kernel streams, with the per-n
// control cost and the reach statistic.  Same arithmetic, same order as the two separate kernels (bit-identical
// outputs: tests/test_rollout_win_emulated_cpu.py).
// `reach` has two slots used alternately by consecutive launches: this launch max-reduces into reach[slot] and clears
// reach[slot ^ 1] for the next one (the host has read it: solve() synchronises on it).
// [emu:begin noise_prepare]
constexpr int NP_NB = 8;            // control sequences per CTA: 1024 CTAs of 8 x 32 threads at config 5 (occupancy; the
                                    // Box-Muller chains are long and latency-bound)
__device__ __forceinline__ void noise_prepare_body(uint64_t* __restrict__ states, float2* __restrict__ noise,
                                                   const float* __restrict__ u_cur, double2* __restrict__ noiseT,
                                                   float* __restrict__ ctrl, float* __restrict__ reach, int slot, int N,
                                                   int T, int npad, float std_v, float std_w, float lambda, float sv2,
                                                   float sw2, float v_lo, float v_hi, float w_lo, float w_hi) {
  __shared__ float2 tile[NP_NB][33];
  const int n0 = blockIdx.x * NP_NB;
  const int tx = threadIdx.x & 31, r = threadIdx.x >> 5;       // generation: row r = control sequence, lane = time step
  const int tn = threadIdx.x & (NP_NB - 1), tt = threadIdx.x >> 3;   // transposed write: 8 consecutive n per time step
  if (blockIdx.x == 0 && threadIdx.x == 0 && reach) reach[slot ^ 1] = 0.0f;
  float acc = 0.0f, vsum = 0.0f;
  for (int t0 = 0; t0 < T; t0 += 32) {
    {                                                          // generators (n0 + r) * T + t0 + tx: contiguous along the lanes
      const int n = n0 + r, t = t0 + tx;
      float2 e = make_float2(0.f, 0.f);
      if (n < N && t < T) {
        const size_t g = (size_t)n * T + t;
        ulonglong2* sp = reinterpret_cast<ulonglong2*>(states) + g;
        const ulonglong2 raw = *sp;
        Xoro s{raw.x, raw.y};
        e.x = fmul(std_v, xoro_normal(s));
        e.y = fmul(std_w, xoro_normal(s));
        noise[g] = e;
        *sp = make_ulonglong2(s.s0, s.s1);
      }
      tile[r][tx] = e;
    }
    __syncthreads();
    {                                                          // rows = t, 8 consecutive n per row: 128-byte segments
      const int t = t0 + tt;
      if (t < T) {
        const float2 e = tile[tn][tt];
        double2 c;
        c.x = f2d(fmaxf(v_lo, fminf(v_hi, fadd(u_cur[2 * t], e.x))));
        c.y = f2d(fmaxf(w_lo, fminf(w_hi, fadd(u_cur[2 * t + 1], e.y))));
        noiseT[(size_t)t * npad + n0 + tn] = c;
      }
    }
    if (threadIdx.x < NP_NB) {                                 // lane tn owns rollout n0 + tn: sums in the reference's order t = 0..T-1
      const int tend = min(32, T - t0);
      for (int j = 0; j < tend; ++j) {
        const float2 e = tile[tn][j];
        const float a = div_approx(u_cur[2 * (t0 + j)], sv2);
        const float b = div_approx(u_cur[2 * (t0 + j) + 1], sw2);
        acc = ffma(ffma(a, e.x, fmul(b, e.y)), lambda, acc);
        vsum = __fadd_ru(vsum, fabsf(fmaxf(v_lo, fminf(v_hi, fadd(u_cur[2 * (t0 + j)], e.x)))));
      }
    }
    __syncthreads();
  }
  if (threadIdx.x < 32) {                                      // whole first warp takes part in the shuffles
    const bool own = threadIdx.x < NP_NB && n0 + tn < N;
    if (own) ctrl[n0 + tn] = acc; else vsum = 0.0f;
    if (reach) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) vsum = fmaxf(vsum, __shfl_xor_sync(0xffffffffu, vsum, o));
      if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned int*>(reach + slot), __float_as_uint(vsum));
    }
  }
}

__global__ void __launch_bounds__(256) noise_prepare_kernel(uint64_t* __restrict__ states, float2* __restrict__ noise,
                                                            const float* __restrict__ u_cur, double2* __restrict__ noiseT,
                                                            float* __restrict__ ctrl, float* __restrict__ reach, int slot,
                                                            int N, int T, int npad, float std_v, float std_w, float lambda,
                                                            float sv2, float sw2, float v_lo, float v_hi, float w_lo,
                                                            float w_hi) {
  noise_prepare_body(states, noise, u_cur, noiseT, ctrl, reach, slot, N, T, npad, std_v, std_w, lambda, sv2, sw2, v_lo,
                     v_hi, w_lo, w_hi);
}

// [emu:end noise_prepare]
// batched stochastic solves: planner blockIdx.y, its buffers and scalars from the descriptor array; N, T and npad are
// the batch's.  Iteration `iter` of a solve uses reach slot d.slot ^ (iter & 1): each planner's slot toggles once per
// iteration, as in its own solve()
// [emu:begin noise_prepare_batch]
__global__ void __launch_bounds__(256) noise_prepare_batch_kernel(const NoisePrepDesc* __restrict__ descs, int N, int T,
                                                                  int npad, int iter,
                                                                  const int* __restrict__ active = nullptr) {
  if (active && !active[blockIdx.y]) return;
  const NoisePrepDesc& d = descs[blockIdx.y];
  noise_prepare_body(d.states, reinterpret_cast<float2*>(d.noise), d.u_cur, reinterpret_cast<double2*>(d.noiseT), d.ctrl,
                     d.reach, d.slot ^ (iter & 1), N, T, npad, d.std_v, d.std_w, d.lambda, d.sv2, d.sw2, d.v_lo, d.v_hi,
                     d.w_lo, d.w_hi);
}
// [emu:end noise_prepare_batch]
void launch_noise_prepare(uint64_t* states, float* noise, const float* u_cur, float* noiseT, float* ctrl, float* reach,
                          int slot, int N, int T, int npad, float lambda, float std_v, float std_w, const float vrange[2],
                          const float wrange[2], cudaStream_t st) {
  noise_prepare_kernel<<<npad / NP_NB, 256, 0, st>>>(states, reinterpret_cast<float2*>(noise), u_cur,
                                                 reinterpret_cast<double2*>(noiseT), ctrl, reach, slot, N, T, npad, std_v,
                                                 std_w, lambda, std_v * std_v, std_w * std_w, vrange[0], vrange[1],
                                                 wrange[0], wrange[1]);
}
void launch_noise_prepare_batch(const NoisePrepDesc* descs, int count, int N, int T, int npad, int iter,
                                const int* active, cudaStream_t st) {
  noise_prepare_batch_kernel<<<dim3((unsigned)(npad / NP_NB), (unsigned)count), 256, 0, st>>>(descs, N, T, npad, iter,
                                                                                               active);
}
void launch_prepare_rollout(const float* noise, const float* u_cur, float* noiseT, float* ctrl, float* reach, int N,
                            int T, int npad, float lambda, float std_v, float std_w, const float vrange[2],
                            const float wrange[2], cudaStream_t st) {
  prepare_rollout_kernel<<<npad / 32, 256, 0, st>>>(reinterpret_cast<const float2*>(noise), u_cur,
                                                   reinterpret_cast<double2*>(noiseT), ctrl, reach, N, T, npad, lambda,
                                                   std_v * std_v, std_w * std_w, vrange[0], vrange[1], wrange[0],
                                                   wrange[1]);
}

// ---------------------------------------------------------------------------------------------
// TMA plumbing (sm_90a): mbarrier + cp.async.bulk.tensor
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

// explicit shared-space loads (a generic pointer into dynamic smem makes the compiler rebuild the
// shared-window base with S2UR/ULEA every iteration)
__device__ __forceinline__ int lds_s8(uint32_t addr, int imm_plane) {
  int v;
  asm("ld.shared.s8 %0, [%1];" : "=r"(v) : "r"(addr + (uint32_t)imm_plane));
  return v;
}
__device__ __forceinline__ double lds_f64(uint32_t addr) {
  double v;
  asm("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ float2 lds_f32x2(uint32_t addr) {
  float2 v;
  asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
// widening / narrowing without the .ftz flush (the reference flushes f32 denormals here; positions,
// headings and clipped controls are never denormal, zero converts exactly either way)
__device__ __forceinline__ double widen(float a) {
  double r; asm("cvt.f64.f32 %0, %1;" : "=d"(r) : "f"(a)); return r;
}
__device__ __forceinline__ float narrow(double a) {
  float r; asm("cvt.rn.f32.f64 %0, %1;" : "=f"(r) : "d"(a)); return r;
}
// opaque to the optimiser: the two values stay in their registers instead of being rematerialised at every use
__device__ __forceinline__ void keep_in_registers(float& a, float& b) { asm volatile("" : "+f"(a), "+f"(b)); }
// 2^29 + 1 in the constant bank: DMUL takes it as a c[][] operand (as a literal it costs two UMOV per step)
__constant__ double k_veltkamp_c = 536870913.0;
#define VELTKAMP_C k_veltkamp_c
// [emu:begin win_kernel]
#ifndef WIN_ROUND_FP64
#define WIN_ROUND_FP64 1
#endif
// float64 value rounded to float32 precision (round-to-nearest-even at bit 29), kept as float64:
// == widen(narrow(a)) for every |a| in the float32 normal range, without a second XU-pipe conversion.
// WIN_ROUND_FP64 = 1 (default): Veltkamp's splitting on the FP64 pipe -- g = RN(a * (2^29 + 1)), hi = RN(g + RN(a - g))
// is a rounded to 53 - 29 = 24 significant bits, ties to even (three round-to-nearest operations that must not be
// contracted into an FMA: hence the intrinsics; pinned against the float32 conversion on 10^7 near-tie values in
// tests/test_rollout_win_emulated_cpu.py).  Three FP64-pipe instructions (a lightly used pipe in this kernel) instead of
// the five integer instructions of the bit-level version below (the integer pipe is the busier one).
// A zero loses its sign (-0 -> +0), which no later operation of the step can see.
__device__ __forceinline__ double round_to_f32_precision(double a) {
#if WIN_ROUND_FP64
  const double g = __dmul_rn(a, VELTKAMP_C);
  return __dadd_rn(g, __dsub_rn(a, g));
#else
  uint64_t b = ((uint64_t)(uint32_t)__double2hiint(a) << 32) | (uint32_t)__double2loint(a);
  b += 0x0FFFFFFFull + ((b >> 29) & 1ull);          // 64-bit add: the carry into the high word is the add's own
  return __hiloint2double((int)(uint32_t)(b >> 32), (int)((uint32_t)b & 0xE0000000u));
#endif
}

// obstacle / unknown penalties (mppi.py:700-701), inside a branch taken when either mask byte is non-zero (a tenth of the
// warp-steps at BASELINE config 5, up to half for the control sequences that graze obstacles).  Inline and off the XU
// pipe: float(v) of the int8 mask value by the magic-number trick (exact for |v| < 2^22) instead of I2F -- as an
// out-of-line call with two conversions queued behind the other warps' MUFU / F2F work the branch was expensive
// enough to make the CTAs whose rollouts cross obstacles the stragglers of the grid.
static __device__ __forceinline__ float add_penalties(float cost, int ob, int un, float obs_cost, float unk_cost) {
  const float fo = fsub(__int_as_float(0x4B400000 + ob), 12582912.0f);
  const float fu = fsub(__int_as_float(0x4B400000 + un), 12582912.0f);
  cost = ffma(fo, obs_cost, cost);
  return ffma(fu, unk_cost, cost);
}

// floor(a / r) from the magic-number sums k, k2 of the two ends of the interval that contains the exact quotient (the
// caller's): while both are integers in range (|index| < 2^21: the sums stay in the binade where one ulp is 1), the
// floor is lo = k - MAGIC if the ends agree, and otherwise lo or hi = lo + 1 -- hi exactly when a >= hi * r, a product
// of a 22-bit integer and a float32, exact in float64.  No division; what the reference's sequence (cell_index_exact:
// three float32 divisions) returns is this same true floor.  Anything else (an interval wider than one integer,
// indices beyond 2^21, NaN) runs that sequence.
static __device__ __forceinline__ int cell_from_interval(float a, float r, float k, float k2) {
  const int lo = __float_as_int(k) - 0x4B400000, hi = __float_as_int(k2) - 0x4B400000;
  if (lo > -(1 << 21) && hi < (1 << 21) && r > 0.0f) {
    if (hi == lo) return lo;
    if (hi - lo == 1) return ((double)a >= (double)hi * (double)r) ? hi : lo;
  }
  return cell_index_exact(a, r);
}

constexpr int WIN_ESCAPE = (int)0x80808080u;   // lookup_slow's report of an escape: four codes -128 (see stage_planner)
enum { WIN_WHOLE = 0, WIN_DETECT = 1, WIN_REDO = 2 };

// everything that is not "cell proven by the magic-number floors and staged in the window" (~0.1 % of the steps near
// cell edges, plus the steps of rollouts that left the window): exact reference cell index, then the staged window
// if the cell is in it, else global memory with the generic kernel's wrap + clamp.  Out of line: one call site, one
// reconvergence region in the hot loop.
template <int WW, int PLANE, bool DETECT>
static __device__ __noinline__ int lookup_slow(float ax, float ay, float res, float inv_lo, float inv_hi, uint32_t sb_win,
                                               unsigned uww, unsigned uwh, int wx0, int wy0, int rows, int cols, int grid_rows,
                                               int grid_cols, int grid_pitch, int mask_pitch,
                                               const int8_t* __restrict__ g_lin, const int8_t* __restrict__ g_ang,
                                               const int8_t* __restrict__ obstacle, const int8_t* __restrict__ unknown) {
  // an exact decision only for the axis whose interval holds an integer: the other axis' cell is proven by its equal
  // floors (the caller's test, repeated here rather than passed in registers)
  const float MAGIC = 12582912.0f;
  const float kx = __fadd_rd(fmaf(ax, inv_lo, -1e-30f), MAGIC), kx2 = __fadd_rd(fmaf(ax, inv_hi, 1e-30f), MAGIC);
  const float ky = __fadd_rd(fmaf(ay, inv_lo, -1e-30f), MAGIC), ky2 = __fadd_rd(fmaf(ay, inv_hi, 1e-30f), MAGIC);
  const int xi = cell_from_interval(ax, res, kx, kx2), yi = cell_from_interval(ay, res, ky, ky2);
  const int wx = xi - wx0, wy = yi - wy0;
  int ql, qa, ob, un;
  if ((unsigned)wx < uww && (unsigned)wy < uwh) {
    const uint32_t ad = sb_win + (uint32_t)(wy * WW + wx);
    ql = lds_s8(ad, 0); qa = lds_s8(ad + PLANE, 0); ob = lds_s8(ad + 2 * PLANE, 0); un = lds_s8(ad + 3 * PLANE, 0);
  } else {
    const int gy2 = min(max(yi < 0 ? yi + grid_rows : yi, 0), grid_rows - 1);
    const int gx2 = min(max(xi < 0 ? xi + grid_cols : xi, 0), grid_cols - 1);
    const int my = min(max(yi < 0 ? yi + rows : yi, 0), rows - 1);
    const int mx = min(max(xi < 0 ? xi + cols : xi, 0), cols - 1);
    ql = __ldg(g_lin + (size_t)gy2 * grid_pitch + gx2);
    qa = __ldg(g_ang + (size_t)gy2 * grid_pitch + gx2);
    ob = __ldg(obstacle + (size_t)my * mask_pitch + mx);
    un = __ldg(unknown + (size_t)my * mask_pitch + mx);
    // window-first sampling: a map cell outside the sampled rectangle holds a stale byte -- an escape, reported as
    // WIN_ESCAPE (cells of the allocation beyond the map are never sampled in any mode)
    constexpr int R = WIN_SAMPLE_RING;
    if (DETECT && gy2 < rows && gx2 < cols &&
        (gx2 < max(wx0 - R, 0) || gx2 >= min(wx0 + (int)uww + R, cols) || gy2 < max(wy0 - R, 0) ||
         gy2 >= min(wy0 + (int)uwh + R, rows)))
      return WIN_ESCAPE;
  }
  return (ql & 0xff) | ((qa & 0xff) << 8) | ((ob & 0xff) << 16) | (un << 24);     // four int8 in one register
}

struct WinSmem {                 // dynamic shared memory carve-up (all offsets multiples of 128)
  int plane;                     // bytes per plane = WW*WH
  int off_lut, off_u, off_bar, total;
};
__host__ __device__ inline WinSmem win_smem_layout(int WW, int WH, int T) {
  WinSmem s;
  s.plane = WW * WH;
  const int planes = (4 * s.plane + 127) & ~127;
  s.off_lut = planes;                              // 2 x 256 doubles
  s.off_u = s.off_lut + 2 * 256 * 8;               // 2T floats
  s.off_bar = (s.off_u + 2 * T * 4 + 15) & ~15;       // mbarrier (8 bytes) + the chunk counter
  s.total = s.off_bar + 16;
  return s;
}

constexpr int WIN_WW = 240;       // window width in cells (inner TMA box extent: 240 B, multiple of 16)

// Work distribution: PERSISTENT grid, one CTA per SM.  The work list is the map-major sequence of 32-rollout chunks
// (map m, control sequences [32c, 32c + 32)); CTA b owns the contiguous share [b*total/G, (b+1)*total/G) of it --
// every SM gets the same number of chunks whatever M and N are (a (tiles, M) grid of one-tile CTAs quantises: 256
// tile units on 132 SMs = two rounds where 1.94 would do).  A share spans one to a few maps: per map the
// CTA stages that map's window once (thread 0 issues the TMA loads after the CTA has left the previous window), then
// its warps pull chunks from a shared-memory counter until the map's part of the share is done -- warps whose
// rollouts reached the goal early simply take the next chunk.  Short shares (a rank of a 4- or 8-GPU solve): see
// a.unit == 0 in the kernel.  A global work queue instead of static shares was measured and dropped (DESIGN.md 4.2).
//
// per-CTA timing / counting hook (tools/rollout_cta_times.py): compiled in only with -DB200MPPI_WIN_DEBUG_HOOK
// (B200MPPI_NVCC_FLAGS of build.py) -- the hot loop's register allocation is tight enough for a dead branch to show
#ifdef B200MPPI_WIN_DEBUG_HOOK
#define WIN_DBG(a) ((a).dbg != nullptr)
#else
#define WIN_DBG(a) false
#endif
// MASK01: every byte of the obstacle / unknown masks is 0 or 1 (checked on the host when they are set): the penalty of a
// step is then two additions of `c` or +0.0 (selected by an integer multiply) instead of the general multiply-adds
//
// BATCH (batched stochastic solves, rollout_win_batch_kernel): the work list is the planner-major, then map-major
// sequence of chunks over the count * M (planner, map) units, and the share logic above reads "map" as "unit".  `g` holds
// the launch-wide fields (p.N, p.M, p.T, npad and the share settings); whenever a CTA reaches a unit of another planner it
// copies that planner's RolloutWinArgs from `descs` into shared memory behind the window (per-step scalars are then
// shared-memory loads, never global ones) and rebuilds the traction tables, s_u and the derived registers from it.
// Single launch: `g` is the planner's own RolloutWinArgs and the tensor maps are kernel parameters.
template <int THREADS, int WH, bool MASK01, bool BATCH, int MODE = WIN_WHOLE>
__device__ __forceinline__ void rollout_win_body(const RolloutWinArgs& g, const CUtensorMap* tm_lin,
                                                 const CUtensorMap* tm_ang, const CUtensorMap* tm_obs,
                                                 const CUtensorMap* tm_unk, const RolloutWinArgs* descs,
                                                 const CUtensorMap* tmaps, int count, const int* active) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int WW = WIN_WW;
  constexpr int PLANE = WW * WH;
  const WinSmem L = win_smem_layout(WW, WH, g.p.T);
  RolloutWinArgs* s_rec = reinterpret_cast<RolloutWinArgs*>(smem + L.total);     // BATCH: the current planner's record
  const RolloutWinArgs& a = BATCH ? *s_rec : g;
  const RolloutParams& p = a.p;
  double* s_lutL = reinterpret_cast<double*>(smem + L.off_lut);
  double* s_lutA = s_lutL + 256;
  float* s_u = reinterpret_cast<float*>(smem + L.off_u);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + L.off_bar);
  int* s_next = reinterpret_cast<int*>(bar + 1);             // chunk counter of the current map

  const int tid = threadIdx.x, lane = tid & 31;
  const int cpm = g.npad >> 5;                               // chunks per map
  int units_n = BATCH ? count * g.p.M : g.p.M;               // maps, or (planner, map) units
  if (MODE == WIN_REDO) {
    // redo: the units are the flagged maps only, in map order (g.unit = 1: dealt chunk by chunk); no flag: every CTA
    // leaves here
    int mine = 0;
    for (int i = tid; i < g.p.M; i += THREADS) mine += g.esc[i] != 0;
    if (tid == 0) *s_next = 0;
    __syncthreads();
    if (mine) atomicAdd(s_next, mine);
    __syncthreads();
    units_n = *s_next;
    __syncthreads();                                        // (s_next is the chunk counter from here on)
    if (units_n == 0) return;
  }
  const long long total = (long long)units_n * cpm;
  // share boundaries are multiples of a.unit chunks (32 = one chunk per warp of the CTA when the shares are long
  // enough: every map segment is then a whole number of passes and all warps reach the end-of-segment barrier
  // together, where chunk-granular shares leave warps parked at that barrier; 1 for short shares)
  //
  // a.unit == 0 (short shares and at least one CTA per map: the 8-GPU regime): shares never cross a map.  Map m gets q
  // or q + 1 of the CTAs (q = CTAs / maps) and its chunks are split evenly among them.  A share that crosses a map
  // boundary costs a second window and, worse, two partial passes (a handful of warps running alone twice).
  long long w_lo, w_hi;
  if (g.unit == 0) {
    const int G = (int)gridDim.x, b = ((int)blockIdx.x + g.rotate) % (int)gridDim.x, q = G / units_n, r = G - q * units_n;    // the first r maps get q + 1 CTAs
    int m, j, k;
    if (b < r * (q + 1)) { m = b / (q + 1); j = b - m * (q + 1); k = q + 1; }
    else { const int b2 = b - r * (q + 1); m = r + b2 / q; j = b2 - (m - r) * q; k = q; }
    w_lo = (long long)m * cpm + (long long)cpm * j / k;
    w_hi = (long long)m * cpm + (long long)cpm * (j + 1) / k;
  } else {
    const long long units = (total + g.unit - 1) / g.unit;
    w_lo = min(total, units * blockIdx.x / gridDim.x * g.unit);
    w_hi = min(total, units * (blockIdx.x + 1) / gridDim.x * g.unit);
  }
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  uint32_t sb_win, sb_lutL, sb_lutA, sb_u;
  float xlo, ylo, res, inv_res, gx, gy, inv_lo, inv_hi;
  int magic_wx, magic_wy;
  unsigned uww, uwh;
  const float MAGIC = 12582912.0f;                          // 1.5 * 2^23
  // everything the CTA derives from its planner's arguments (once; BATCH: at every planner switch)
  auto stage_planner = [&]() {
    // traction tables: (lo + ratio*q) * dt exactly as the reference evaluates it (fma.rn.f64, mul.f64)
    const double dt64 = f2d(p.dt);
    for (int i = tid; i < 256; i += THREADS) {
      const double q = (double)(i - 128);
      s_lutL[i] = fma(p.lin_ratio, q, f2d(p.lin_lo)) * dt64;
      s_lutA[i] = fma(p.ang_ratio, q, f2d(p.ang_lo)) * dt64;
    }
    // window-first sampling: an escape reads the codes of WIN_ESCAPE, whose linear traction is NaN here -- the state, and
    // with it the cost, turn NaN (NaN stays NaN through every later operation), the map is flagged after the loop and
    // its costs are recomputed by the REDO launch on complete maps.  A genuine code -128, or a NaN cost without an
    // escape, only costs a redo that yields the same costs.
    if (MODE == WIN_DETECT && tid == 0) s_lutL[0] = __hiloint2double(0x7ff80000, 0);
    for (int i = tid; i < 2 * g.p.T; i += THREADS) s_u[i] = a.u_cur[i];

    sb_win = smem_u32(smem);
    sb_lutL = smem_u32(s_lutL) + 128 * 8;     // index by the signed int8 value directly
    sb_lutA = smem_u32(s_lutA) + 128 * 8;
    sb_u = smem_u32(s_u);
    // keep the shared-window addresses in registers (opaque to the optimiser, which would otherwise
    // re-derive them from SR_CgaCtaId with S2UR/ULEA inside the loop)
    asm volatile("" : "+r"(sb_win), "+r"(sb_lutL), "+r"(sb_lutA), "+r"(sb_u));
    xlo = p.g.xlo; ylo = p.g.ylo; res = p.g.res; inv_res = p.g.inv_res;
    gx = p.xgoal[0]; gy = p.xgoal[1];
    magic_wx = 0x4B400000 + a.wx0; magic_wy = 0x4B400000 + a.wy0;
    asm volatile("" : "+r"(magic_wx), "+r"(magic_wy));       // keep the folded constants (else re-derived per step)
    // interval half-width 2.4e-7 (relative): the exact quotient q = a/res satisfies |fl(a*fl(inv*(1-+d))) - q(1-+d)| <=
    // 3 * 2^-24 |q| = 1.79e-7 |q| (roundings of 1/res, of the scaled reciprocal, of the FMA), so d = 2.4e-7 keeps q
    // inside [lower end, upper end] with a third to spare; a wider interval only sends more steps to the exact sequence
    inv_lo = inv_res * (1.0f - 2.4e-7f); inv_hi = inv_res * (1.0f + 2.4e-7f);
    keep_in_registers(inv_lo, inv_hi);                       // (else re-derived from inv_res on every step)
    uww = (unsigned)a.ww; uwh = (unsigned)a.wh;              // staged AND inside the map (<= WW, WH)
  };
  int cur = -1;                                              // BATCH: the planner staged in s_rec
  if (!BATCH) stage_planner();

  const long long dbg_t0 = WIN_DBG(g) ? (long long)globaltimer_ns() : 0;
  uint32_t phase = 0;
  for (long long w = w_lo; w < w_hi;) {
    const int u = (int)(w / cpm);
    int m = BATCH ? u % g.p.M : u;
    if (MODE == WIN_REDO) {                                 // the u-th flagged map (CTA-uniform: every thread scans)
      for (int i = 0, seen = 0; i < g.p.M; ++i)
        if (g.esc[i] && seen++ == u) { m = i; break; }
    }
    const int c_lo = (int)(w - (long long)u * cpm);
    const int c_hi = (int)min((long long)cpm, w_hi - (long long)u * cpm);       // this map's part of the share
    w += c_hi - c_lo;
    if constexpr (BATCH) {
      if (active && !active[u / g.p.M]) continue;           // a stopped planner (closed-loop trials): CTA-uniform
    }
    __syncthreads();                                        // every warp has left the previous window (and the tables are written)
    if constexpr (BATCH) {
      const int k = u / g.p.M;                              // CTA-uniform
      if (k != cur) {
        cur = k;
        const unsigned* src = reinterpret_cast<const unsigned*>(descs + k);
        unsigned* dst = reinterpret_cast<unsigned*>(s_rec);
        for (int i = tid; i < (int)(sizeof(RolloutWinArgs) / 4); i += THREADS) dst[i] = src[i];
        tm_lin = tmaps + 4 * k; tm_ang = tm_lin + 1; tm_obs = tm_lin + 2; tm_unk = tm_lin + 3;
        if (tid == 0) {
          // tensor maps in global memory, written by a host copy: acquire them for the tensor-map proxy before use
          // (CUDA Programming Guide, tensor maps passed in global memory)
          for (int i = 0; i < 4; ++i)
            asm volatile ("fence.proxy.tensormap::generic.acquire.sys [%0], 128;" ::"l"(tm_lin + i) : "memory");
        }
        __syncthreads();                                    // the record is in shared memory
        stage_planner();                                    // the barrier after the TMA issue below publishes the tables
      }
    }
    if (tid == 0) {
      *s_next = c_lo;
      // order the CTA's generic-proxy reads of the previous window before the async-proxy writes of the next one
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      mbar_expect_tx(bar, 4u * (uint32_t)PLANE);
      tma_load_3d(smem, tm_lin, bar, a.wx0, a.wy0, m);
      tma_load_3d(smem + PLANE, tm_ang, bar, a.wx0, a.wy0, m);
      tma_load_2d(smem + 2 * PLANE, tm_obs, bar, a.wx0, a.wy0);
      tma_load_2d(smem + 3 * PLANE, tm_unk, bar, a.wx0, a.wy0);
    }
    __syncthreads();                                        // s_next visible
    mbar_wait(bar, phase);
    phase ^= 1u;
    // the barrier above releases all 32 warps in lockstep: they would hit the XU / LSU / FP64 sections of the step
    // together, pass after pass.  Spread the warps of a scheduler over one step period (a.stagger cycles per slot)
    if (g.stagger > 0) {
      const long long t0 = clock64();
      const long long wait = (long long)(tid >> 7) * g.stagger;
      while (clock64() - t0 < wait) { }
    }
    const int8_t* __restrict__ g_lin = a.lin_grid + (size_t)m * p.g.grid_rows * p.g.grid_pitch;
    const int8_t* __restrict__ g_ang = a.ang_grid + (size_t)m * p.g.grid_rows * p.g.grid_pitch;

    // How the warps get their chunks: from the shared counter (a warp that is done takes the next chunk; the hardware
    // favours some warps of a scheduler, they simply run more chunks and the issue slots stay full).  The alternative
    // kept for A/B timing (a.sync_passes, B200MPPI_WIN_SYNC=1): pass by pass -- warp w takes chunk c_lo + 32*pass + w and
    // the CTA meets at a barrier after every pass.  It is slower even for two-pass shares: a pass started in lockstep
    // ends with its low-priority warps running alone at a fraction of the issue rate.
    for (int pass = 0;; ++pass) {
      int c;
      if (g.sync_passes) {
        if (c_lo + pass * (THREADS / 32) >= c_hi) break;    // CTA-uniform
        if (pass > 0) __syncthreads();
        c = c_lo + pass * (THREADS / 32) + (tid >> 5);
      } else {
        c = 0;
        if (lane == 0) c = atomicAdd(s_next, 1);
        c = __shfl_sync(0xffffffffu, c, 0);
        if (c >= c_hi) break;
      }
      const bool has = c < c_hi;                            // pass mode: no chunk left for this warp in the last pass
      const int n = has ? (c << 5) + lane : lane;
      const bool live = has && n < g.p.N;                   // ragged last chunk (n is padded to whole warps): such lanes
      const int Tn = live ? g.p.T : 0;                      // run zero steps and store nothing, but stay with their warp
    const double2* __restrict__ ep = reinterpret_cast<const double2*>(a.noiseT) + n;
    float x = p.x0[0], y = p.x0[1], th = p.x0[2];
    // the float64 state is carried UNROUNDED across the back edge (rx, ry, rt: the float64 FMA results, initially the
    // float32 state itself) and rounded to float32 precision at the top of the next step: the FMA of a step then
    // writes straight into the carried registers (no register moves at the end of the loop body)
    double rx = widen(x), ry = widen(y), rt = widen(th);
    float cost = 0.0f, d2 = 1e9f;
    double2 c2 = __ldg(ep);                                 // controls of step t (loaded during step t-1, see below)
    int t = 0;
    for (; t < Tn; ++t) {
      ep += g.npad;
      // ---- cell index of both axes: floor(a/res) by round-down magic-number addition on the FP32 pipe, taken
      //      at BOTH ends of an interval that contains the exact quotient a/res (relative half-width 2.4e-7,
      //      1.34x the worst accumulated rounding error, see inv_lo / inv_hi; the +-1e-30 covers a == 0 and flushed
      //      denormals).  Equal floors at both ends prove the cell -- it is then what the reference's exact
      //      sequence (the true floor of a/res) yields; otherwise run that sequence.
      const float ax = fsub(x, xlo), ay = fsub(y, ylo);
      const float kx = __fadd_rd(fmaf(ax, inv_lo, -1e-30f), MAGIC), kx2 = __fadd_rd(fmaf(ax, inv_hi, 1e-30f), MAGIC);
      const float ky = __fadd_rd(fmaf(ay, inv_lo, -1e-30f), MAGIC), ky2 = __fadd_rd(fmaf(ay, inv_hi, 1e-30f), MAGIC);
      // window-relative cell straight from the magic-number sums (bits(k) - bits(MAGIC) = floor)
      int wx = __float_as_int(kx) - magic_wx, wy = __float_as_int(ky) - magic_wy;
      // ---- traction / mask lookup.  ONE rare region for everything that is not "cell proven and staged": an
      //      integer may lie inside one of the intervals (run the exact reference sequence), or the cell lies outside
      //      the staged window (read global memory; out-of-map indices wrap + clamp like the generic kernel)
      int ql, qa, ob, un;
      const bool fast = (__float_as_int(kx) == __float_as_int(kx2)) & (__float_as_int(ky) == __float_as_int(ky2)) &
                        ((unsigned)wx < uww) & ((unsigned)wy < uwh);
      if (__builtin_expect(fast, 1)) {
        const uint32_t ad = sb_win + (uint32_t)(wy * WW + wx);
        ql = lds_s8(ad, 0); qa = lds_s8(ad, PLANE); ob = lds_s8(ad, 2 * PLANE); un = lds_s8(ad, 3 * PLANE);
      } else {
        if (WIN_DBG(g)) {                                   // debug hook: lane-steps on the slow path / outside the window
          atomicAdd(reinterpret_cast<unsigned long long*>(g.dbg) + 6 * blockIdx.x + 4, 1ull);
          if (!(((unsigned)wx < uww) & ((unsigned)wy < uwh)))
            atomicAdd(reinterpret_cast<unsigned long long*>(g.dbg) + 6 * blockIdx.x + 5, 1ull);
        }
        const int pk = lookup_slow<WW, PLANE, MODE == WIN_DETECT>(ax, ay, res, inv_lo, inv_hi, sb_win, uww, uwh, a.wx0, a.wy0,
                                                                  p.g.rows, p.g.cols, p.g.grid_rows, p.g.grid_cols,
                                                                  p.g.grid_pitch, p.g.mask_pitch, g_lin, g_ang, a.obstacle,
                                                                  a.unknown);
        ql = (int)(int8_t)pk; qa = (int)(int8_t)(pk >> 8); ob = (int)(int8_t)(pk >> 16); un = pk >> 24;
      }
      // ---- noisy clipped control (mppi.py:686-689): `c2`, precomputed per (n, t) by the prepare kernel
      // ---- unicycle step (mppi.py:692-694): float64 FMA, one rounding to float32 per component.  The
      //      float64 copies hold the float32-rounded state, so the reference's f2d(x) costs nothing.
      const double dv = lds_f64(sb_lutL + (uint32_t)(ql * 8)) * c2.x;
      const float cs = cos_approx(th);
      const float sn = sin_approx(th);
      // float64 copies of the float32-rounded state, without a second XU-pipe conversion (widen(narrow(.)) was
      // slower: the XU pipe is this kernel's busiest)
      const double x64 = round_to_f32_precision(rx);
      const double y64 = round_to_f32_precision(ry);
      const double th64 = round_to_f32_precision(rt);
      rx = fma(dv, widen(cs), x64);
      ry = fma(dv, widen(sn), y64);
      rt = fma(lds_f64(sb_lutA + (uint32_t)(qa * 8)), c2.y, th64);
      // `c2` is dead from here on: fetch the next step's controls straight into it -- the rest of this step and the
      // cell lookup of the next one (~70 instructions per warp, 32 warps per SM) cover the L2 latency
      c2 = __ldg(ep);                                       // (row T exists: the buffer has T + 1 rows, no guard needed)
      x = narrow(rx); y = narrow(ry); th = narrow(rt);
      // ---- stage cost (mppi.py:696-701)
      const float dx = fsub(gx, x), dy = fsub(gy, y);
      d2 = ffma(dx, dx, fmul(dy, dy));
      cost = fadd(cost, ffma(sqrt_approx(d2), p.dist_weight, p.dt));
      if (MASK01) {
        // ffma(1, c, cost) == cost + c and ffma(0, c, cost) == cost == cost + 0: add c or +0.0, selected by an integer
        // multiply of c's bit pattern with the mask byte (no predicate, no branch, no conversion)
        cost = fadd(cost, __int_as_float(ob * __float_as_int(p.obs_cost)));
        cost = fadd(cost, __int_as_float(un * __float_as_int(p.unk_cost)));
      } else if ((ob | un) != 0) {
        cost = add_penalties(cost, ob, un, p.obs_cost, p.unk_cost);
      }
      if (d2 <= p.tol2) break;                              // goal reached (mppi.py:703-706)
    }
    // the loop is left early exactly when d2 <= tol2 and otherwise ends with d2 > tol2 (d2 = 1e9 for T = 0), so the
    // reference's goal_reached flag is recovered from d2 -- no flag register (and no constant) inside the loop
    if (WIN_DBG(g)) {                                       // debug hook: steps this warp ran for the chunk (its slowest lane)
      const int steps = __reduce_max_sync(0xffffffffu, t < Tn ? t + 1 : t);
      if (lane == 0) atomicAdd(reinterpret_cast<unsigned long long*>(g.dbg) + 6 * blockIdx.x + 5, (unsigned long long)steps << 40);
    }
    const float not_reached = (d2 <= p.tol2) ? 0.0f : 1.0f;
    cost = fadd(cost, a.ctrl[n]);                                           // control cost (mppi.py:708-710)
    const double num = f2d(not_reached) * f2d(sqrt_approx(d2));              // terminal cost (mppi.py:26-28)
    cost = fadd(cost, d2f(num / (f2d(p.v_post) + 1e-6)));
    // plain byte store, no ordering needed.  Only live lanes read cells: a padding lane's cost adds ctrl[n] beyond N,
    // which nothing writes (whatever the allocation held, NaN included), and must not flag the map
    if (MODE == WIN_DETECT && live && cost != cost) a.esc[m] = 1;
    if (live) *cost_ptr(a.dst, m, n) = cost;                // map-major: the warp's 32 lanes store one 128-byte line
    }
  }
  if (WIN_DBG(g)) __syncthreads();                          // the CTA's end, not the end of thread 0's warp
  if (WIN_DBG(g) && tid == 0) {                                // per-CTA wall time (tools/rollout_cta_times.py)
    g.dbg[6 * blockIdx.x + 0] = dbg_t0;
    g.dbg[6 * blockIdx.x + 1] = (long long)globaltimer_ns();
    g.dbg[6 * blockIdx.x + 2] = w_lo | ((long long)sm_id() << 40);           // SM id in the upper bits
    g.dbg[6 * blockIdx.x + 3] = w_hi;
  }
  // sharded solve, peer-memory exchange: the costs above went straight into the receive buffers of the ranks that
  // reduce them; the LAST CTA to get here raises this rank's epoch flag in every peer (p2p.cu has the protocol)
  if (g.sig.ws > 0) {
    // one fence per CTA: the barrier orders every thread's cost stores before thread 0, whose (cumulative) system-scope
    // fence then orders them before its ticket -- the pattern of a cooperative grid barrier.  (A fence by each of the
    // 1024 threads, as in the first version, is slower with stores in flight over NVLink.)
    if (g.stagger == -1) __threadfence_system();            // A/B hook: the first version
    __syncthreads();
    if (tid == 0) {
      __threadfence_system();
      const unsigned prev = atomicAdd(g.sig.counter, 1u);
      if (prev == gridDim.x - 1) {
        *g.sig.counter = 0;
        __threadfence_system();
        for (int q = 0; q < g.sig.ws; ++q) st_flag_sys(g.sig.peer_flags[q] + g.sig.rank, g.sig.epoch);
      }
    }
  }
}

// MODE: WIN_WHOLE (complete maps), WIN_DETECT (window-first sampling: flag the maps whose lanes escape, a.esc) or
// WIN_REDO (rerun the flagged maps once completed: same body, same lane arithmetic)
template <int THREADS, int WH, bool MASK01, int MODE = WIN_WHOLE>
__global__ void __launch_bounds__(THREADS, 1) rollout_win_kernel(const RolloutWinArgs a,
                                                                 const __grid_constant__ CUtensorMap tm_lin,
                                                                 const __grid_constant__ CUtensorMap tm_ang,
                                                                 const __grid_constant__ CUtensorMap tm_obs,
                                                                 const __grid_constant__ CUtensorMap tm_unk) {
  rollout_win_body<THREADS, WH, MASK01, false, MODE>(a, &tm_lin, &tm_ang, &tm_obs, &tm_unk, nullptr, nullptr, 1, nullptr);
}

// [emu:end win_kernel]
// [emu:begin win_batch]
template <int THREADS, int WH, bool MASK01>
__global__ void __launch_bounds__(THREADS, 1) rollout_win_batch_kernel(const RolloutWinArgs g,
                                                                       const RolloutWinArgs* __restrict__ descs,
                                                                       const CUtensorMap* __restrict__ tmaps, int count,
                                                                       const int* __restrict__ active = nullptr) {
  rollout_win_body<THREADS, WH, MASK01, true>(g, nullptr, nullptr, nullptr, nullptr, descs, tmaps, count, active);
}
// [emu:end win_batch]
// ---------------------------------------------------------------------------------------------
// host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// uint8 tensor map: rank 3 (cols, rows, maps) or rank 2 (cols, rows); box = (WW, WH[, 1])
bool make_u8_tensor_map(void* out_map, const void* base, int rank, int cols, int rows, int maps, int pitch,
                        int WW, int WH) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)maps};
  cuuint64_t strides[2] = {(cuuint64_t)pitch, (cuuint64_t)pitch * (cuuint64_t)rows};
  cuuint32_t box[3] = {(cuuint32_t)WW, (cuuint32_t)WH, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = fn(reinterpret_cast<CUtensorMap*>(out_map), CU_TENSOR_MAP_DATA_TYPE_UINT8, (cuuint32_t)rank,
                        const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

constexpr int WIN_THREADS = 1024;
static long long* win_debug_buffer = nullptr;   // b200mppi_debug_rollout_cta_times: 6 x int64 per CTA (start ns, end ns, share lo / hi,
                                                // lane-steps on the slow path, of which outside the window)
void rollout_win_set_debug(long long* dev) { win_debug_buffer = dev; }
constexpr int WIN_SYNC_MAX_PASSES = 0;    // shares of at most this many passes are run pass by pass (see the kernel);
                                          // 0 = never: slower than the shared counter even at 2 passes per CTA (a rank
                                          // of an 8-GPU solve) -- a pass started in lockstep ends
                                          // with its low-priority warps alone, the counter keeps the favoured warps busy
constexpr int WIN_STAGGER_DEFAULT = 0;    // cycles between the warps of a scheduler after a window barrier (B200MPPI_WIN_STAGGER)
static int win_grid_override = 0;         // B200MPPI_WIN_GRID (tuning / test hook): number of persistent CTAs
constexpr int WIN_MAX_SMEM = 232448;      // 227 KB: per-block opt-in limit on sm_90 (H100)

void rollout_win_geometry(int T, int* WW, int* WH, size_t* smem) {
  // 4 byte planes + tables must fit 227 KB; inner box extent a multiple of 16 B and <= 256; plane size a
  // multiple of 128 B (TMA destination alignment).  Two compiled heights: 232 rows (T <= 700), 224 rows.
  const int wh = (win_smem_layout(WIN_WW, 232, T).total <= WIN_MAX_SMEM) ? 232 : 224;
  *WW = WIN_WW; *WH = wh;
  *smem = (size_t)win_smem_layout(WIN_WW, wh, T).total;
}

int rollout_win_threads() { return WIN_THREADS; }

int device_sm_count() {
  int dev = 0, sms = 132;                                   // H100 SXM
  cudaGetDevice(&dev);
  static int sm_count[64] = {};
  if (dev >= 0 && dev < 64) {
    if (!sm_count[dev]) cudaDeviceGetAttribute(&sm_count[dev], cudaDevAttrMultiProcessorCount, dev);
    if (sm_count[dev] > 0) sms = sm_count[dev];
  }
  return sms;
}

cudaError_t launch_rollout_win(const RolloutWinArgs& a, const void* tm_lin, const void* tm_ang, const void* tm_obs,
                               const void* tm_unk, cudaStream_t st) {
  const WinSmem L = win_smem_layout(a.WW, a.WH, a.p.T);
  typedef void (*WinKernel)(const RolloutWinArgs, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap);
  static const WinKernel kernels[3][2][2] = {
      {{rollout_win_kernel<WIN_THREADS, 232, false, WIN_WHOLE>, rollout_win_kernel<WIN_THREADS, 232, true, WIN_WHOLE>},
       {rollout_win_kernel<WIN_THREADS, 224, false, WIN_WHOLE>, rollout_win_kernel<WIN_THREADS, 224, true, WIN_WHOLE>}},
      {{rollout_win_kernel<WIN_THREADS, 232, false, WIN_DETECT>, rollout_win_kernel<WIN_THREADS, 232, true, WIN_DETECT>},
       {rollout_win_kernel<WIN_THREADS, 224, false, WIN_DETECT>, rollout_win_kernel<WIN_THREADS, 224, true, WIN_DETECT>}},
      {{rollout_win_kernel<WIN_THREADS, 232, false, WIN_REDO>, rollout_win_kernel<WIN_THREADS, 232, true, WIN_REDO>},
       {rollout_win_kernel<WIN_THREADS, 224, false, WIN_REDO>, rollout_win_kernel<WIN_THREADS, 224, true, WIN_REDO>}}};
  {
    // the opt-in is per device (per-context function): a process may run planners on several GPUs
    static bool attr_set[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !attr_set[dev]) {
      for (int r = 0; r < 3; ++r)
        for (int i = 0; i < 2; ++i)
          for (int j = 0; j < 2; ++j) {
            const cudaError_t e = cudaFuncSetAttribute(kernels[r][i][j], cudaFuncAttributeMaxDynamicSharedMemorySize, WIN_MAX_SMEM);
            if (e != cudaSuccess) return e;
          }
      if (dev >= 0 && dev < 64) attr_set[dev] = true;
    }
  }
  if (a.WW != WIN_WW || (a.WH != 232 && a.WH != 224) || L.total > WIN_MAX_SMEM) return cudaErrorInvalidValue;
  // persistent: one CTA per SM (1024 threads and 222 KB of shared memory fill an SM), never more CTAs than chunks
  const int sms = device_sm_count();
  static bool env_read = false;
  if (!env_read) {
    if (const char* e = getenv("B200MPPI_WIN_GRID")) win_grid_override = atoi(e);
    env_read = true;
  }
  // every SM takes part as soon as there are 8 chunks (256 rollouts) for each; smaller problems use fewer CTAs
  const long long total = (long long)a.p.M * (a.npad / 32);
  const int ctas = (int)std::min<long long>(std::max<long long>(total / 8, 1), sms);
  const dim3 grid(win_grid_override > 0 ? win_grid_override : ctas);
  RolloutWinArgs b = a;
  static int stagger = WIN_STAGGER_DEFAULT;
  static bool stagger_read = false;
  if (!stagger_read) {
    if (const char* e = getenv("B200MPPI_WIN_STAGGER")) stagger = atoi(e);
    stagger_read = true;
  }
  b.stagger = stagger;
  static int rotate = -1;
  if (rotate < 0) { const char* e = getenv("B200MPPI_WIN_ROTATE"); rotate = e ? atoi(e) : 0; if (rotate < 0) rotate = 0; }
  b.rotate = rotate;
  b.dbg = win_debug_buffer;
  static int sync_mode = -1;                                // B200MPPI_WIN_SYNC = 0 | 1 (A/B hook), default: by share length
  static bool sync_read = false;
  if (!sync_read) {
    if (const char* e = getenv("B200MPPI_WIN_SYNC")) sync_mode = atoi(e);
    sync_read = true;
  }
  // whole passes (32 chunks) per share once a share is at least 4 passes long (no end-of-segment stragglers); shorter
  // shares stay chunk-granular: rounding a fractional pass count per CTA (a rank of a 4-GPU solve) to a whole one costs
  // more than it saves
  b.unit = (total / (32LL * grid.x) >= 4) ? 32 : ((int)grid.x >= a.p.M ? 0 : 1);
  static int unit_override = -1;                            // B200MPPI_WIN_UNIT = 0 | 1 | 32 (A/B hook)
  static bool unit_read = false;
  if (!unit_read) {
    if (const char* e = getenv("B200MPPI_WIN_UNIT")) unit_override = atoi(e);
    unit_read = true;
  }
  if (unit_override == 1 || unit_override == 32 || (unit_override == 0 && (int)grid.x >= a.p.M)) b.unit = unit_override;
  if (a.redo) b.unit = 1;                                   // a few flagged maps over every CTA, chunk by chunk
  const long long passes = (total + 32LL * grid.x - 1) / (32LL * grid.x);
  b.sync_passes = sync_mode >= 0 ? (sync_mode != 0) : (passes <= WIN_SYNC_MAX_PASSES);
  const CUtensorMap& t0 = *reinterpret_cast<const CUtensorMap*>(tm_lin);
  const CUtensorMap& t1 = *reinterpret_cast<const CUtensorMap*>(tm_ang);
  const CUtensorMap& t2 = *reinterpret_cast<const CUtensorMap*>(tm_obs);
  const CUtensorMap& t3 = *reinterpret_cast<const CUtensorMap*>(tm_unk);
  kernels[!a.esc ? WIN_WHOLE : a.redo ? WIN_REDO : WIN_DETECT][a.WH == 232 ? 0 : 1][a.masks01 ? 1 : 0]<<<grid, WIN_THREADS, L.total, st>>>(b, t0, t1, t2, t3);
  return cudaGetLastError();
}

// the planner record the batched kernel keeps behind the window
static size_t win_batch_smem(int WH, int T) {
  return (size_t)win_smem_layout(WIN_WW, WH, T).total + sizeof(RolloutWinArgs);
}

int rollout_win_batch_height(int T) { return win_batch_smem(232, T) <= (size_t)WIN_MAX_SMEM ? 232 : 224; }

// The launch-wide choices of launch_rollout_win (persistent CTAs, share unit) over units = count * M; its tuning hooks
// (B200MPPI_WIN_*) and the debug hook are not applied to batched launches.
cudaError_t launch_rollout_win_batch(const RolloutWinArgs& g, const RolloutWinArgs* descs, const void* tmaps, int count,
                                     bool masks01, const int* active, cudaStream_t st) {
  typedef void (*WinBatchKernel)(const RolloutWinArgs, const RolloutWinArgs*, const CUtensorMap*, int, const int*);
  static const WinBatchKernel kernels[2][2] = {
      {rollout_win_batch_kernel<WIN_THREADS, 232, false>, rollout_win_batch_kernel<WIN_THREADS, 232, true>},
      {rollout_win_batch_kernel<WIN_THREADS, 224, false>, rollout_win_batch_kernel<WIN_THREADS, 224, true>}};
  {
    static bool attr_set[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !attr_set[dev]) {
      for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2; ++j) {
          const cudaError_t e = cudaFuncSetAttribute(kernels[i][j], cudaFuncAttributeMaxDynamicSharedMemorySize, WIN_MAX_SMEM);
          if (e != cudaSuccess) return e;
        }
      if (dev >= 0 && dev < 64) attr_set[dev] = true;
    }
  }
  const size_t smem = win_batch_smem(g.WH, g.p.T);
  if (g.WW != WIN_WW || (g.WH != 232 && g.WH != 224) || smem > (size_t)WIN_MAX_SMEM || count < 1) return cudaErrorInvalidValue;
  const int units = count * g.p.M;
  const long long total = (long long)units * (g.npad / 32);
  const dim3 grid((unsigned)std::min<long long>(std::max<long long>(total / 8, 1), device_sm_count()));
  RolloutWinArgs b = g;
  b.unit = (total / (32LL * grid.x) >= 4) ? 32 : ((int)grid.x >= units ? 0 : 1);
  b.sync_passes = (total + 32LL * grid.x - 1) / (32LL * grid.x) <= WIN_SYNC_MAX_PASSES;
  b.stagger = WIN_STAGGER_DEFAULT; b.rotate = 0; b.dbg = nullptr; b.sig = CostSignal{};
  kernels[g.WH == 232 ? 0 : 1][masks01 ? 1 : 0]<<<grid, WIN_THREADS, smem, st>>>(
      b, descs, reinterpret_cast<const CUtensorMap*>(tmaps), count, active);
  return cudaGetLastError();
}

}  // namespace b200
