// common.cuh -- shared device helpers of the MPPI engine (sm_90a, H100).
//
// The arithmetic helpers mirror, instruction for instruction, what NVVM emits for the reference's
// Numba kernels with fastmath=True (PTX census: SURVEY.md 2.3; re-derived with
// numba.cuda.compile_ptx of mppi_numba/mppi.py).  They are written as inline PTX so that nvcc
// cannot re-associate or re-contract them: parity with the reference is decided by these.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

// ---------------------------------------------------------------- approximate f32 ops (MUFU paths)
__device__ __forceinline__ float sin_approx(float x) {
  float r; asm("sin.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r;
}
__device__ __forceinline__ float cos_approx(float x) {
  float r; asm("cos.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r;
}
__device__ __forceinline__ float sqrt_approx(float x) {
  float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r;
}
__device__ __forceinline__ float div_approx(float a, float b) {
  float r; asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float div_full(float a, float b) {
  float r; asm("div.full.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float div_rn(float a, float b) {
  float r; asm("div.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
// explicitly rounded, never contracted
__device__ __forceinline__ float fadd(float a, float b) {
  float r; asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float fsub(float a, float b) {
  float r; asm("sub.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float fmul(float a, float b) {
  float r; asm("mul.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r;
}
__device__ __forceinline__ float ffma(float a, float b, float c) {
  float r; asm("fma.rn.ftz.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c)); return r;
}
__device__ __forceinline__ float ffloor(float a) {
  float r; asm("cvt.rmi.ftz.f32.f32 %0, %1;" : "=f"(r) : "f"(a)); return r;
}
__device__ __forceinline__ double f2d(float a) {          // cvt.ftz.f64.f32
  double r; asm("cvt.ftz.f64.f32 %0, %1;" : "=d"(r) : "f"(a)); return r;
}
__device__ __forceinline__ float d2f(double a) {          // cvt.rn.ftz.f32.f64
  float r; asm("cvt.rn.ftz.f32.f64 %0, %1;" : "=f"(r) : "d"(a)); return r;
}

// ---------------------------------------------------------------- Python float32 `//` as Numba lowers it
// int32((x - lo) // res)   (mppi.py:679-680).  EXACT mirror of what runs on the GPU
// (numba/cpython/numbers.py real_divmod -> abs, div.rn, floor, remainder, div.full, sign fix, floor,
// snap-to-nearest, cvt.rzi).  NVVM emits the remainder as `mul.ftz.f32` + `sub.ftz.f32` WITHOUT a
// rounding modifier, which ptxas contracts into one FFMA (verified in the SASS of the reference's
// PTX and by state traces against the reference on the GPU): the remainder is exact,
// so the sequence yields the true floor of a/res.  `a` is already the float32 difference x - lo.
// [emu:begin cell_index]
static __device__ __noinline__ int cell_index_exact(float a, float r) {
  if (r == 0.0f) return (int)div_full(a, r);
  const float aa = fabsf(a), rr = fabsf(r);
  const float t = div_rn(aa, rr);
  float m = ffma(-ffloor(t), rr, aa);           // FFMA.FTZ m = -floor(t)*|r| + |a|  (contracted)
  m = (a < 0.0f) ? -m : m;
  float q = div_full(fsub(a, m), r);
  if (m != 0.0f && ((r < 0.0f) != (m < 0.0f))) q = fadd(q, -1.0f);
  float res;
  if (q == 0.0f || q != q) {
    res = div_full(fmul(a, fmul(q, q)), r);
  } else {
    const float fl = ffloor(q);
    res = (fsub(q, fl) > 0.5f) ? fadd(fl, 1.0f) : fl;
  }
  int k; asm("cvt.rzi.ftz.s32.f32 %0, %1;" : "=r"(k) : "f"(res));
  return k;
}

// Fast path: floor(a * (1/r)) is provably the same integer unless a/r lies within a few ulp of an
// integer (|y - a/r| <= 2^-23 |y|); only then run the exact sequence.  Keeps the hot loop at a
// handful of instructions while staying bit-identical to the reference's cell choice.
__device__ __forceinline__ int cell_index(float a, float r, float inv_r) {
  const float y = a * inv_r;
  const float fl = floorf(y);
  const float frac = y - fl;
  const float eps = fmaf(fabsf(y), 4.8e-7f, 1e-6f);
  if (frac > eps && frac < 1.0f - eps) return (int)fl;
  return cell_index_exact(a, r);
}

// [emu:end cell_index]

// ---------------------------------------------------------------- xoroshiro128+ (numba/cuda/random.py:81-99)
// [emu:begin xoro]
struct Xoro { uint64_t s0, s1; };
__device__ __forceinline__ uint64_t rotl64(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
__device__ __forceinline__ uint64_t xoro_next(Xoro& s) {
  const uint64_t s0 = s.s0;
  uint64_t s1 = s.s1;
  const uint64_t result = s0 + s1;
  s1 ^= s0;
  s.s0 = rotl64(s0, 55) ^ s1 ^ (s1 << 14);
  s.s1 = rotl64(s1, 36);
  return result;
}
// [emu:end xoro]
// uint64_to_unit_float32 (random.py:130-154): float32( float64(x >> 11) * 2^-53 )
__device__ __forceinline__ float xoro_unit_f32(uint64_t x) {
  return __double2float_rn(__ull2double_rn(x >> 11) * (1.0 / 9007199254740992.0));
}

// xoroshiro128p_normal_float32 (numba/cuda/random.py:176-197): Box-Muller in float32, two draws,
// sine branch discarded.  Compiled by Numba this uses libdevice's PRECISE logf/cosf (the helper is
// jitted without the kernel's fastmath flag) and sqrt.approx.ftz (module-wide NVVM option) --
// SURVEY.md 2.3; logf/cosf below are the same libdevice routines.
// [emu:begin normal]
__device__ __forceinline__ float xoro_normal(Xoro& s) {
  const float u1 = xoro_unit_f32(xoro_next(s));
  const float u2 = xoro_unit_f32(xoro_next(s));
  const float two_pi = 6.283185307179586f;
  return fmul(sqrt_approx(fmul(-2.0f, logf(u1))), cosf(fmul(two_pi, u2)));
}
// [emu:end normal]

// Threshold of sample_grids_numba, q(r) = int8(ceil(f64(f32((r >> 11) * 2^-53)) * 100 * alpha)) (terrain.py:682-684),
// as a lookup on the RAW 64-bit draw r: q is a monotone step function of r; bucket = top 8 bits of r; inside a
// bucket q rises at most once, at the raw value thr[bucket] (thr = 0 with qbase = q - 1: "already risen").
// One 64-bit entry per bucket: thr | qbase.  The breakpoints are (53-bit draw) << 11, so the low 11 bits of thr are
// free and hold qbase (<= 127); r >= thr  <=>  (r | 0x7ff) >= (thr | qbase).
// Tables come from build_sample_thresholds (sample.cu), which verifies that alpha is representable this way.
// Shared by the sampler kernel and the host-side check b200mppi_debug_sample_threshold.
// [emu:begin threshold]
__host__ __device__ __forceinline__ uint32_t sample_threshold_q(uint64_t r, const uint64_t* table) {
  const uint64_t e = table[r >> 56];
  return ((uint32_t)e & 0x7ffu) + ((r | 0x7ffULL) >= e ? 1u : 0u);
}
// [emu:end threshold]

// ---------------------------------------------------------------- system-scope flags (peer-memory exchange)
__device__ __forceinline__ void st_flag_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_flag_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ unsigned sm_id() {
  unsigned v;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(v));
  return v;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// A kernel that consumes what the peers pushed (peer-memory exchange, p2p.cu): every CTA waits until flags[s] >= epoch
// for every rank s < ws (ws = 0: nothing to wait for) before it reads the data.  Bounded: after timeout_ns the wait
// gives up and records 1 + s in *status (the host reports it after the solve) -- a missing rank must not hang the GPU.
struct FlagWait {
  const uint32_t* flags;
  int ws;
  uint32_t epoch;
  unsigned long long timeout_ns;
  int* status;
};
__device__ __forceinline__ void flag_wait(const FlagWait& w) {
  if (w.ws <= 0) return;
  const int s = threadIdx.x;
  if (s < w.ws) {
    const uint64_t t0 = globaltimer_ns();
    unsigned spins = 0;
    while ((int32_t)(ld_flag_sys(w.flags + s) - w.epoch) < 0) {
      if ((++spins & 1023u) == 0 && globaltimer_ns() - t0 > w.timeout_ns) {
        atomicExch(w.status, 1 + s);
        break;
      }
    }
    __threadfence_system();
  }
  __syncthreads();
}

// ---------------------------------------------------------------- small reductions
// [emu:begin warp_min]
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// [emu:end warp_min]
// [emu:begin warp_sum]
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// [emu:end warp_sum]

// ---------------------------------------------------------------- kernel parameter blocks
// [emu:begin params]
struct MapGeom {
  float res, inv_res;
  float xlo, ylo;          // padded_xlimits[0], padded_ylimits[0]
  int rows, cols;          // padded map Hp, Wp (mask shape)
  int grid_rows, grid_cols;  // Rmax, Cmax of the sample buffers (allocation dims)
  int grid_pitch;          // bytes per row of the sample buffers (>= grid_cols, multiple of 16)
  int mask_pitch;          // bytes per row of the obstacle / unknown / risk planes (multiple of 16)
};

struct RolloutParams {
  MapGeom g;
  float dt, x0[3], xgoal[2], tol2, v_post, lambda, u_std[2], vrange[2], wrange[2];
  float obs_cost, unk_cost, dist_weight;
  float lin_lo, ang_lo;
  double lin_ratio, ang_ratio;   // 0.01*(hi-lo) in float64 (mppi.py:674-675)
  int T, N, M;                   // N = local rollouts of this rank
};

// [emu:end params]
}  // namespace b200
