// rollout.cu -- the N x M x T unicycle rollout with cost accumulation, CVaR over M, and the
// visualisation rollouts.  Reference: mppi_numba/mppi.py:613-755 (rollout_numba), :916-1009
// (rollout_det_dyn_numba), :1013-1111 (rollout_det_dyn_w_speed_map_numba), :1194-1351 (vis).
//
// Arithmetic mirrors the compiled reference kernels operation by operation (float64 FMA state
// update rounded once to float32, approximate sin/cos/sqrt, the exact FMA contractions NVVM chose);
// see common.cuh.  What is re-designed is everything around that arithmetic: thread mapping
// (lanes of a warp share a MAP and differ in control sequence n, the reference does the opposite),
// memory staging, and the reduction.
#include "kernels.h"

namespace b200 {

// [emu:begin rollout]
// ---------------------------------------------------------------------------------------------
// One state step, shared by every rollout flavour.  Returns the squared goal distance.
struct StepConst {
  float xlo, ylo, res, inv_res;
  float v_lo, v_hi, w_lo, w_hi;
  float gx, gy, dt, w_dist;
  double dt64, lin_ratio, ang_ratio, lin_lo64, ang_lo64;
};

__device__ __forceinline__ StepConst make_step_const(const RolloutParams& p) {
  StepConst c;
  c.xlo = p.g.xlo; c.ylo = p.g.ylo; c.res = p.g.res; c.inv_res = p.g.inv_res;
  c.v_lo = p.vrange[0]; c.v_hi = p.vrange[1]; c.w_lo = p.wrange[0]; c.w_hi = p.wrange[1];
  c.gx = p.xgoal[0]; c.gy = p.xgoal[1]; c.dt = p.dt; c.w_dist = p.dist_weight;
  c.dt64 = f2d(p.dt); c.lin_ratio = p.lin_ratio; c.ang_ratio = p.ang_ratio;
  c.lin_lo64 = f2d(p.lin_lo); c.ang_lo64 = f2d(p.ang_lo);
  return c;
}

// wrap negative indices like Numba's array indexing does (PTX: selp shape, 0 on idx < 0), then clamp
// so that an out-of-map state can never read outside the allocation (the reference has no bounds
// check at all -- README.md:164-165; inside the padded map both are no-ops).
__device__ __forceinline__ int wrap_clamp(int i, int n) {
  i = (i < 0) ? i + n : i;
  return min(max(i, 0), n - 1);
}

// advance (x, y, th) by one step given the int8 traction percentages; mppi.py:682-694
__device__ __forceinline__ void unicycle_step(const StepConst& c, int ql, int qa, float v, float w,
                                              float& x, float& y, float& th) {
  const double vtr = fma(c.lin_ratio, (double)ql, c.lin_lo64);
  const double wtr = fma(c.ang_ratio, (double)qa, c.ang_lo64);
  const double dv = (vtr * c.dt64) * f2d(v);
  const float cs = cos_approx(th);
  const float sn = sin_approx(th);
  x = d2f(fma(dv, f2d(cs), f2d(x)));
  y = d2f(fma(dv, f2d(sn), f2d(y)));
  th = d2f(fma(wtr * c.dt64, f2d(w), f2d(th)));
}

__device__ __forceinline__ float goal_dist2(const StepConst& c, float x, float y) {
  const float dx = fsub(c.gx, x);
  const float dy = fsub(c.gy, y);
  return ffma(dx, dx, fmul(dy, dy));
}

// terminal cost, mppi.py:26-28:  float32( ((1 - reached) * f64(sqrt(d2))) / (f64(v_post) + 1e-6) )
__device__ __forceinline__ float term_cost(float d2, float v_post, bool reached) {
  const double num = (1.0 - (reached ? 1.0 : 0.0)) * f2d(sqrt_approx(d2));
  return d2f(num / (f2d(v_post) + 1e-6));
}

// one term of the control cost, mppi.py:708-710
__device__ __forceinline__ float ctrl_term(float u0, float u1, float e0, float e1, float sv2, float sw2) {
  const float a = div_approx(u0, sv2);
  const float b = div_approx(u1, sw2);
  return ffma(a, e0, fmul(b, e1));
}

// ---------------------------------------------------------------------------------------------
// Generic rollout kernel: one thread per (n, m); lanes of a warp = consecutive n on the SAME map.
// MODE 0: stochastic (per-(m,n) cost -> a.dst);  MODE 1: det dynamics;  MODE 2: nominal + speed map.
template <int MODE>
__device__ __forceinline__ void rollout_body(const RolloutArgs& a) {
  const RolloutParams& p = a.p;
  extern __shared__ float s_u[];           // u_cur (T,2)
  for (int i = threadIdx.x; i < 2 * p.T; i += blockDim.x) s_u[i] = a.u_cur[i];
  __syncthreads();

  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = (MODE == 0) ? blockIdx.y : 0;
  if (n >= p.N) return;

  const StepConst c = make_step_const(p);
  const int8_t* __restrict__ lin = a.lin_grid + (size_t)m * p.g.grid_rows * p.g.grid_pitch;
  const int8_t* __restrict__ ang = a.ang_grid + (size_t)m * p.g.grid_rows * p.g.grid_pitch;
  const float2* __restrict__ eps = reinterpret_cast<const float2*>(a.noise) + (size_t)n * p.T;

  float x = p.x0[0], y = p.x0[1], th = p.x0[2];
  float cost = 0.0f;
  float d2 = 1e9f;
  bool reached = false;

  for (int t = 0; t < p.T; ++t) {
    const int xi = cell_index(fsub(x, c.xlo), c.res, c.inv_res);
    const int yi = cell_index(fsub(y, c.ylo), c.res, c.inv_res);
    const int gy = wrap_clamp(yi, p.g.grid_rows), gx = wrap_clamp(xi, p.g.grid_cols);
    const int my = wrap_clamp(yi, p.g.rows), mx = wrap_clamp(xi, p.g.cols);
    const int ql = __ldg(lin + (size_t)gy * p.g.grid_pitch + gx);
    const int qa = __ldg(ang + (size_t)gy * p.g.grid_pitch + gx);
    const int ob = __ldg(a.obstacle + (size_t)my * p.g.mask_pitch + mx);
    const int un = __ldg(a.unknown + (size_t)my * p.g.mask_pitch + mx);
    const float2 e = __ldg(eps + t);
    const float v = fmaxf(c.v_lo, fminf(c.v_hi, fadd(s_u[2 * t], e.x)));
    const float w = fmaxf(c.w_lo, fminf(c.w_hi, fadd(s_u[2 * t + 1], e.y)));

    unicycle_step(c, ql, qa, v, w, x, y, th);
    d2 = goal_dist2(c, x, y);

    float dt_eff = c.dt;
    if (MODE == 2) {
      const int rk = __ldg(a.risk + (size_t)my * p.g.mask_pitch + mx);
      const double eff = fma(c.lin_ratio, (double)rk, c.lin_lo64);
      dt_eff = d2f(c.dt64 / (eff + 1e-6));
    }
    cost = fadd(cost, ffma(sqrt_approx(d2), c.w_dist, dt_eff));
    cost = ffma((float)ob, p.obs_cost, cost);
    cost = ffma((float)un, p.unk_cost, cost);
    if (d2 <= p.tol2) { reached = true; break; }
  }

  const float sv2 = fmul(p.u_std[0], p.u_std[0]);
  const float sw2 = fmul(p.u_std[1], p.u_std[1]);
  if (MODE == 0) {                      // control cost, then terminal (mppi.py:708-713)
    for (int t = 0; t < p.T; ++t) {
      const float2 e = __ldg(eps + t);
      cost = ffma(ctrl_term(s_u[2 * t], s_u[2 * t + 1], e.x, e.y, sv2, sw2), p.lambda, cost);
    }
    cost = fadd(cost, term_cost(d2, p.v_post, reached));
    *cost_ptr(a.dst, m, n) = cost;
  } else {                              // terminal, then control (mppi.py:1004-1009)
    cost = fadd(cost, term_cost(d2, p.v_post, reached));
    for (int t = 0; t < p.T; ++t) {
      const float2 e = __ldg(eps + t);
      cost = ffma(ctrl_term(s_u[2 * t], s_u[2 * t + 1], e.x, e.y, sv2, sw2), p.lambda, cost);
    }
    a.costs[n] = cost;
  }
}

template <int MODE>
__global__ void __launch_bounds__(128) rollout_kernel(const RolloutArgs a) {
  rollout_body<MODE>(a);
}

// ---------------------------------------------------------------------------------------------
// MODE 3: the map-free "barebone" MPPI of the reference's barebone_mppi_numba.ipynb (cell 3, rollout_numba):
// nominal float32 unicycle, stage cost w*d^2, circular obstacles, terminal cost (1-reached)*d^2.
// Contractions follow the SASS of the compiled notebook kernel (dv = FMUL(v, dt); x = FFMA(dv, cos, x);
// theta = FFMA(w, dt, theta); d^2 - r^2 as one FFMA; the obstacle indicator enters through a float64 FMA).
__device__ __forceinline__ void rollout_barebone_body(const RolloutArgs& a) {
  const RolloutParams& p = a.p;
  extern __shared__ float s_u[];
  for (int i = threadIdx.x; i < 2 * p.T; i += blockDim.x) s_u[i] = a.u_cur[i];
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= p.N) return;
  const float2* __restrict__ eps = reinterpret_cast<const float2*>(a.noise) + (size_t)n * p.T;
  const double obs_c64 = f2d(p.obs_cost);
  float x = p.x0[0], y = p.x0[1], th = p.x0[2];
  float cost = 0.0f, d2 = 1e9f;
  bool reached = false;
  for (int t = 0; t < p.T; ++t) {
    const float2 e = __ldg(eps + t);
    const float v = fmaxf(p.vrange[0], fminf(p.vrange[1], fadd(s_u[2 * t], e.x)));
    const float w = fmaxf(p.wrange[0], fminf(p.wrange[1], fadd(s_u[2 * t + 1], e.y)));
    const float dv = fmul(v, p.dt);
    const float cs = cos_approx(th), sn = sin_approx(th);
    x = ffma(dv, cs, x);
    y = ffma(dv, sn, y);
    th = ffma(w, p.dt, th);
    const float dx = fsub(p.xgoal[0], x), dy = fsub(p.xgoal[1], y);
    d2 = ffma(dx, dx, fmul(dy, dy));
    cost = ffma(d2, p.dist_weight, cost);
    for (int k = 0; k < a.num_obstacles; ++k) {
      const float ox = __ldg(a.obstacles + 3 * k), oy = __ldg(a.obstacles + 3 * k + 1), orad = __ldg(a.obstacles + 3 * k + 2);
      const float ddx = fsub(x, ox), ddy = fsub(y, oy);
      const float diff = ffma(-orad, orad, ffma(ddx, ddx, fmul(ddy, ddy)));
      const double inside = 1.0 - f2d(diff > 0.0f ? 1.0f : 0.0f);
      cost = d2f(fma(inside, obs_c64, f2d(cost)));
    }
    if (d2 <= p.tol2) { reached = true; break; }
  }
  cost = fadd(cost, d2f((reached ? 0.0 : 1.0) * f2d(d2)));
  const float sv2 = fmul(p.u_std[0], p.u_std[0]), sw2 = fmul(p.u_std[1], p.u_std[1]);
  for (int t = 0; t < p.T; ++t) {
    const float2 e = __ldg(eps + t);
    cost = ffma(ctrl_term(s_u[2 * t], s_u[2 * t + 1], e.x, e.y, sv2, sw2), p.lambda, cost);
  }
  a.costs[n] = cost;
}

__global__ void __launch_bounds__(128) rollout_barebone_kernel(const RolloutArgs a) {
  rollout_barebone_body(a);
}

// [emu:end rollout]
// [emu:begin rollout_batch]
// batched one-map solves (modes 1, 2, 3): planner blockIdx.y, its full RolloutArgs (geometry, maps, noise, u, costs)
// from the descriptor array; N and T are the batch's, so the grid and the 2T floats of shared memory are too.  A
// planner with active[y] == 0 is left untouched (active null: every planner runs)
template <int MODE>
__global__ void __launch_bounds__(128) rollout_batch_kernel(const RolloutArgs* __restrict__ descs,
                                                            const int* __restrict__ active = nullptr) {
  if (active && !active[blockIdx.y]) return;
  if constexpr (MODE == 3) rollout_barebone_body(descs[blockIdx.y]);
  else rollout_body<MODE>(descs[blockIdx.y]);
}

// mixed batches whose one-map planners mix det dynamics and speed map: each planner's rollout_body of its own mode
// (descs[y].mode, 1 or 2), gated by `active` as above
__global__ void __launch_bounds__(128) rollout_batch_mixed_kernel(const RolloutArgs* __restrict__ descs,
                                                                  const int* __restrict__ active = nullptr) {
  if (active && !active[blockIdx.y]) return;
  if (descs[blockIdx.y].mode == 1) rollout_body<1>(descs[blockIdx.y]);
  else rollout_body<2>(descs[blockIdx.y]);
}
// [emu:end rollout_batch]
void launch_rollout(const RolloutArgs& a, cudaStream_t st) {
  const int threads = 128;
  if (a.mode == 3) {
    rollout_barebone_kernel<<<(a.p.N + threads - 1) / threads, threads, (size_t)2 * a.p.T * sizeof(float), st>>>(a);
    return;
  }
  const dim3 grid((a.p.N + threads - 1) / threads, a.mode == 0 ? a.p.M : 1);
  const size_t smem = (size_t)2 * a.p.T * sizeof(float);
  if (a.mode == 0) rollout_kernel<0><<<grid, threads, smem, st>>>(a);
  else if (a.mode == 1) rollout_kernel<1><<<grid, threads, smem, st>>>(a);
  else rollout_kernel<2><<<grid, threads, smem, st>>>(a);
}

void launch_rollout_batch(const RolloutArgs* descs, int count, int mode, int N, int T, const int* active,
                          cudaStream_t st) {
  const int threads = 128;
  const dim3 grid((N + threads - 1) / threads, count);
  const size_t smem = (size_t)2 * T * sizeof(float);
  if (mode == ROLLOUT_MODE_PER_DESC) rollout_batch_mixed_kernel<<<grid, threads, smem, st>>>(descs, active);
  else if (mode == 1) rollout_batch_kernel<1><<<grid, threads, smem, st>>>(descs, active);
  else if (mode == 2) rollout_batch_kernel<2><<<grid, threads, smem, st>>>(descs, active);
  else rollout_batch_kernel<3><<<grid, threads, smem, st>>>(descs, active);
}

// ---------------------------------------------------------------------------------------------
// CVaR over the M map samples of one control sequence (mppi.py:718-755): mean of the
// numel = ceil(M * alpha) LARGEST costs.  One warp per n; the reference's O(M^2) odd-even sort with
// 2*ceil(M/2) block barriers is replaced by a bitwise radix SELECT of the numel-th largest key done
// with warp shuffles/ballots: 32 rounds of (compare, warp-sum), no shared memory, no barriers.
// [emu:begin cvar]   (tests/emu_cvar.py compiles the text between these markers for the host)
__device__ __forceinline__ uint32_t float_key(float f) {   // order-preserving float -> uint
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ float key_float(uint32_t k) {   // inverse of float_key
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

constexpr int CVAR_MAX_PER_LANE = 32;   // warp kernel: M <= 1024 (the reference's one-block limit, mppi.py:199)
constexpr int CVAR_LARGE_MAX_MAPS = 16384;   // CTA kernel: 64 KB of keys (Config clamps M to 15000, config.py:63)
constexpr int CVAR_THREADS = 256;
constexpr int CVAR_TILE_FLOATS = 8192 + 32;  // shared-memory tile of the warp kernel: NB control sequences x (M + 1)

// control sequences per CTA: 32 (one 128-byte line per map row) while the tile fits, fewer for many maps
__host__ __device__ inline int cvar_block_n(int M) {
  int nb = 32;
  while (nb > 1 && nb * (M + 1) > CVAR_TILE_FLOATS) nb >>= 1;
  return nb;
}

// costs_mn is map-major (M rows, row stride ld): a CTA loads the M x NB slab of its NB control sequences with
// coalesced row segments, transposes it through shared memory, then each warp selects for NB/8 of them.
// PER = values held per lane (compile time: the select loop is fully unrolled over them); value j = map j sits in
// slot j / 32 of lane j % 32 whatever the number of ranks the maps came from.
template <int PER>
__device__ __forceinline__ void cvar_body(const float* __restrict__ costs_mn, float* __restrict__ costs, int n_cnt, int ld,
                                          int M, int numel) {
  __shared__ float s_tile[CVAR_TILE_FLOATS];
  const int NB = cvar_block_n(M);
  const int n0 = blockIdx.x * NB;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // slab load: NB is a power of two; eight independent L2 loads in flight per thread before the shared-memory stores
  // (issue is in order: a store waiting for its load would hold back the next load)
  const int nb_shift = 31 - __clz(NB);
  for (int base = tid; base < M * NB; base += 8 * CVAR_THREADS) {
    float x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int idx = base + k * CVAR_THREADS;
      const int m = idx >> nb_shift, j = idx & (NB - 1);
      x[k] = (idx < M * NB && n0 + j < n_cnt) ? __ldcg(costs_mn + (size_t)m * ld + n0 + j) : 0.0f;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int idx = base + k * CVAR_THREADS;
      if (idx < M * NB) s_tile[(idx & (NB - 1)) * (M + 1) + (idx >> nb_shift)] = x[k];
    }
  }
  __syncthreads();
  for (int j = warp; j < NB; j += CVAR_THREADS / 32) {
    if (n0 + j >= n_cnt) break;                               // warp-uniform
    const float* row = s_tile + j * (M + 1);
    float v[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int k = i * 32 + lane;
      v[i] = (k < M) ? row[k] : -INFINITY;
    }
    float sum = 0.0f;
    if (numel >= M) {
#pragma unroll
      for (int i = 0; i < PER; ++i) if (i * 32 + lane < M) sum += v[i];
      sum = warp_sum(sum);
    } else {
      // find the key of the numel-th largest value
      uint32_t prefix = 0;
      for (int bit = 31; bit >= 0; --bit) {
        const uint32_t cand = prefix | (1u << bit);
        int cnt = 0;
#pragma unroll
        for (int i = 0; i < PER; ++i) cnt += (float_key(v[i]) >= cand) ? 1 : 0;
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (cnt >= numel) prefix = cand;
      }
      // sum everything strictly above the k-th key, then add the k-th value for the remaining slots
      // (all holders of the k-th key hold the same float: the key map is a bijection)
      int greater = 0;
#pragma unroll
      for (int i = 0; i < PER; ++i) {
        if (float_key(v[i]) > prefix) { sum += v[i]; ++greater; }
      }
      sum = warp_sum(sum);
      greater = __reduce_add_sync(0xffffffffu, greater);
      sum += (float)(numel - greater) * key_float(prefix);
    }
    if (lane == 0) costs[n0 + j] = (float)((double)sum / (double)numel);
  }
}

template <int PER>
__global__ void __launch_bounds__(CVAR_THREADS) cvar_kernel(const float* __restrict__ costs_mn,
                                                            float* __restrict__ costs, int n_cnt, int ld, int M, int numel,
                                                            const FlagWait fw) {
  flag_wait(fw);                                              // sharded solve: the peers' costs have arrived
  cvar_body<PER>(costs_mn, costs, n_cnt, ld, M, numel);
}

// M > 1024 (the reference switches to rollout_oversized_numba, mppi.py:199-203, 760-913, whose "sort" swaps
// unconditionally, so only its alpha = 1 mean is meaningful; this kernel computes the INTENDED statistic, the
// mean of the ceil(M*alpha) largest costs, for any M that fits shared memory).  One CTA per control
// sequence, the M keys in shared memory, the same bitwise radix select with a CTA-wide count per bit.
constexpr int CVAR_LARGE_THREADS = 256;

// control sequence n (blockIdx.x) by thread tid (threadIdx.x); M * 4 bytes of dynamic shared memory.  The kernels read
// n and tid themselves: read here, the thread index of cvar_large_kernel would be hoisted above its flag_wait, and that
// kernel's code would change with the split.
__device__ __forceinline__ void cvar_large_body(const float* __restrict__ costs_mn, float* __restrict__ costs, int n_cnt,
                                                int ld, int M, int numel, int n, int tid) {
  extern __shared__ uint32_t s_keys[];
  __shared__ int s_cnt[2][CVAR_LARGE_THREADS / 32];
  __shared__ float s_sum[CVAR_LARGE_THREADS / 32];
  const int lane = tid & 31, warp = tid >> 5;
  for (int j = tid; j < M; j += CVAR_LARGE_THREADS) s_keys[j] = float_key(__ldcg(costs_mn + (size_t)j * ld + n));
  __syncthreads();
  uint32_t prefix = 0;
  int greater_total = 0;
  if (numel < M) {
    for (int bit = 31; bit >= 0; --bit) {
      const uint32_t cand = prefix | (1u << bit);
      int cnt = 0;
      for (int j = tid; j < M; j += CVAR_LARGE_THREADS) cnt += (s_keys[j] >= cand) ? 1 : 0;
      cnt = __reduce_add_sync(0xffffffffu, cnt);
      if (lane == 0) s_cnt[bit & 1][warp] = cnt;
      __syncthreads();
      int total = 0;
#pragma unroll
      for (int w = 0; w < CVAR_LARGE_THREADS / 32; ++w) total += s_cnt[bit & 1][w];
      if (total >= numel) prefix = cand;
    }
  }
  float sum = 0.0f;
  int greater = 0;
  for (int j = tid; j < M; j += CVAR_LARGE_THREADS) {
    const uint32_t k = s_keys[j];
    if (numel >= M || k > prefix) { sum += key_float(k); ++greater; }
  }
  sum = warp_sum(sum);
  greater = __reduce_add_sync(0xffffffffu, greater);
  __syncthreads();                           // the last select round has finished reading s_cnt
  if (lane == 0) { s_sum[warp] = sum; s_cnt[0][warp] = greater; }
  __syncthreads();
  if (tid == 0) {
    float tot = 0.0f;
    for (int w = 0; w < CVAR_LARGE_THREADS / 32; ++w) { tot += s_sum[w]; greater_total += s_cnt[0][w]; }
    if (numel < M) tot += (float)(numel - greater_total) * key_float(prefix);
    costs[n] = (float)((double)tot / (double)numel);
  }
}

__global__ void __launch_bounds__(CVAR_LARGE_THREADS) cvar_large_kernel(const float* __restrict__ costs_mn,
                                                                        float* __restrict__ costs, int n_cnt, int ld,
                                                                        int M, int numel, const FlagWait fw) {
  flag_wait(fw);
  cvar_large_body(costs_mn, costs, n_cnt, ld, M, numel, blockIdx.x, threadIdx.x);
}

// [emu:end cvar]
// batched stochastic solves: planner blockIdx.y; every planner has the batch's n_cnt and M (hence PER and the grid)
// [emu:begin cvar_batch]
template <int PER>
__global__ void __launch_bounds__(CVAR_THREADS) cvar_batch_kernel(const CvarDesc* __restrict__ descs) {
  const CvarDesc& d = descs[blockIdx.y];
  if (d.active && !*d.active) return;
  cvar_body<PER>(d.costs_mn, d.costs, d.n_cnt, d.ld, d.M, d.numel);
}
// [emu:end cvar_batch]
// M > 1024: the CTA kernel, grid (n_cnt, count), control sequence blockIdx.x of planner blockIdx.y
// [emu:begin cvar_large_batch]
__global__ void __launch_bounds__(CVAR_LARGE_THREADS) cvar_large_batch_kernel(const CvarDesc* __restrict__ descs) {
  const CvarDesc& d = descs[blockIdx.y];
  if (d.active && !*d.active) return;
  cvar_large_body(d.costs_mn, d.costs, d.n_cnt, d.ld, d.M, d.numel, blockIdx.x, threadIdx.x);
}
// [emu:end cvar_large_batch]
int cvar_max_maps() { return CVAR_LARGE_MAX_MAPS; }
int cvar_warp_max_maps() { return 32 * CVAR_MAX_PER_LANE; }

int cvar_numel(int M, float cvar_alpha) {
  int numel = (int)ceil((double)M * (double)cvar_alpha);    // mppi.py:744 (float32 alpha, f64 product)
  if (numel < 1) numel = 1;
  if (numel > M) numel = M;
  return numel;
}

void launch_cvar_batch(const CvarDesc* descs, int count, int n_cnt, int M, cudaStream_t st) {
  if (M > 32 * CVAR_MAX_PER_LANE) {
    cudaFuncSetAttribute(cvar_large_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,   // per device
                         CVAR_LARGE_MAX_MAPS * (int)sizeof(uint32_t));
    const dim3 grid((unsigned)n_cnt, (unsigned)count);
    cvar_large_batch_kernel<<<grid, CVAR_LARGE_THREADS, (size_t)M * sizeof(uint32_t), st>>>(descs);
    return;
  }
  const int nb = cvar_block_n(M);
  const dim3 grid((unsigned)((n_cnt + nb - 1) / nb), (unsigned)count);
  const int per = (M + 31) / 32;
  if (per <= 1) cvar_batch_kernel<1><<<grid, CVAR_THREADS, 0, st>>>(descs);
  else if (per <= 2) cvar_batch_kernel<2><<<grid, CVAR_THREADS, 0, st>>>(descs);
  else if (per <= 4) cvar_batch_kernel<4><<<grid, CVAR_THREADS, 0, st>>>(descs);
  else if (per <= 8) cvar_batch_kernel<8><<<grid, CVAR_THREADS, 0, st>>>(descs);
  else if (per <= 16) cvar_batch_kernel<16><<<grid, CVAR_THREADS, 0, st>>>(descs);
  else cvar_batch_kernel<32><<<grid, CVAR_THREADS, 0, st>>>(descs);
}

void launch_cvar(const float* costs_mn, float* costs, int n_cnt, int ld, int M, float cvar_alpha, const FlagWait& fw,
                 cudaStream_t st) {
  const int numel = cvar_numel(M, cvar_alpha);
  if (M > 32 * CVAR_MAX_PER_LANE) {
    const size_t smem = (size_t)M * sizeof(uint32_t);
    cudaFuncSetAttribute(cvar_large_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,   // per device
                         CVAR_LARGE_MAX_MAPS * (int)sizeof(uint32_t));
    cvar_large_kernel<<<(unsigned)n_cnt, CVAR_LARGE_THREADS, smem, st>>>(costs_mn, costs, n_cnt, ld, M, numel, fw);
    return;
  }
  const int nb = cvar_block_n(M);
  const unsigned blocks = (unsigned)((n_cnt + nb - 1) / nb);
  const int per = (M + 31) / 32;
  if (per <= 1) cvar_kernel<1><<<blocks, CVAR_THREADS, 0, st>>>(costs_mn, costs, n_cnt, ld, M, numel, fw);
  else if (per <= 2) cvar_kernel<2><<<blocks, CVAR_THREADS, 0, st>>>(costs_mn, costs, n_cnt, ld, M, numel, fw);
  else if (per <= 4) cvar_kernel<4><<<blocks, CVAR_THREADS, 0, st>>>(costs_mn, costs, n_cnt, ld, M, numel, fw);
  else if (per <= 8) cvar_kernel<8><<<blocks, CVAR_THREADS, 0, st>>>(costs_mn, costs, n_cnt, ld, M, numel, fw);
  else if (per <= 16) cvar_kernel<16><<<blocks, CVAR_THREADS, 0, st>>>(costs_mn, costs, n_cnt, ld, M, numel, fw);
  else cvar_kernel<32><<<blocks, CVAR_THREADS, 0, st>>>(costs_mn, costs, n_cnt, ld, M, numel, fw);
}

// ---------------------------------------------------------------------------------------------
// Visualisation rollouts (mppi.py:1194-1351).  mode != 0: block 0 rolls out u_cur without noise,
// block b > 0 rolls out clip(u_prev + eps[b]) ; mode 0: u_cur over the first V sampled maps.
// [emu:begin vis]
__device__ __forceinline__ void state_rollout_body(const VisArgs& a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.V) return;
  const RolloutParams& p = a.p;
  const StepConst c = make_step_const(p);
  const int m = (a.mode == 0) ? b : 0;
  const int8_t* lin = a.lin_grid + (size_t)m * p.g.grid_rows * p.g.grid_pitch;
  const int8_t* ang = a.ang_grid + (size_t)m * p.g.grid_rows * p.g.grid_pitch;
  float* out = a.out + (size_t)b * (p.T + 1) * 3;
  float x = p.x0[0], y = p.x0[1], th = p.x0[2];
  out[0] = x; out[1] = y; out[2] = th;
  const bool noisy = (a.mode != 0) && (b != 0);
  if (a.mode == 3) {                      // map-free variant (notebook cell 3, get_state_rollout_across_control_noise)
    for (int t = 0; t < p.T; ++t) {
      float v, w;
      if (noisy) {
        const float* e = a.noise + ((size_t)b * p.T + t) * 2;
        v = fmaxf(c.v_lo, fminf(c.v_hi, fadd(a.u_prev[2 * t], e[0])));
        w = fmaxf(c.w_lo, fminf(c.w_hi, fadd(a.u_prev[2 * t + 1], e[1])));
      } else {
        v = a.u_cur[2 * t];
        w = a.u_cur[2 * t + 1];
      }
      const float dv = fmul(v, p.dt);
      const float cs = cos_approx(th), sn = sin_approx(th);
      x = ffma(dv, cs, x); y = ffma(dv, sn, y); th = ffma(w, p.dt, th);
      out[(t + 1) * 3 + 0] = x; out[(t + 1) * 3 + 1] = y; out[(t + 1) * 3 + 2] = th;
    }
    return;
  }
  for (int t = 0; t < p.T; ++t) {
    const int xi = cell_index(fsub(x, c.xlo), c.res, c.inv_res);
    const int yi = cell_index(fsub(y, c.ylo), c.res, c.inv_res);
    const int gy = wrap_clamp(yi, p.g.grid_rows), gx = wrap_clamp(xi, p.g.grid_cols);
    const int ql = lin[(size_t)gy * p.g.grid_pitch + gx];
    const int qa = ang[(size_t)gy * p.g.grid_pitch + gx];
    float v, w;
    if (noisy) {
      const float* e = a.noise + ((size_t)b * p.T + t) * 2;
      v = fmaxf(c.v_lo, fminf(c.v_hi, fadd(a.u_prev[2 * t], e[0])));
      w = fmaxf(c.w_lo, fminf(c.w_hi, fadd(a.u_prev[2 * t + 1], e[1])));
    } else {
      v = a.u_cur[2 * t];
      w = a.u_cur[2 * t + 1];
    }
    unicycle_step(c, ql, qa, v, w, x, y, th);
    out[(t + 1) * 3 + 0] = x; out[(t + 1) * 3 + 1] = y; out[(t + 1) * 3 + 2] = th;
  }
}

__global__ void state_rollout_kernel(const VisArgs a) {
  state_rollout_body(a);
}

// [emu:end vis]
// [emu:begin vis_batch]
// the visualisation rollouts of `count` planners of equal V and T, planner blockIdx.y: its VisArgs from the descriptor,
// the RolloutParams (x0 included) read where the batch's rollout descriptors hold them, the output at d.out + out_off
// (closed-loop trials: the record of this step).  A planner with active[y] == 0 is left untouched (active null: every
// planner runs).
__global__ void state_rollout_batch_kernel(const VisBatchDesc* __restrict__ descs, const int* __restrict__ active,
                                           size_t out_off) {
  if (active && !active[blockIdx.y]) return;
  const VisBatchDesc& d = descs[blockIdx.y];
  VisArgs a;
  a.p = *d.p;
  a.mode = d.mode; a.V = d.V;
  a.lin_grid = d.lin_grid; a.ang_grid = d.ang_grid;
  a.noise = d.noise; a.u_cur = d.u_cur; a.u_prev = d.u_prev;
  a.out = d.out + out_off;
  state_rollout_body(a);
}
// [emu:end vis_batch]
void launch_state_rollout(const VisArgs& a, cudaStream_t st) {
  state_rollout_kernel<<<(a.V + 31) / 32, 32, 0, st>>>(a);
}

void launch_state_rollout_batch(const VisBatchDesc* descs, int count, int V, const int* active, size_t out_off,
                                cudaStream_t st) {
  state_rollout_batch_kernel<<<dim3((unsigned)((V + 31) / 32), (unsigned)count), 32, 0, st>>>(descs, active, out_off);
}

}  // namespace b200
