// reduce.cu -- control-noise sampling and the softmax-weighted control update.
// Reference: sample_noise_numba (mppi_numba/mppi.py:1354-1370), update_useq_numba (:1113-1191),
// shift_optimal_control_sequence (:539-542).
//
// The reference's update runs in ONE warp with 2*N*T global float atomics.  Here it is a two-level
// online-softmax reduction: every CTA owns a slab of rollouts, uses its local min as the softmax
// baseline, and streams its slab of the (N, 2T) noise matrix once with coalesced float2 loads;
// CTA partials (beta, S, V[2T]) are merged with the exp(-(beta_c-beta)/lambda) rescale -- the same
// merge that joins the ranks of a multi-GPU solve after the single all-gather.
#include "kernels.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// xoroshiro128p_normal_float32 (numba/cuda/random.py:176-197): Box-Muller in float32, two draws,
// sine branch discarded.  Compiled by Numba this uses libdevice's PRECISE logf/cosf (the helper is
// jitted without the kernel's fastmath flag) and sqrt.approx.ftz (module-wide NVVM option) --
// SURVEY.md 2.3; logf/cosf below are the same libdevice routines.
// [emu:begin noise]   (tests/emu_noise.py compiles the text between these markers for the host)
// xoro_normal: common.cuh (shared with the fused noise + controls kernel of rollout_win.cu)

// one thread per generator g = n*T + t (mppi.py:1367); generator and noise accesses are both
// contiguous in g, so loads/stores are fully coalesced 16 B / 8 B per lane.
__device__ __forceinline__ void sample_noise_body(uint64_t* __restrict__ states, float2* __restrict__ noise,
                                                  int64_t count, float std_v, float std_w, float* __restrict__ reach) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= count) return;
  if (g == 0 && reach) *reach = 0.0f;          // the prepare kernel that follows max-reduces into it
  ulonglong2* sp = reinterpret_cast<ulonglong2*>(states) + g;
  const ulonglong2 raw = *sp;
  Xoro s{raw.x, raw.y};
  float2 e;
  e.x = fmul(std_v, xoro_normal(s));
  e.y = fmul(std_w, xoro_normal(s));
  noise[g] = e;
  *sp = make_ulonglong2(s.s0, s.s1);
}

__global__ void __launch_bounds__(256) sample_noise_kernel(uint64_t* __restrict__ states,
                                                           float2* __restrict__ noise, int64_t count,
                                                           float std_v, float std_w, float* __restrict__ reach) {
  sample_noise_body(states, noise, count, std_v, std_w, reach);
}

// [emu:end noise]
// [emu:begin noise_batch]
// batched one-map solves: planner blockIdx.y, its generators / noise / u_std from the descriptor array; a planner with
// active[y] == 0 is left untouched (active null: every planner runs)
__global__ void __launch_bounds__(256) sample_noise_batch_kernel(const NoiseDesc* __restrict__ descs, int64_t count,
                                                                 const int* __restrict__ active = nullptr) {
  if (active && !active[blockIdx.y]) return;
  const NoiseDesc& d = descs[blockIdx.y];
  sample_noise_body(d.states, reinterpret_cast<float2*>(d.noise), count, d.std_v, d.std_w, nullptr);
}
// [emu:end noise_batch]

void launch_sample_noise(uint64_t* states, float* noise, int n_local, int T, float std_v, float std_w,
                         float* reach, cudaStream_t st) {
  const int64_t count = (int64_t)n_local * T;
  const int threads = 256;
  sample_noise_kernel<<<(unsigned)((count + threads - 1) / threads), threads, 0, st>>>(
      states, reinterpret_cast<float2*>(noise), count, std_v, std_w, reach);
}

void launch_sample_noise_batch(const NoiseDesc* descs, int count, int n_local, int T, const int* active,
                               cudaStream_t st) {
  const int64_t per = (int64_t)n_local * T;
  const int threads = 256;
  sample_noise_batch_kernel<<<dim3((unsigned)((per + threads - 1) / threads), (unsigned)count), threads, 0, st>>>(
      descs, per, active);
}

// ---------------------------------------------------------------------------------------------
// [emu:begin update]   (tests/emu_update.py compiles the text between these markers for the host)
// weight of one rollout, mppi.py:1154:  float32( exp( (-1.0/f64(lambda)) * f64(c - beta) ) )
__device__ __forceinline__ float softmax_weight(float c, float beta, float lambda) {
  return __double2float_rn(exp((-1.0 / (double)lambda) * (double)fsub(c, beta)));
}

constexpr int UPD_THREADS = 256;

int update_num_ctas(int N) {
  // slabs of >= 32 rollouts, at most 296 CTAs (~2 per SM of an H100).  A constant, not the device's SM count:
  // the CTA partition fixes the summation order of u, which must not depend on the GPU it runs on
  int ctas = (N + 31) / 32;
  if (ctas > 296) ctas = 296;
  if (ctas < 1) ctas = 1;
  return ctas;
}

// merge `count` partials (beta, S, V[2T]) -> out (same layout).  One CTA.
__device__ void merge_partials(const float* __restrict__ parts, int count, int T, float lambda,
                               float* out_beta, float* out_S, float* s_scale /* smem[count] */) {
  __shared__ float s_b;
  float mn = INFINITY;
  for (int i = threadIdx.x; i < count; i += blockDim.x) mn = fminf(mn, __ldcg(parts + (size_t)i * (2 * T + 2)));
  mn = warp_min(mn);
  __shared__ float s_red[UPD_THREADS / 32];
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = mn;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = s_red[0];
    for (int i = 1; i < UPD_THREADS / 32; ++i) v = fminf(v, s_red[i]);
    s_b = v;
  }
  __syncthreads();
  const float beta = s_b;
  for (int i = threadIdx.x; i < count; i += blockDim.x) {
    const float b = __ldcg(parts + (size_t)i * (2 * T + 2));
    s_scale[i] = (b == INFINITY) ? 0.0f : softmax_weight(b, beta, lambda);
  }
  __syncthreads();
  float S = 0.0f;                                   // block reduction in a fixed order (deterministic)
  for (int i = threadIdx.x; i < count; i += blockDim.x) S = fmaf(__ldcg(parts + (size_t)i * (2 * T + 2) + 1), s_scale[i], S);
  S = warp_sum(S);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = S;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.0f;
    for (int i = 0; i < UPD_THREADS / 32; ++i) t += s_red[i];
    *out_beta = beta;
    *out_S = t;
  }
  __syncthreads();
}

constexpr int MAX_PARTS = 512;

// u_cur (clipped) from merged partials: u[j] <- clip(u[j] + (sum_i V_i[j] * scale_i) / W), and the normalised
// weights of this rank's rollouts, weights[n] = w_raw[n] * exp(-(beta_cta - beta)/lambda) / W   (mppi.py:1173-1174).
// W == 0 (every cost +inf, so every partial has scale 0 and V = 0): a zero step, u[j] <- clip(u[j]), and weight 0 --
// 0 / 0 would make u NaN, which the clip turns into the upper bounds.
// `first` / `step`: the CTA's share of the weight slabs (the u update is done by the caller's CTA 0).
__device__ void apply_update(const UpdateArgs& a, const float* __restrict__ parts, int count, const float* s_scale,
                             float beta, float W, bool do_u, int first, int step) {
  const int stride = 2 * a.T + 2;
  if (do_u) {
    for (int j = threadIdx.x; j < 2 * a.T; j += blockDim.x) {
      float v = 0.0f;
      for (int i = 0; i < count; ++i) v = fmaf(__ldcg(parts + (size_t)i * stride + 2 + j), s_scale[i], v);
      const float u = (W == 0.0f) ? a.u_cur[j] : a.u_cur[j] + v / W;
      const float lo = (j & 1) ? a.wrange[0] : a.vrange[0];
      const float hi = (j & 1) ? a.wrange[1] : a.vrange[1];
      a.u_cur[j] = fmaxf(lo, fminf(hi, u));
    }
  }
  for (int c = first; c < a.num_ctas; c += step) {
    const float bc = __ldcg(a.cta_partials + (size_t)c * stride);
    const float sc = (bc == INFINITY) ? 0.0f : softmax_weight(bc, beta, a.lambda) / W;
    const int r0 = c * a.rows_per_cta, r1 = min(r0 + a.rows_per_cta, a.N);
    for (int r = r0 + threadIdx.x; r < r1; r += blockDim.x) a.weights[r] = __ldcg(a.w_raw + r) * sc;
  }
}

// grid = num_ctas; CTA c owns rows [c*rows_per_cta, ...).  Thread j owns float2 column j (one time
// step) for j < T, looping if T > blockDim.  The LAST CTA to finish (atomic ticket) merges the CTA partials into
// this rank's partial (beta, S, V[2T]) -- in CTA order, so the result does not depend on which CTA is last -- and,
// depending on `tail`:
//   UPD_TAIL_RANK   stops there (the staged exchange gathers rank_partial with a collective),
//   UPD_TAIL_APPLY  one rank: applies the update (u_cur, normalised weights) -- the whole update is ONE launch,
//   UPD_TAIL_BCAST  stores the partial into slot `rank` of every peer's gather buffer and raises its epoch flag
//                   (the all-gather of the peer-memory exchange, p2p.cu has the protocol).
// UPD_TAIL_APPLY also stores the new u into tl.u_prev / tl.u_out where those are set (batched solves).
__device__ __forceinline__ void update_partial_body(const UpdateArgs& a, const UpdateTail& tl) {
  __shared__ float s_red[UPD_THREADS / 32];
  __shared__ float s_w[64];
  __shared__ float s_beta;
  __shared__ bool s_last;
  const int r0 = blockIdx.x * a.rows_per_cta;
  const int r1 = min(r0 + a.rows_per_cta, a.N);
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float* part = a.cta_partials + (size_t)blockIdx.x * (2 * a.T + 2);

  // local baseline
  float mn = INFINITY;
  for (int r = r0 + tid; r < r1; r += blockDim.x) mn = fminf(mn, a.costs[r]);
  mn = warp_min(mn);
  if (lane == 0) s_red[wid] = mn;
  __syncthreads();
  if (tid == 0) {
    float v = s_red[0];
    for (int i = 1; i < UPD_THREADS / 32; ++i) v = fminf(v, s_red[i]);
    s_beta = v;
  }
  __syncthreads();
  const float beta = s_beta;

  const float2* __restrict__ eps = reinterpret_cast<const float2*>(a.noise);
  float S = 0.0f;
  // accumulators for up to 4 column-chunks (T <= 4*UPD_THREADS = 1024, the reference's own cap)
  float2 acc[4] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
  // a slab whose every cost is +inf: c - beta would be inf - inf = NaN.  Its rollouts get the reference's weight
  // exp(-inf) = 0 (its beta is the global minimum) and the slab's partial is S = 0, V = 0 with beta = +inf, which
  // merge_partials gives scale 0.  The branch is uniform over the CTA.
  if (beta == INFINITY) {
    for (int r = r0 + tid; r < r1; r += blockDim.x) a.w_raw[r] = 0.0f;
  } else {
    for (int rb = r0; rb < r1; rb += 64) {
      const int nr = min(64, r1 - rb);
      __syncthreads();
      if (tid < nr) {
        const float w = softmax_weight(a.costs[rb + tid], beta, a.lambda);
        s_w[tid] = w;
        a.w_raw[rb + tid] = w;
      }
      __syncthreads();
      // rows in batches of eight: the loads of a batch are issued before its FMAs (issue is in order -- an FMA waiting
      // for its row would hold back the next row's load); accumulation order is the row order, as before
      for (int i0 = 0; i0 < nr; i0 += 8) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int j = tid + k * UPD_THREADS;
          if (j < a.T) {
            float2 e[8];
#pragma unroll
            for (int q = 0; q < 8; ++q)
              e[q] = (i0 + q < nr) ? __ldg(eps + (size_t)(rb + i0 + q) * a.T + j) : make_float2(0.f, 0.f);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              if (i0 + q < nr) {
                const float w = s_w[i0 + q];
                acc[k].x = fmaf(w, e[q].x, acc[k].x);
                acc[k].y = fmaf(w, e[q].y, acc[k].y);
              }
            }
          }
        }
        if (tid == 0)
          for (int q = 0; q < 8 && i0 + q < nr; ++q) S += s_w[i0 + q];
      }
    }
  }
  if (tid == 0) { part[0] = (r1 > r0) ? beta : INFINITY; part[1] = S; }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int j = tid + k * UPD_THREADS;
    if (j < a.T) { part[2 + 2 * j] = acc[k].x; part[3 + 2 * j] = acc[k].y; }
  }

  // ---- ticket: the last CTA of the grid carries on, the others are done
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned prev = atomicAdd(tl.counter, 1u);
    s_last = (prev == gridDim.x - 1);
    if (s_last) *tl.counter = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();

  __shared__ float s_scale[MAX_PARTS];
  __shared__ float s_bS[2];
  merge_partials(a.cta_partials, a.num_ctas, a.T, a.lambda, &s_bS[0], &s_bS[1], s_scale);
  const int stride = 2 * a.T + 2;
  const float W = s_bS[1];
  // V[j] = sum_i V_i[j] * scale_i in CTA order (one column per thread, loads batched 32 at a time -- the chain of
  // FMAs is sequential, the L2 loads behind it must not be)
  for (int j = tid; j < 2 * a.T; j += blockDim.x) {
    float v = 0.0f;
    int i = 0;
    for (; i + 32 <= a.num_ctas; i += 32) {
      float x[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) x[k] = __ldcg(a.cta_partials + (size_t)(i + k) * stride + 2 + j);
#pragma unroll
      for (int k = 0; k < 32; ++k) v = fmaf(x[k], s_scale[i + k], v);
    }
    for (; i + 8 <= a.num_ctas; i += 8) {
      float x[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) x[k] = __ldcg(a.cta_partials + (size_t)(i + k) * stride + 2 + j);
#pragma unroll
      for (int k = 0; k < 8; ++k) v = fmaf(x[k], s_scale[i + k], v);
    }
    for (; i < a.num_ctas; ++i) v = fmaf(__ldcg(a.cta_partials + (size_t)i * stride + 2 + j), s_scale[i], v);
    a.rank_partial[2 + j] = v;
    if (tl.mode == UPD_TAIL_APPLY) {               // one rank: this partial is the only one -- apply straight away
      const float u = (W == 0.0f) ? a.u_cur[j] : a.u_cur[j] + v / W;      // W == 0: every cost +inf (apply_update)
      const float lo = (j & 1) ? a.wrange[0] : a.vrange[0];
      const float hi = (j & 1) ? a.wrange[1] : a.vrange[1];
      const float un = fmaxf(lo, fminf(hi, u));
      a.u_cur[j] = un;
      if (tl.u_prev) tl.u_prev[j] = un;
      if (tl.u_out) tl.u_out[j] = un;
    }
  }
  if (tid == 0) { a.rank_partial[0] = s_bS[0]; a.rank_partial[1] = W; }
  if (tl.mode == UPD_TAIL_APPLY) {
    // normalised weights (mppi.py:1173-1174): the merge scale of a rollout's CTA is exp(-(beta_cta - beta)/lambda)
    for (int r = tid; r < a.N; r += blockDim.x)
      a.weights[r] = (W == 0.0f) ? 0.0f : __ldcg(a.w_raw + r) * (s_scale[r / a.rows_per_cta] / W);
  }
  if (tl.mode == UPD_TAIL_BCAST) {
    __syncthreads();                                // rank_partial complete (this CTA wrote all of it)
    for (int q = 0; q < tl.ws; ++q) {
      float* dst = tl.peer_gather[q] + (size_t)tl.rank * stride;
      for (int j = tid; j < stride; j += blockDim.x) dst[j] = a.rank_partial[j];
    }
    __threadfence_system();
    __syncthreads();
    if (tid < tl.ws) {
      __threadfence_system();
      st_flag_sys(tl.peer_flags[tid] + tl.rank, tl.epoch);
    }
  }
}

__global__ void __launch_bounds__(UPD_THREADS) update_partial_kernel(const UpdateArgs a, const UpdateTail tl) {
  update_partial_body(a, tl);
}

// gathered rank partials -> u_cur (clipped), plus this rank's normalised weights.  wait_flags != null: the partials
// arrive through the peer-memory exchange -- every CTA first waits (bounded) until all ranks' epoch flags are up.
__global__ void __launch_bounds__(UPD_THREADS) update_apply_kernel(const UpdateArgs a,
                                                                   const float* __restrict__ gathered,
                                                                   int count, const FlagWait fw) {
  __shared__ float s_scale[MAX_PARTS];
  __shared__ float s_bS[2];
  flag_wait(fw);
  merge_partials(gathered, count, a.T, a.lambda, &s_bS[0], &s_bS[1], s_scale);
  apply_update(a, gathered, count, s_scale, s_bS[0], s_bS[1], blockIdx.x == 0, blockIdx.x, gridDim.x);
}

// [emu:end update]
// [emu:begin update_batch]
// batched one-map solves: planner blockIdx.y, each with its own CTA partials, ticket counter, weights and u; a planner
// with active[y] == 0 is left untouched, its ticket counter included (active null: every planner runs)
__global__ void __launch_bounds__(UPD_THREADS) update_partial_batch_kernel(const UpdateBatchDesc* __restrict__ descs,
                                                                           const int* __restrict__ active = nullptr) {
  if (active && !active[blockIdx.y]) return;
  const UpdateBatchDesc& d = descs[blockIdx.y];
  update_partial_body(d.a, d.tl);
}
// [emu:end update_batch]

void launch_update_partial(const UpdateArgs& a, const UpdateTail& tl, cudaStream_t st) {
  update_partial_kernel<<<a.num_ctas, UPD_THREADS, 0, st>>>(a, tl);
}

void launch_update_partial_batch(const UpdateBatchDesc* descs, int count, int num_ctas, const int* active,
                                 cudaStream_t st) {
  update_partial_batch_kernel<<<dim3((unsigned)num_ctas, (unsigned)count), UPD_THREADS, 0, st>>>(descs, active);
}

void launch_update_finish(const UpdateArgs& a, const float* gathered, int count, const FlagWait& fw, cudaStream_t st) {
  int ctas = a.num_ctas < 32 ? a.num_ctas : 32;
  if (ctas < 1) ctas = 1;
  update_apply_kernel<<<ctas, UPD_THREADS, 0, st>>>(a, gathered, count, fw);
}

__global__ void shift_u_kernel(float* u, int T, int shifts) {
  // u[:-s] = u[s:]  (tail keeps its values, mppi.py:540-541); single CTA, staged through smem
  extern __shared__ float s[];
  for (int i = threadIdx.x; i < 2 * T; i += blockDim.x) s[i] = u[i];
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * (T - shifts); i += blockDim.x) u[i] = s[i + 2 * shifts];
}

void launch_shift_u(float* u, int T, int shifts, cudaStream_t st) {
  if (shifts <= 0 || shifts >= T) return;
  shift_u_kernel<<<1, 256, (size_t)2 * T * sizeof(float), st>>>(u, T, shifts);
}

// ---------------------------------------------------------------------------------------------
// Plant step of a closed-loop trial, as the benchmark's trial() computes it in float64 (no contraction: every product
// and sum is rounded on its own, in the loop's order).
// [emu:begin trial]
// CPython's float `//` (float_floor_div): fmod, subtract, divide, floor, with its sign and snap-to-nearest corrections
__device__ __forceinline__ double py_floordiv(double vx, double wx) {
  double mod = fmod(vx, wx);
  double div = __ddiv_rn(__dsub_rn(vx, mod), wx);
  if (mod != 0.0) {
    if ((wx < 0.0) != (mod < 0.0)) div = __dsub_rn(div, 1.0);
  }
  if (div != 0.0) {
    double fl = floor(div);
    if (__dsub_rn(div, fl) > 0.5) fl = __dadd_rn(fl, 1.0);
    return fl;
  }
  return copysign(0.0, __ddiv_rn(vx, wx));
}

// u[:-1] = u[1:] in place by one warp, the last row kept (shift_and_update with num_shifts 1): chunk c reads floats
// [c+2, c+34) before any lane writes [c, c+32)
__device__ __forceinline__ void warp_shift_u(float* u, int T, int lane) {
  const int n = 2 * (T - 1);
  for (int c = 0; c < n; c += 32) {
    const int i = c + lane;
    const float x = i < n ? u[i + 2] : 0.0f;
    __syncwarp();
    if (i < n) u[i] = x;
  }
}

// The x0 the planner's next rollout starts from, as set_params passes it (float32), and for a windowed (stochastic)
// rollout the window around it
__device__ __forceinline__ void set_next_x0(const TrialDev& d, float x, float y, float th) {
  d.x0_out[0] = x; d.x0_out[1] = y; d.x0_out[2] = th;
  if (d.win) win_origin(x, y, d.win_pxl, d.win_pyl, d.win_res, d.win_cols, d.win_rows, d.win);
}

// Recording sequences: whether planner k records at its next step, step `step` of the episode of slot `slot`, and
// where that record goes (SeqArgs).
__device__ __forceinline__ void seq_record_next(const SeqArgs& q, int k, int slot, int step) {
  if (!q.rec_flag) return;
  const int on = step % q.rec_every == 0;
  q.rec_flag[k] = on;
  if (on) q.rec_out[(size_t)k * q.rec_stride] = q.rec + ((size_t)slot * q.rec_R + step / q.rec_every) * q.rec_per;
}

// One warp per planner (warp k of the grid = planner k): apply u_cur[0], shift u_cur by one row (the last row kept),
// record the step, and stop the planner on the goal, on leaving the padded map or after max_steps steps.
// Barebone trials (TrialDev::lin null) step the notebook's nominal unicycle (traction 1: dt * 1.0 == dt), have no map
// to leave, and count in contacts[slot] the steps whose new pose lies in one of the planner's obstacles.
// SEQ (trial sequences, SeqArgs): the planner steps its running episode e, slot first[k] + e of the descriptors and
// histories.  When that episode stops and another follows (reset_x0, or a stop other than LEFT_MAP), its result is
// written, the plant restarts from the next start pose with zero metrics, and the planner stays active; with reset_x0
// the next solve also plans from that pose (x0_out and the window).  Without it x0_out keeps the final pose, as the
// benchmark's planner keeps its params['x0'] across episodes.  active_count falls when the sequence ends.  A recording
// sequence also marks whether the planner records at its next step (seq_record_next; 0 once its sequence ends).
template <bool SEQ = false>
__device__ __forceinline__ void plant_step_body(const PlantArgs& a, int k, int lane, const SeqArgs& q = SeqArgs{}) {
  if (k >= a.K || !a.active[k]) return;
  const int slot = SEQ ? q.first[k] + q.episode[k] : k;
  const TrialDev& d = a.trials[slot];
  float* u = d.u_cur;
  float v = 0.0f, w = 0.0f;
  if (lane == 0) { v = u[0]; w = u[1]; }
  __syncwarp();
  warp_shift_u(u, a.T, lane);
  if (lane != 0) return;
  TrialState& s = a.state[k];
  const int t = SEQ ? s.steps : a.step;
  float* uh = a.uhist + ((size_t)slot * a.max_steps + t) * 2;
  uh[0] = v; uh[1] = w;
  const double x = s.x[0], y = s.x[1], th = s.x[2];
  double lt = 1.0, at = 1.0;
  if (d.lin) {
    // TractionGrid.get: int((x - xlo) // res), (0, 0) outside [0, W) x [0, H)
    const double fx = py_floordiv(__dsub_rn(x, d.xlo), d.res), fy = py_floordiv(__dsub_rn(y, d.ylo), d.res);
    lt = 0.0; at = 0.0;
    if (fx >= 0.0 && fx < (double)d.W && fy >= 0.0 && fy < (double)d.H) {
      const size_t cell = (size_t)fy * (size_t)d.W + (size_t)fx;
      lt = d.lin[cell]; at = d.ang[cell];
    }
  }
  const double dtl = __dmul_rn(d.dt, lt);
  const double xn = __dadd_rn(x, __dmul_rn(__dmul_rn(dtl, cos(th)), (double)v));
  const double yn = __dadd_rn(y, __dmul_rn(__dmul_rn(dtl, sin(th)), (double)v));
  const double thn = __dadd_rn(th, __dmul_rn(__dmul_rn(d.dt, at), (double)w));
  s.x[0] = xn; s.x[1] = yn; s.x[2] = thn;
  double* xh = a.xhist + ((size_t)slot * (a.max_steps + 1) + t + 1) * 3;
  xh[0] = xn; xh[1] = yn; xh[2] = thn;
  // the next rollout starts from float32(x_next), as set_params would pass it
  set_next_x0(d, __double2float_rn(xn), __double2float_rn(yn), __double2float_rn(thn));
  const double dx = __dsub_rn(xn, d.xgoal[0]), dy = __dsub_rn(yn, d.xgoal[1]);
  const double dist = __dsub_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy))), d.tol);
  s.cum_obj = __dadd_rn(s.cum_obj, __dadd_rn(d.dt, dist));
  s.cum_dist = __dadd_rn(s.cum_dist, dist);
  s.dist = dist;
  s.steps = t + 1;
  if (a.contacts) {
    // (x - ox)^2 + (y - oy)^2 <= r^2 in float64 from the float32 obstacle: the rollout's rule (only diff > 0 is outside);
    // one contact per step however many obstacles overlap there
    bool hit = false;
    for (int j = 0; j < d.num_obstacles && !hit; ++j) {
      const double ex = __dsub_rn(xn, (double)d.obstacles[3 * j]), ey = __dsub_rn(yn, (double)d.obstacles[3 * j + 1]);
      const double r = (double)d.obstacles[3 * j + 2];
      hit = __dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)) <= __dmul_rn(r, r);
    }
    if (hit) a.contacts[slot] += 1;
  }
  int status = TRIAL_RUNNING;
  if (dist <= 0.0) status = TRIAL_GOAL;
  else if (d.lin && !(xn >= d.pxlim[0] && xn <= d.pxlim[1] && yn >= d.pylim[0] && yn <= d.pylim[1]))
    status = TRIAL_LEFT_MAP;
  else if (t + 1 >= a.max_steps) status = TRIAL_MAX_STEPS;
  if (status != TRIAL_RUNNING) {
    if constexpr (SEQ) {
      TrialState& r = q.results[slot];
      r = s;
      r.status = status;
      if (slot + 1 < q.first[k + 1] && (q.reset_x0 || status != TRIAL_LEFT_MAP)) {
        const double* x0 = q.start + (size_t)(slot + 1) * 3;
        s.x[0] = x0[0]; s.x[1] = x0[1]; s.x[2] = x0[2];
        s.cum_obj = 0.0; s.cum_dist = 0.0; s.dist = 0.0;
        s.steps = 0;
        q.episode[k] += 1;
        if (q.reset_x0) {
          set_next_x0(d, __double2float_rn(x0[0]), __double2float_rn(x0[1]), __double2float_rn(x0[2]));
        }
        seq_record_next(q, k, slot + 1, 0);
        return;
      }
      if (q.rec_flag) q.rec_flag[k] = 0;
    }
    s.status = status;
    a.active[k] = 0;
    atomicSub(a.active_count, 1);
  } else if constexpr (SEQ) {
    seq_record_next(q, k, slot, t + 1);
  }
}

__global__ void __launch_bounds__(128) plant_step_kernel(const PlantArgs a) {
  plant_step_body(a, (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), (int)(threadIdx.x & 31));
}

__global__ void __launch_bounds__(128) plant_step_seq_kernel(const PlantArgs a, const SeqArgs q) {
  plant_step_body<true>(a, (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), (int)(threadIdx.x & 31), q);
}
// [emu:end trial]

// ---------------------------------------------------------------------------------------------
// Device loops (b200mppi_batch_loop_open): the solve's controls out, the caller's pose in, and stops.  A planner whose
// active flag is 0 is left untouched by all three.
// [emu:begin loop]
// One CTA per planner: its u_cur into row `row` of the caller's (K, T, 2) controls, NaN for a planner that no longer
// runs.  A running planner counts the solve and keeps the x0 it planned from.
__device__ __forceinline__ void loop_export_body(const LoopArgs& a, float* __restrict__ out, int k) {
  LoopState& s = a.state[k];
  const TrialDev& d = a.dev[k];
  const bool on = a.active[k] != 0;
  float* o = out + (size_t)s.row * 2 * a.T;
  for (int j = threadIdx.x; j < 2 * a.T; j += blockDim.x) o[j] = on ? d.u_cur[j] : __int_as_float(0x7fc00000);
  if (on && threadIdx.x == 0) {
    s.solves += 1;
    for (int c = 0; c < 3; ++c) s.x0[c] = d.x0_out[c];
  }
}

// One warp per planner (warp k of the grid = planner k), as the plant step: shift u_cur by one row, take the pose of row
// `row` of x (float64, or float32 widened; row_stride bytes apart) and count the shift.  A pose outside the padded map
// limits (float64 lo <= v <= hi; NaN fails), where the planner's next solve would be refused, stops the planner
// (TRIAL_LEFT_MAP); otherwise its next rollout plans from float32 of the pose (set_next_x0).
__device__ __forceinline__ void loop_ingest_body(const LoopArgs& a, const unsigned char* __restrict__ x, int dtype,
                                                 long long row_stride, int k, int lane) {
  if (k >= a.K || !a.active[k]) return;
  const TrialDev& d = a.dev[k];
  warp_shift_u(d.u_cur, a.T, lane);
  if (lane != 0) return;
  LoopState& s = a.state[k];
  const unsigned char* r = x + (long long)s.row * row_stride;
  double p[3];
  float f[3];
  for (int c = 0; c < 3; ++c) {
    if (dtype == LOOP_POSE_F32) {
      f[c] = reinterpret_cast<const float*>(r)[c];
      p[c] = (double)f[c];
    } else {
      p[c] = reinterpret_cast<const double*>(r)[c];
      f[c] = __double2float_rn(p[c]);
    }
    s.x[c] = p[c];
  }
  s.shifts += 1;
  if (s.bounded && !(p[0] >= s.pxlim[0] && p[0] <= s.pxlim[1] && p[1] >= s.pylim[0] && p[1] <= s.pylim[1])) {
    s.status = TRIAL_LEFT_MAP;
    a.active[k] = 0;
    atomicSub(a.active_count, 1);
    return;
  }
  set_next_x0(d, f[0], f[1], f[2]);
}

__global__ void __launch_bounds__(128) loop_ingest_kernel(const LoopArgs a, const unsigned char* __restrict__ x, int dtype,
                                                          long long row_stride) {
  loop_ingest_body(a, x, dtype, row_stride, (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5),
                   (int)(threadIdx.x & 31));
}

// One thread per planner: a running planner whose entry of the caller's mask (int32, or one byte: bool / uint8) is
// nonzero stops for good (LOOP_STOPPED)
__device__ __forceinline__ void loop_stop_body(const LoopArgs& a, const void* __restrict__ mask, int elem_bytes, int k) {
  if (k >= a.K || !a.active[k]) return;
  LoopState& s = a.state[k];
  const bool stop = elem_bytes == 1 ? reinterpret_cast<const unsigned char*>(mask)[s.row] != 0
                                    : reinterpret_cast<const int*>(mask)[s.row] != 0;
  if (!stop) return;
  s.status = LOOP_STOPPED;
  a.active[k] = 0;
  atomicSub(a.active_count, 1);
}

__global__ void __launch_bounds__(128) loop_stop_kernel(const LoopArgs a, const void* __restrict__ mask, int elem_bytes) {
  loop_stop_body(a, mask, elem_bytes, (int)(blockIdx.x * blockDim.x + threadIdx.x));
}
// [emu:end loop]

// [emu:begin loop_clock]
// The solve clock (LoopClock), run by one CTA of the export launch that ends solve s = clock[0]: it prepares
// solve s + 1.  Only two inputs of a loop solve change from one solve to the next, and both move here:
//   - each kind's sampler set: the staged set of parity (s + 1) & 1 is copied into the current set, which the solve's
//     sampler launches read (every running planner has sampled its pair exactly s + 1 times before that solve);
//   - the reach slot of every stochastic planner's noise and box descriptor becomes the slot of the solve's first
//     iteration, staged slot ^ (((s + 1) * num_opt) & 1): iteration k then reads slot ^ (k & 1), the slot the by-value
//     iteration index (s + 1) * num_opt + k selects.
// The clock advances last, after the CTA's barrier.  At 2^31 - 1 solves it stops and sets clock[1] instead of wrapping.
__device__ __forceinline__ void loop_clock_body(const LoopClock& a) {
  if (!a.clock) return;
  const int s = a.clock[0];
  const unsigned next = (unsigned)s + 1u;
  static_assert(sizeof(SampleGridsV2Args) % sizeof(unsigned long long) == 0, "sampler sets copied in 8-byte words");
  constexpr int words = (int)(sizeof(SampleGridsV2Args) / sizeof(unsigned long long));
  for (int k = 0; k < 2; ++k) {
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(a.set_par[k][next & 1u]);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(a.set_cur[k]);
    for (int j = threadIdx.x; j < a.G[k] * words; j += blockDim.x) dst[j] = src[j];
  }
  const int flip = (int)((next * (unsigned)a.num_opt) & 1u);
  for (int r = threadIdx.x; r < a.K2; r += blockDim.x) {
    a.nprep[r].slot = a.slot0[r] ^ flip;
    a.box[r].slot = a.slot0[a.K2 + r] ^ flip;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s == 0x7fffffff) a.clock[1] = 1;
    else a.clock[0] = s + 1;
  }
}
// [emu:end loop_clock]

// [emu:begin loop_task]
// Element c of a caller's row r: float64, or float32 widened exactly; *f is what set_params would pass (float32)
__device__ __forceinline__ double loop_elem(const unsigned char* r, int dtype, int c, float* f) {
  if (dtype == LOOP_POSE_F32) {
    *f = reinterpret_cast<const float*>(r)[c];
    return (double)*f;
  }
  const double v = reinterpret_cast<const double*>(r)[c];
  *f = __double2float_rn(v);
  return v;
}

// One thread per planner: a running planner takes the goal of row `row` of g (2 elements, float64 or float32; rows
// row_stride bytes apart).  Its rollout descriptor's goal becomes float32 of it, as set_params passes it, and the
// float64 value is kept for the commit.  Nothing is checked: set_params takes any goal.
__device__ __forceinline__ void loop_goal_body(const LoopArgs& a, const LoopTaskArgs& ta,
                                               const unsigned char* __restrict__ g, int dtype, long long row_stride,
                                               int k) {
  if (k >= a.K || !a.active[k]) return;
  LoopTask& q = ta.task[k];
  const unsigned char* r = g + (long long)a.state[k].row * row_stride;
  for (int c = 0; c < 2; ++c) {
    float f;
    q.goal[c] = loop_elem(r, dtype, c, &f);
    q.xgoal_out[c] = f;
  }
  q.took_goal = 1;
}

__global__ void __launch_bounds__(128) loop_goal_kernel(const LoopArgs a, const LoopTaskArgs ta,
                                                        const unsigned char* __restrict__ g, int dtype,
                                                        long long row_stride) {
  loop_goal_body(a, ta, g, dtype, row_stride, (int)(blockIdx.x * blockDim.x + threadIdx.x));
}

// One warp per planner (warp k of the grid = planner k): a running planner takes the first n triples [x, y, r] of row
// `row` of obs (count = O' triples per row, contiguous, float64 or float32; rows row_stride bytes apart), n =
// counts[row] (counts null: O').  Float32 of each element goes into the planner's slice of the loop's buffer, which
// its rollout descriptor reads, the float64 values into the shadow for the commit, and the descriptor's obstacle count
// becomes n.  A count outside [0, O'], which the host's set_obstacles refuses, stops the planner for good
// (LOOP_BAD_OBSTACLES); its rollouts keep the last set it took.
__device__ __forceinline__ void loop_obstacles_body(const LoopArgs& a, const LoopTaskArgs& ta,
                                                    const unsigned char* __restrict__ obs, int dtype, int count,
                                                    long long row_stride, const int* __restrict__ counts, int k,
                                                    int lane) {
  if (k >= a.K || !a.active[k]) return;
  LoopState& s = a.state[k];
  const int n = counts ? counts[s.row] : count;
  if (n < 0 || n > count) {
    if (lane == 0) {
      s.status = LOOP_BAD_OBSTACLES;
      a.active[k] = 0;
      atomicSub(a.active_count, 1);
    }
    return;
  }
  const unsigned char* r = obs + (long long)s.row * row_stride;
  float* o = ta.obs + (size_t)k * ta.O * 3;
  double* o64 = ta.obs64 + (size_t)k * ta.O * 3;
  for (int j = lane; j < 3 * n; j += 32) {
    float f;
    o64[j] = loop_elem(r, dtype, j, &f);
    o[j] = f;
  }
  if (lane != 0) return;
  LoopTask& q = ta.task[k];
  *q.num_obstacles_out = n;
  q.num_obstacles = n;
  q.took_obstacles = 1;
}

__global__ void __launch_bounds__(128) loop_obstacles_kernel(const LoopArgs a, const LoopTaskArgs ta,
                                                             const unsigned char* __restrict__ obs, int dtype,
                                                             int count, long long row_stride,
                                                             const int* __restrict__ counts) {
  loop_obstacles_body(a, ta, obs, dtype, count, row_stride, counts,
                      (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), (int)(threadIdx.x & 31));
}
// [emu:end loop_task]

// the export of a loop solve, and (CTA 0) the preparation of the next
__global__ void __launch_bounds__(128) loop_export_kernel(const LoopArgs a, float* __restrict__ out, const LoopClock c) {
  loop_export_body(a, out, (int)blockIdx.x);
  if (blockIdx.x == 0) loop_clock_body(c);
}

void launch_loop_export(const LoopArgs& a, const LoopClock& c, float* u_out, cudaStream_t st) {
  loop_export_kernel<<<(unsigned)a.K, 128, 0, st>>>(a, u_out, c);
}

void launch_loop_ingest(const LoopArgs& a, const void* x, int dtype, long long row_stride, cudaStream_t st) {
  loop_ingest_kernel<<<(unsigned)((a.K + 3) / 4), 128, 0, st>>>(a, reinterpret_cast<const unsigned char*>(x), dtype,
                                                                 row_stride);
}

void launch_loop_stop(const LoopArgs& a, const void* mask, int elem_bytes, cudaStream_t st) {
  loop_stop_kernel<<<(unsigned)((a.K + 127) / 128), 128, 0, st>>>(a, mask, elem_bytes);
}

void launch_loop_goal(const LoopArgs& a, const LoopTaskArgs& ta, const void* g, int dtype, long long row_stride,
                      cudaStream_t st) {
  loop_goal_kernel<<<(unsigned)((a.K + 127) / 128), 128, 0, st>>>(a, ta, reinterpret_cast<const unsigned char*>(g),
                                                                  dtype, row_stride);
}

void launch_loop_obstacles(const LoopArgs& a, const LoopTaskArgs& ta, const void* obs, int dtype, int count,
                           long long row_stride, const int* counts, cudaStream_t st) {
  loop_obstacles_kernel<<<(unsigned)((a.K + 3) / 4), 128, 0, st>>>(a, ta, reinterpret_cast<const unsigned char*>(obs),
                                                                    dtype, count, row_stride, counts);
}

void launch_plant_step(const PlantArgs& a, cudaStream_t st) {
  plant_step_kernel<<<(unsigned)((a.K + 3) / 4), 128, 0, st>>>(a);
}

void launch_plant_step_seq(const PlantArgs& a, const SeqArgs& q, cudaStream_t st) {
  plant_step_seq_kernel<<<(unsigned)((a.K + 3) / 4), 128, 0, st>>>(a, q);
}

}  // namespace b200
