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
// batched one-map solves: planner blockIdx.y, its generators / noise / u_std from the descriptor array
__global__ void __launch_bounds__(256) sample_noise_batch_kernel(const NoiseDesc* __restrict__ descs, int64_t count) {
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

void launch_sample_noise_batch(const NoiseDesc* descs, int count, int n_local, int T, cudaStream_t st) {
  const int64_t per = (int64_t)n_local * T;
  const int threads = 256;
  sample_noise_batch_kernel<<<dim3((unsigned)((per + threads - 1) / threads), (unsigned)count), threads, 0, st>>>(descs, per);
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
// `first` / `step`: the CTA's share of the weight slabs (the u update is done by the caller's CTA 0).
__device__ void apply_update(const UpdateArgs& a, const float* __restrict__ parts, int count, const float* s_scale,
                             float beta, float W, bool do_u, int first, int step) {
  const int stride = 2 * a.T + 2;
  if (do_u) {
    for (int j = threadIdx.x; j < 2 * a.T; j += blockDim.x) {
      float v = 0.0f;
      for (int i = 0; i < count; ++i) v = fmaf(__ldcg(parts + (size_t)i * stride + 2 + j), s_scale[i], v);
      float u = a.u_cur[j] + v / W;
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
      const float u = a.u_cur[j] + v / W;
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
    for (int r = tid; r < a.N; r += blockDim.x) a.weights[r] = __ldcg(a.w_raw + r) * (s_scale[r / a.rows_per_cta] / W);
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
// batched one-map solves: planner blockIdx.y, each with its own CTA partials, ticket counter, weights and u
__global__ void __launch_bounds__(UPD_THREADS) update_partial_batch_kernel(const UpdateBatchDesc* __restrict__ descs) {
  const UpdateBatchDesc& d = descs[blockIdx.y];
  update_partial_body(d.a, d.tl);
}
// [emu:end update_batch]

void launch_update_partial(const UpdateArgs& a, const UpdateTail& tl, cudaStream_t st) {
  update_partial_kernel<<<a.num_ctas, UPD_THREADS, 0, st>>>(a, tl);
}

void launch_update_partial_batch(const UpdateBatchDesc* descs, int count, int num_ctas, cudaStream_t st) {
  update_partial_batch_kernel<<<dim3((unsigned)num_ctas, (unsigned)count), UPD_THREADS, 0, st>>>(descs);
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

}  // namespace b200
