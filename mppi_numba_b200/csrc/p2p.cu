// Peer-memory (NVLink / NVSwitch) exchange for the sharded solve: the two collectives of a multi-rank
// solve() -- the all-to-all of per-(n,m) rollout costs and the all-gather of the (2T+2)-float softmax
// partials -- done by this library's own kernels with plain stores into the peers' memory plus epoch flags,
// instead of two NCCL calls, whose fixed latency is a large part of a sharded solve (tools/nccl_latency.py).
//
// Protocol (one "exchange" = one epoch e, a counter that only grows):
//   producer rank r:  data stores into peer d's buffer -> __threadfence_system() -> flags_d[r] = e (st.release.sys)
//                     -- the stores and the flag come from the kernel that PRODUCES the data: the windowed rollout
//                     kernel's epilogue (costs, rollout_win.cu), the last CTA of update_partial_kernel (softmax
//                     partial, reduce.cu); only the generic rollout kernel needs the separate push kernel below
//   consumer rank d:  the kernel that CONSUMES the data (CVaR, update_apply) starts with flag_wait (common.cuh): every
//                     CTA spins with ld.acquire.sys until flags_d[s] >= e for every s (bounded by a timeout), then
//                     reads the data with L2 (.cg) loads
// Buffers are written by exactly one producer per slot, flags only grow, the gather buffer is double
// buffered by epoch parity (a fast rank may start exchange e+1 before a slow one has consumed e).
#include "common.cuh"
#include "kernels.h"

namespace b200 {

// ---- all-to-all of cost blocks (only for rollouts that did not store straight into the peers -- the generic
// rollout kernel): block d of the local staged array (ws, Mc, n_red), contiguous n_red*Mc floats, goes to block
// `rank` of peer d's receive buffer (ws, Mc, n_red).  grid = (ctas_per_peer, ws).
__global__ void __launch_bounds__(256) p2p_push_kernel(const P2PPushArgs a) {
  const int d = blockIdx.y;
  const size_t block_elems = (size_t)a.n_red * a.Mc;
  const float* src = a.costs_nm + (size_t)d * block_elems;
  float* dst = a.peer_recv[d] + (size_t)a.rank * block_elems;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t gtid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if ((block_elems & 3) == 0) {                 // 16-byte stores: both bases are 256-byte aligned
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (size_t i = gtid; i < block_elems / 4; i += stride) d4[i] = s4[i];
  } else {
    for (size_t i = gtid; i < block_elems; i += stride) dst[i] = src[i];
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned total = gridDim.x * gridDim.y;
    const unsigned prev = atomicAdd(a.counter, 1u);
    if (prev == total - 1) {                     // last CTA of the grid: everything of this rank is out
      *a.counter = 0;
      __threadfence_system();
      for (int p = 0; p < a.ws; ++p) st_flag_sys(a.peer_flags[p] + a.rank, a.epoch);
    }
  }
}

void launch_p2p_push(const P2PPushArgs& a, cudaStream_t st) {
  const size_t block_elems = (size_t)a.n_red * a.Mc;
  size_t per_thread = (block_elems & 3) == 0 ? 4 : 1;
  size_t ctas = (block_elems / per_thread + 256 * 4 - 1) / (256 * 4);      // ~4 stores per thread
  if (ctas < 1) ctas = 1;
  if (ctas > 64) ctas = 64;
  p2p_push_kernel<<<dim3((unsigned)ctas, (unsigned)a.ws), 256, 0, st>>>(a);
}

}  // namespace b200
