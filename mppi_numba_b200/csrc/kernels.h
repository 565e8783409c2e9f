// kernels.h -- host-callable launchers of the engine's CUDA kernels (internal; the public
// surface is include/b200mppi.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "common.cuh"

namespace b200 {

// sample_grids_numba (terrain.py:633-694), bit-exact stream layout.
struct SampleGridsArgs {
  int8_t* grid;            // (num_maps, grid_rows, pitch) int8
  const int8_t* cum;       // cumulative PMF, (rows, cols, bpad) int8-as-uint8 (saturated at 127)
  uint64_t* states;        // (num_gen, 2)
  const int8_t* qvals;     // int8[bpad] quantised bin values (terrain.py:689)
  int num_bins, bpad;
  int rows, cols;          // padded PMF dims
  int grid_rows, pitch;
  int tx, ty, num_maps;
  double alpha_dyn;
};
void launch_sample_grids(const SampleGridsArgs& a, cudaStream_t st);
// v2 (staged, integer-threshold, optionally lin+ang fused) sampler -- see sample.cu
// [emu:begin sampler_args]
struct SampleTdm {
  int8_t* grid; const int8_t* cum; const uint64_t* states; uint64_t* states_out; const int8_t* qvals; int bpad;
};
struct SampleGridsV2Args {
  SampleTdm t[2];
  const uint64_t* thresholds;   // device, SAMPLE_TABLE_WORDS u64: thr | qbase per bucket (sample_threshold_q)
  const uint64_t* jump;         // device, [(segs-1)*2][128][2]: A^(s*seg_rows*width) for width class 0 / 1
  int rows, cols, grid_rows, pitch, tx, ty, num_maps;
  int segs, seg_rows;           // row segments per generator tile (jump-ahead split), rows per segment
  // reach box (sample_box_full() = the whole map): only rows [row_lo, row_hi) of tile rows [tix_lo, ...) and tile
  // columns [tiy_lo, tiy_lo + nact) are sampled; gm maps per CTA; write_states: the last segment of every
  // generator stores its advanced state (whole-map walks only -- a boxed launch leaves the states to
  // advance_states_kernel, which jumps every generator over its whole tile)
  int gm, tix_lo, tiy_lo, nact, row_lo, row_hi, write_states;
  // reach DISC inside the box (disc_r = 0: none): centre cell (disc_cx, disc_cy) and radius in cells, margins included;
  // a CTA samples only the tile columns its rows can reach (sample.cu)
  float disc_cx, disc_cy, disc_r;
};
constexpr int SG_GM = 8;          // maps per CTA of a whole-map launch
constexpr int SG_GM_MAX = 32;
inline void sample_box_full(SampleGridsV2Args& a) {
  a.gm = SG_GM; a.tix_lo = 0; a.tiy_lo = 0; a.nact = a.ty; a.row_lo = 0; a.row_hi = a.rows; a.write_states = 1;
  a.disc_cx = a.disc_cy = a.disc_r = 0.0f;
}
void build_jump_matrices(const int64_t* ks, int count, uint64_t* out);
void build_jump_series(int64_t k0, int64_t k1, int segs, uint64_t* out);     // (s-1)*2 + c -> A^(s * k_c), s = 1 .. segs-1
// q(r) of a RAW 64-bit draw r as a table lookup over its top 8 bits (see sample_threshold_q in common.cuh):
// table = thr[256] | qbase[256] (u64, qbase in the low 11 bits).  false if alpha is not representable that way.
constexpr int SAMPLE_TABLE_WORDS = 256;
// [emu:end sampler_args]
bool build_sample_thresholds(double alpha, int q_cap, uint64_t* table /*[SAMPLE_TABLE_WORDS]*/);
bool sample_grids_v2_fits(const SampleGridsV2Args& a, int nt);
void launch_sample_grids_v2(const SampleGridsV2Args& a, int nt, cudaStream_t st);
// batched one-map solves: equal launch configuration (grid, threads, shared memory, kernel variant)
bool sample_grids_v2_same_launch(const SampleGridsV2Args& a, const SampleGridsV2Args& b);
// ONE fused (nt = 2) launch for `count` pairs: descs = device array of their args, geom = any of them (host)
void launch_sample_grids_v2_batch(const SampleGridsV2Args& geom, const SampleGridsV2Args* descs, int count,
                                  cudaStream_t st);
// tile classes of a generator: (full | last) tile height x (full | last) tile width -> draws per whole-map walk
void sample_tile_draws(int rows, int cols, int tx, int ty, int64_t ks[4]);
// states_out[g] = states[g] advanced by the draws of a whole-map walk of generator g's tile (GF(2) jump with
// `mats` = [4][128][2] u64, the matrices of sample_tile_draws' four counts); out1 may be null
void launch_advance_states(const uint64_t* states, uint64_t* out0, uint64_t* out1, const uint64_t* mats, int rows,
                           int cols, int tx, int ty, int num_maps, cudaStream_t st);
// builds the (rows, cols, bpad) cumulative table from the (B, rows, cols) PMF
void launch_build_cum(const int8_t* pmf, int8_t* cum, int num_bins, int bpad, int rows, int cols,
                      cudaStream_t st);

void launch_collapse_pad(const int8_t* raw, int8_t* out, int8_t* risk, int* bad_columns, const float* bin_values, int B,
                         int H, int W, int keep_r, int keep_c, int pad, int risk_pitch, double alpha, float lo,
                         float range, int mode, cudaStream_t st);

// sample_noise_numba (mppi.py:1354-1370): generators (n_global*T + t); writes noise (N,T,2).
// `reach` (may be null): a device float the kernel zeroes for the prepare kernel's max-reduction
void launch_sample_noise(uint64_t* states, float* noise, int n_local, int T, float std_v,
                         float std_w, float* reach, cudaStream_t st);
// batched one-map solves: one launch samples the noise of `count` planners of equal N and T (planner = blockIdx.y)
// [emu:begin noise_desc]
struct NoiseDesc {
  uint64_t* states;         // (N*T, 2)
  float* noise;             // (N, T, 2)
  float std_v, std_w;
};
// [emu:end noise_desc]
void launch_sample_noise_batch(const NoiseDesc* descs, int count, int n_local, int T, cudaStream_t st);

// Where the per-(map, control sequence) cost of a stochastic rollout goes.  Layout is MAP-MAJOR: row m holds the
// costs of the control sequences on sampled map m, so the 32 lanes of a warp (consecutive n, same map) store one
// 128-byte line.  The control sequences are split into blocks of n_per (one block unless the maps are sharded over
// ranks: block d then belongs to rank d, which reduces those control sequences, and base[d] may point straight into
// rank d's receive buffer -- the all-to-all of the sharded solve is the rollout kernel's own epilogue).
// [emu:begin cost_dst]
constexpr int P2P_MAX_PEERS = 16;
struct CostDst {
  float* base[P2P_MAX_PEERS];   // block d: rows = maps, row stride ld, column = n - d*n_per
  int n_per;                    // control sequences per block
  int ld;                       // floats per row
  int row0;                     // row of this rank's map 0 inside a block
};
__host__ __device__ __forceinline__ float* cost_ptr(const CostDst& d, int m, int n) {
  const int b = n / d.n_per;
  return d.base[b] + (size_t)(d.row0 + m) * d.ld + (n - b * d.n_per);
}
// epoch flags raised in every peer once ALL CTAs of the kernel have stored (ws = 0: nothing to signal)
struct CostSignal {
  uint32_t* peer_flags[P2P_MAX_PEERS];   // peer d's cost flags [ws]; this rank writes entry `rank`
  unsigned* counter;                     // local, zero between launches
  int ws, rank;
  uint32_t epoch;
};
// [emu:end cost_dst]

// rollout kernels (mppi.py:613-1111)
// [emu:begin rollout_args]
struct RolloutArgs {
  RolloutParams p;
  int mode;
  const int8_t* lin_grid;   // (M|1, grid_rows, pitch)
  const int8_t* ang_grid;
  const int8_t* obstacle;   // (rows, cols)
  const int8_t* unknown;
  const int8_t* risk;       // (rows, cols) or null
  const float* noise;       // (N, T, 2)
  const float* u_cur;       // (T, 2)
  CostDst dst;              // MODE_TDM: per-(m, n) costs
  float* costs;             // (N)
  const float* obstacles;   // MODE_BAREBONE: (num_obstacles, 3) = x, y, radius
  int num_obstacles;
};
// [emu:end rollout_args]
void launch_rollout(const RolloutArgs& a, cudaStream_t st);
// batched one-map solves (mode 1, 2, 3): descs = device array of `count` RolloutArgs of equal N and T (blockIdx.y)
void launch_rollout_batch(const RolloutArgs* descs, int count, int mode, int N, int T, cudaStream_t st);
// windowed (TMA-staged) stochastic rollout kernel -- rollout_win.cu
// [emu:begin win_args]
struct RolloutWinArgs {
  RolloutParams p;
  int WW, WH, wx0, wy0;     // window size / origin in cells (origin inside the map, wx0 a multiple of 16)
  int ww, wh;               // the part of the window that lies inside the map: staged cells [0, ww) x [0, wh)
  int npad;                 // row length of noiseT
  int masks01;              // every obstacle / unknown byte is 0 or 1 (selects the kernel variant with the cheap penalties)
  int unit;                 // share granularity in chunks (set by launch_rollout_win)
  int sync_passes;          // 1: chunks dealt pass by pass with a CTA barrier in between (short shares), 0: shared counter
  long long* dbg;           // per-CTA timing record or null (debug hook)
  int rotate;               // debug: share of CTA b is the one of (b + rotate) % CTAs (B200MPPI_WIN_ROTATE; which SM runs which work)
  int stagger;              // cycles by which the warps of a scheduler are spread after a window barrier (0: none)
  const int8_t* lin_grid; const int8_t* ang_grid; const int8_t* obstacle; const int8_t* unknown;
  const float* noiseT;      // [T][npad] double2: clipped noisy controls (v, w), already widened to f64
  const float* ctrl;        // [npad]
  const float* u_cur;
  CostDst dst;              // per-(m, n) costs
  CostSignal sig;           // sharded solve with the peer-memory exchange: flags to raise when the kernel is done
};
// [emu:end win_args]
// reach (may be null): *reach = max(*reach, max_n sum_t |clipped v[n,t]|) -- bounds how far a rollout can travel
void launch_prepare_rollout(const float* noise, const float* u_cur, float* noiseT, float* ctrl, float* reach, int N,
                            int T, int npad, float lambda, float std_v, float std_w, const float vrange[2],
                            const float wrange[2], cudaStream_t st);
// sample_noise + prepare_rollout in one launch (solve(), windowed stochastic rollouts); reach[2]: slot is max-reduced
// into, slot ^ 1 cleared for the next launch
void launch_noise_prepare(uint64_t* states, float* noise, const float* u_cur, float* noiseT, float* ctrl, float* reach,
                          int slot, int N, int T, int npad, float lambda, float std_v, float std_w, const float vrange[2],
                          const float wrange[2], cudaStream_t st);
bool make_u8_tensor_map(void* out_map, const void* base, int rank, int cols, int rows, int maps, int pitch,
                        int WW, int WH);
void rollout_win_geometry(int T, int* WW, int* WH, size_t* smem);
int device_sm_count();                          // SMs of the current device (cached per device)
void rollout_win_set_debug(long long* dev);    // device buffer of 4 int64 per CTA (<= 1024 CTAs) or null
cudaError_t launch_rollout_win(const RolloutWinArgs& a, const void* tm_lin, const void* tm_ang, const void* tm_obs,
                               const void* tm_unk, cudaStream_t st);
// CVaR over M (mppi.py:718-755): costs[n] = mean of the ceil(M*alpha) largest of costs_mn[:, n]
// costs_mn is map-major: (M, n_cnt) with row stride ld -- the local buffer of a one-rank solve, or the receive buffer
// of a map-sharded solve (rows g*M/ws .. = rank g's maps): the same kernel, the same values per lane, hence
// bit-identical CVaR costs whatever the number of ranks.
int cvar_max_maps();   // largest M the CVaR kernels accept
// fw: flags to wait for before the costs are read (sharded solve, peer-memory exchange); FlagWait{} = none
void launch_cvar(const float* costs_mn, float* costs, int n_cnt, int ld, int M, float cvar_alpha, const FlagWait& fw,
                 cudaStream_t st);

// update_useq_numba (mppi.py:1113-1191) as an online-softmax two-level reduction
// [emu:begin update_args]
struct UpdateArgs {
  const float* costs;     // (N)
  const float* noise;     // (N, T, 2)
  float* w_raw;           // (N) exp(-(c-beta_cta)/lambda)
  float* cta_partials;    // (num_ctas, 2T+2): beta, S, V[2T]
  float* rank_partial;    // (2T+2)
  float* u_cur;           // (T,2) in/out
  float* weights;         // (N) normalised
  int N, T, num_ctas, rows_per_cta;
  float lambda, vrange[2], wrange[2];
};
// [emu:end update_args]
// what the LAST CTA of update_partial_kernel does once all CTA partials are written (reduce.cu)
// [emu:begin update_tail]
enum { UPD_TAIL_RANK = 0, UPD_TAIL_APPLY = 1, UPD_TAIL_BCAST = 2 };
struct UpdateTail {
  unsigned* counter;                    // ticket counter, zero between launches
  int mode;
  float* peer_gather[P2P_MAX_PEERS];    // UPD_TAIL_BCAST: peer d's gather buffer of this epoch's parity, (ws, 2T+2)
  uint32_t* peer_flags[P2P_MAX_PEERS];  // peer d's partial flags [ws]
  int ws, rank;
  uint32_t epoch;
  float* u_prev;                        // UPD_TAIL_APPLY, when set: the new u is also stored here (T,2) ...
  float* u_out;                         // ... and here (batched solves: u_prev alias, contiguous (K,T,2) result)
};
// [emu:end update_tail]
// [emu:begin update_desc]
struct UpdateBatchDesc {               // one planner of a batched update launch (blockIdx.y)
  UpdateArgs a;
  UpdateTail tl;
};
// [emu:end update_desc]
int update_num_ctas(int N);
void launch_update_partial(const UpdateArgs& a, const UpdateTail& tl, cudaStream_t st);
// batched one-map solves: `count` planners of equal N (hence equal num_ctas), UPD_TAIL_APPLY each
void launch_update_partial_batch(const UpdateBatchDesc* descs, int count, int num_ctas, cudaStream_t st);
// combine `count` partials (each 2T+2 floats; this rank's own partial is entry `self`) into u and weights
void launch_update_finish(const UpdateArgs& a, const float* gathered, int count, const FlagWait& fw, cudaStream_t st);

void launch_shift_u(float* u, int T, int shifts, cudaStream_t st);

// visualisation rollouts (mppi.py:1194-1351)
// [emu:begin vis_args]
struct VisArgs {
  RolloutParams p;
  int mode, V;
  const int8_t* lin_grid; const int8_t* ang_grid;
  const float* noise; const float* u_cur; const float* u_prev;
  float* out;   // (V, T+1, 3)
};
// [emu:end vis_args]
void launch_state_rollout(const VisArgs& a, cudaStream_t st);

// peer-memory exchange of the sharded solve (p2p.cu)
struct P2PPushArgs {
  const float* costs_nm;              // local staged blocks (ws, Mc, n_red): block d = this rank's maps x rank d's control sequences
  float* peer_recv[P2P_MAX_PEERS];    // peer d's receive buffer (ws, Mc, n_red): block `rank` is written
  uint32_t* peer_flags[P2P_MAX_PEERS];// peer d's cost flags [ws]
  unsigned* counter;                  // local, zero between launches
  int ws, rank, n_red, Mc;
  uint32_t epoch;
};
void launch_p2p_push(const P2PPushArgs& a, cudaStream_t st);

// host: numba-compatible generator states (random.py:226-241)
void create_xoroshiro_states(uint64_t* host_out, int64_t first, int64_t count, uint64_t seed);

}  // namespace b200
