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
// shared memory / fit of a staged launch over tile columns [tiy_lo, tiy_lo + nact) with gm maps per CTA (nt TDMs)
__host__ __device__ inline size_t sample_v2_smem_hd(int tiy_lo, int nact, int ty, int cols, int bpad, int gm, int nt) {
  const int ncol = (cols + ty - 1) / ty;
  const int cfirst = tiy_lo * ncol < cols ? tiy_lo * ncol : cols;
  const int cs1 = (tiy_lo + nact) * ncol < cols ? (tiy_lo + nact) * ncol : cols;
  const int wcols = cs1 - (cfirst & ~15);
  const int row_bytes_al = (wcols * bpad + 15) & ~15;
  const int stage_pitch = (wcols + 15) & ~15;
  size_t stage = (size_t)nt * gm * stage_pitch;
  if (stage < (size_t)2 * 128 * 16) stage = (size_t)2 * 128 * 16;           // the jump matrices overlay it
  return (size_t)nt * row_bytes_al + stage + SAMPLE_TABLE_WORDS * 8 + (size_t)nt * 128;
}
__host__ __device__ inline bool sample_v2_fits_hd(int tiy_lo, int nact, int ty, int cols, int bpad0, int bpad1, int gm,
                                                  int nt) {
  return gm >= 1 && gm <= SG_GM_MAX && nact >= 1 && tiy_lo >= 0 && tiy_lo + nact <= ty &&
         ((nact * gm + 31) / 32) * 32 <= 256 && bpad0 <= 32 &&
         sample_v2_smem_hd(tiy_lo, nact, ty, cols, bpad0, gm, nt) <= 200 * 1024 && (nt == 1 || bpad0 == bpad1);
}

// The reach box of a solve's map sampling (planner_reach_box + plan_box in api.cu; the batched trial sampler decides it
// on the device with the same function).  A rollout moves at most |traction| * |v| * dt per step, so it stays within
// R = dt * max|traction| * S of x0, S = sum_t |v_t| -- bounded by T * max|vrange| (static box) or by `reach`, the max
// over the N control sequences actually drawn.  Whole maps (0) whenever the bound is not airtight: the box would leave
// the map (out-of-map indices wrap), non-finite inputs, a reach beyond the speed limit.  Float64 operations are
// explicitly rounded on the device, so host and device decide alike.
// Float32 rounding moves a rollout further than that: every step stores x = f32(x + dv cos th), up to half an ulp of |x|
// away, so far from the origin (georeferenced maps) a displacement just above half an ulp rounds up to a whole one at
// every step.  reach_radius adds that drift and the rounding of f32(x - xlo) in the cell index.
#ifdef __CUDA_ARCH__
#define RB_MUL(a, b) __dmul_rn(a, b)
#define RB_ADD(a, b) __dadd_rn(a, b)
#define RB_SUB(a, b) __dsub_rn(a, b)
#define RB_DIV(a, b) __ddiv_rn(a, b)
#else
#define RB_MUL(a, b) ((a) * (b))
#define RB_ADD(a, b) ((a) + (b))
#define RB_SUB(a, b) ((a) - (b))
#define RB_DIV(a, b) ((a) / (b))
#endif
struct ReachBoxConst {          // a planner's constants of the decision
  int mode;                     // 0: whole maps (box off or no windowed rollout), 1: static bound, 2: reach statistic
                                //    (box_mode 2 with num_opt 1: the device path then reads the statistic)
  int disc;                     // narrow to the reach disc (B200MPPI_SAMPLE_DISC)
  int T;
  float vr0, vr1, dt, tr_abs_max, res, pxl, pyl;
  int rows, cols;
  // the staged launch of TDM 0 (apply_box, sample_grids_v2_fits): nt = 2 fused pair, 1 one TDM, 0 generic kernel
  int nt, tx, ty, num_maps, bpad0, bpad1;
};
struct ReachBox {
  int geo;                      // the box exists (inside the map, finite bound) -- TDM 1 of an unfused pair may use it
  int how;                      // the decision for TDM 0: 0 whole maps, 1 static box, 2 box from the reach statistic
  int row_lo, row_hi, col_lo, col_hi;     // cells [row_lo, row_hi) x [col_lo, col_hi) (whole map when how = 0)
  float cx, cy, r;              // reach disc in cells (r = 0: none)
  int tiy_lo, nact, gm;         // the boxed launch's tile columns and maps per CTA (how != 0)
};
// R in metres for a path length S (sum_t |v_t|) from a start x0 with |x0| + |y0| <= A and |x0 - pxl| + |y0 - pyl| <= B:
// every cell a rollout reads at steps 0 .. T-1 lies within R of x0, per axis and in Euclidean distance.
//   R0 = dt * max|traction| * S * 1.0002: the exact path (1.0002: cos/sin.approx may exceed 1 by ~1e-6).
//   Each of the T state roundings is off by at most u |x|, |x| <= A + D (D: the distance travelled so far), so
//   D <= R0 + T u (A + D), i.e. D <= (R0 + T u A) / (1 - T u).  u = 2^-24 rounded up also covers the float64 rounding of
//   the FMA before the narrowing to float32.
//   The cell index rounds x - xlo once more: u (|x0 - pxl| + |y0 - pyl| + 2 D).
// Negative (no usable bound) when T u is not small.
__host__ __device__ inline double reach_radius(const ReachBoxConst& c, double S, double A, double B) {
  const double u = 5.9605e-8;                            // 2^-24 = 5.96046e-8
  const double Tu = RB_MUL((double)c.T, u);
  if (!(Tu < 0.5)) return -1.0;
  const double R0 = RB_MUL(RB_MUL(RB_MUL((double)c.dt, (double)c.tr_abs_max), S), 1.0002);
  if (!(R0 >= 0.0)) return -1.0;                         // negative or NaN
  const double D = RB_DIV(RB_ADD(R0, RB_MUL(Tu, A)), RB_SUB(1.0, Tu));
  return RB_ADD(D, RB_MUL(u, RB_ADD(B, RB_MUL(2.0, D))));
}
__host__ __device__ inline int reach_box_decide(const ReachBoxConst& c, float x0x, float x0y, const float* reach,
                                                ReachBox* b) {
  b->geo = 0; b->how = 0;
  b->row_lo = 0; b->row_hi = c.rows; b->col_lo = 0; b->col_hi = c.cols;
  b->cx = b->cy = b->r = 0.0f;
  b->tiy_lo = 0; b->nact = c.ty; b->gm = 0;
  if (c.mode == 0) return 0;
  double S = RB_MUL((double)c.T, fmax(fabs((double)c.vr0), fabs((double)c.vr1)));
  int how = 1;
  if (reach) {
    if (!((double)*reach <= S)) return 0;               // NaN or beyond the speed limit: not a usable bound
    S = (double)*reach;
    how = 2;
  }
  // R from the start's own coordinates; the box adds a cell of margin on each side below
  const double res = (double)c.res, x = (double)x0x, y = (double)x0y;
  const double R = reach_radius(c, S, RB_ADD(fabs(x), fabs(y)),
                                RB_ADD(fabs(RB_SUB(x, (double)c.pxl)), fabs(RB_SUB(y, (double)c.pyl))));
  if (!(R >= 0.0 && R <= 1.7976931348623157e308)) return 0;      // negative, NaN or infinite
  const double fx0 = RB_DIV(RB_SUB(RB_SUB(x, R), (double)c.pxl), res);
  const double fx1 = RB_DIV(RB_SUB(RB_ADD(x, R), (double)c.pxl), res);
  const double fy0 = RB_DIV(RB_SUB(RB_SUB(y, R), (double)c.pyl), res);
  const double fy1 = RB_DIV(RB_SUB(RB_ADD(y, R), (double)c.pyl), res);
  if (!(fx0 > 2.0 && fy0 > 2.0 && fx1 < RB_SUB((double)c.cols, 3.0) && fy1 < RB_SUB((double)c.rows, 3.0))) return 0;
  b->geo = 1;
  b->col_lo = (int)floor(fx0) - 1; b->col_hi = (int)floor(fx1) + 3;      // [lo, hi)
  b->row_lo = (int)floor(fy0) - 1; b->row_hi = (int)floor(fy1) + 3;
  // the same bound as a disc: a rollout stays within Euclidean distance R of x0, so the cell it reads lies within
  // R/res + sqrt(2) cells of the robot's (fractional) cell position; + 1.5 for float32 effects, rounded up
  b->cx = (float)RB_DIV(RB_SUB(x, (double)c.pxl), res);
  b->cy = (float)RB_DIV(RB_SUB(y, (double)c.pyl), res);
  b->r = c.disc ? (float)RB_ADD(RB_DIV(R, res), 3.0) * 1.0001f : 0.0f;
  // apply_box's narrowing of TDM 0's staged launch; a box whose launch does not fit samples whole maps
  const int ncol = (c.cols + c.ty - 1) / c.ty;
  b->tiy_lo = b->col_lo / ncol;
  b->nact = (b->col_hi - 1) / ncol - b->tiy_lo + 1;
  int gm = 128 / b->nact;                                // ~4 warps per CTA whatever the number of active tile columns
  if (gm > SG_GM_MAX) gm = SG_GM_MAX;
  if (gm > c.num_maps) gm = c.num_maps;
  if (gm < 1) gm = 1;
  b->gm = gm;
  if (c.nt == 0 || !sample_v2_fits_hd(b->tiy_lo, b->nact, c.ty, c.cols, c.bpad0, c.bpad1, gm, c.nt)) return 0;
  b->how = how;
  return how;
}
// [emu:end sampler_args]
bool build_sample_thresholds(double alpha, int q_cap, uint64_t* table /*[SAMPLE_TABLE_WORDS]*/);
bool sample_grids_v2_fits(const SampleGridsV2Args& a, int nt);
void launch_sample_grids_v2(const SampleGridsV2Args& a, int nt, cudaStream_t st);
// batched one-map solves: equal launch configuration (grid, threads, shared memory, kernel variant)
bool sample_grids_v2_same_launch(const SampleGridsV2Args& a, const SampleGridsV2Args& b);
// ONE fused (nt = 2) launch for `count` pairs: descs = device array of their args, geom = any of them (host)
// active (device, may be null): active[pair] == 0 -> that pair's CTAs return at once (closed-loop trials)
void launch_sample_grids_v2_batch(const SampleGridsV2Args& geom, const SampleGridsV2Args* descs, int count,
                                  const int* active, cudaStream_t st);
// closed-loop trials of a stochastic batch: each pair's reach box decided on the device, from the x0 the plant step
// wrote and the reach statistic of the step's first iteration (slot ^ (iter & 1)).  The decision goes to `record`:
// [how, row_lo, row_hi, col_lo, col_hi] as b200mppi_planner_sample_box reports it.
// [emu:begin box_desc]
struct SampleBoxDesc {
  ReachBoxConst c;
  const float* x0;              // RolloutWinArgs::p.x0 of the pair's planner in the batch's device descriptors
  const float* reach;           // the planner's two reach slots
  int slot;                     // slot of the call's first iteration
  int* record;                  // [5]
  const uint64_t* jump_tile;    // [4][128][2] whole-tile advance matrices (advance_states_batch_kernel)
};
// [emu:end box_desc]
// ONE launch for `count` fused pairs of equal geometry (geom: a whole-map plan with the boxed launch's segs / seg_rows /
// jump and maps per CTA gm): mrows tile rows x the row segments x ncact tile columns, sized for the largest box of the
// static bound; every CTA narrows to its pair's box and disc, whole maps loop over row and column groups.  No state
// stores: launch_advance_states_batch advances the states.
void launch_sample_grids_v2_box_batch(const SampleGridsV2Args& geom, const SampleGridsV2Args* descs,
                                      const SampleBoxDesc* boxes, int count, const int* active, int iter, int mrows,
                                      int ncact, cudaStream_t st);
// the launch above holds ncact tile columns with geom.gm maps per CTA (threads, shared memory)
bool sample_box_batch_fits(const SampleGridsV2Args& geom, int ncact);
// launch_advance_states for `count` pairs (pair blockIdx.y): descs[y].t[0].states -> both TDMs' states_out
void launch_advance_states_batch(const SampleGridsV2Args* descs, const SampleBoxDesc* boxes, int count, int rows,
                                 int cols, int tx, int ty, int num_maps, const int* active, cudaStream_t st);
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
void launch_sample_noise_batch(const NoiseDesc* descs, int count, int n_local, int T, const int* active,
                               cudaStream_t st);

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
void launch_rollout_batch(const RolloutArgs* descs, int count, int mode, int N, int T, const int* active,
                          cudaStream_t st);
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
// batched stochastic solves: one noise + prepare launch for `count` planners of equal N, T (planner = blockIdx.y)
// [emu:begin noise_prep_desc]
struct NoisePrepDesc {
  uint64_t* states;         // (N*T, 2)
  float* noise;             // (N, T, 2)
  const float* u_cur;       // (T, 2)
  float* noiseT;            // [T + 1][npad] double2
  float* ctrl;              // [npad]
  float* reach;             // the planner's two reach slots
  int slot;                 // slot of the solve's first iteration
  float std_v, std_w, lambda, sv2, sw2, v_lo, v_hi, w_lo, w_hi;
};
// [emu:end noise_prep_desc]
// active (device, may be null): active[y] == 0 -> that planner is left untouched (closed-loop trials)
void launch_noise_prepare_batch(const NoisePrepDesc* descs, int count, int N, int T, int npad, int iter,
                                const int* active, cudaStream_t st);
bool make_u8_tensor_map(void* out_map, const void* base, int rank, int cols, int rows, int maps, int pitch,
                        int WW, int WH);
void rollout_win_geometry(int T, int* WW, int* WH, size_t* smem);
int device_sm_count();                          // SMs of the current device (cached per device)
void rollout_win_set_debug(long long* dev);    // device buffer of 4 int64 per CTA (<= 1024 CTAs) or null
cudaError_t launch_rollout_win(const RolloutWinArgs& a, const void* tm_lin, const void* tm_ang, const void* tm_obs,
                               const void* tm_unk, cudaStream_t st);
// batched stochastic solves: the window height of a batched launch (its shared memory also holds one planner record)
int rollout_win_batch_height(int T);
// ONE persistent launch over the (planner, map) units of `count` planners of equal N, M, T: g = the launch-wide fields
// (p.N, p.M, p.T, npad, WH), descs = device array of each planner's own RolloutWinArgs, tmaps = device array (64-byte
// aligned) of 4 encoded tensor maps per planner (lin, ang, obstacle, unknown); masks01: every planner's masks are 0/1
// active (device, may be null): the units of a planner with active[k] == 0 are skipped (closed-loop trials)
cudaError_t launch_rollout_win_batch(const RolloutWinArgs& g, const RolloutWinArgs* descs, const void* tmaps, int count,
                                     bool masks01, const int* active, cudaStream_t st);
// CVaR over M (mppi.py:718-755): costs[n] = mean of the ceil(M*alpha) largest of costs_mn[:, n]
// costs_mn is map-major: (M, n_cnt) with row stride ld -- the local buffer of a one-rank solve, or the receive buffer
// of a map-sharded solve (rows g*M/ws .. = rank g's maps): the same kernel, the same values per lane, hence
// bit-identical CVaR costs whatever the number of ranks.
int cvar_max_maps();   // largest M the CVaR kernels accept
// fw: flags to wait for before the costs are read (sharded solve, peer-memory exchange); FlagWait{} = none
void launch_cvar(const float* costs_mn, float* costs, int n_cnt, int ld, int M, float cvar_alpha, const FlagWait& fw,
                 cudaStream_t st);
int cvar_warp_max_maps();   // largest M of the warp kernel (the one the batched launch runs)
// batched stochastic solves: one warp-kernel launch for `count` planners of equal n_cnt and M (planner = blockIdx.y)
// [emu:begin cvar_desc]
struct CvarDesc {
  const float* costs_mn;    // map-major (M, ld)
  float* costs;             // (n_cnt)
  int n_cnt, ld, M, numel;  // numel = ceil(M * cvar_alpha) clamped to [1, M], as launch_cvar computes it
  const int* active;        // may be null: *active == 0 -> the planner is left untouched (closed-loop trials)
};
// [emu:end cvar_desc]
int cvar_numel(int M, float cvar_alpha);
void launch_cvar_batch(const CvarDesc* descs, int count, int n_cnt, int M, cudaStream_t st);

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
void launch_update_partial_batch(const UpdateBatchDesc* descs, int count, int num_ctas, const int* active,
                                 cudaStream_t st);
// combine `count` partials (each 2T+2 floats; this rank's own partial is entry `self`) into u and weights
void launch_update_finish(const UpdateArgs& a, const float* gathered, int count, const FlagWait& fw, cudaStream_t st);

void launch_shift_u(float* u, int T, int shifts, cudaStream_t st);

// closed-loop trials of a batch (b200mppi_batch_run_trials): the plant step of every running planner, one warp each
// [emu:begin trial_args]
enum { TRIAL_RUNNING = 0, TRIAL_GOAL = 1, TRIAL_MAX_STEPS = 2, TRIAL_LEFT_MAP = 3 };
// The window of a rollout from x0 (fill_win_args in api.cu, and the plant step of stochastic trials): WW x WH cells
// centred on the robot's cell, kept INSIDE the map (origin clamped, extents cut), the x origin floored to a multiple of
// 16 (TMA: 16-byte aligned inner start coordinate, also for negatives).  A staged cell is then always a map cell; indices
// outside the map take the generic kernel's wrap + clamp.  f = &RolloutWinArgs::WW: {WW, WH, wx0, wy0, ww, wh}.
__host__ __device__ inline void win_origin(float x0x, float x0y, float pxl, float pyl, float res, int cols, int rows,
                                           int* f) {
#ifdef __CUDA_ARCH__
  const int xi0 = (int)floor(__ddiv_rn(__dsub_rn((double)x0x, (double)pxl), (double)res));
  const int yi0 = (int)floor(__ddiv_rn(__dsub_rn((double)x0y, (double)pyl), (double)res));
#else
  const int xi0 = (int)floor(((double)x0x - (double)pxl) / (double)res);
  const int yi0 = (int)floor(((double)x0y - (double)pyl) / (double)res);
#endif
  const int WW = f[0], WH = f[1];
  int cx = xi0 - WW / 2, cy = yi0 - WH / 2;
  if (cx > cols - WW) cx = cols - WW;
  if (cx < 0) cx = 0;
  if (cy > rows - WH) cy = rows - WH;
  if (cy < 0) cy = 0;
  f[2] = cx & ~15;
  f[3] = cy;
  f[4] = WW < cols - f[2] ? WW : cols - f[2];
  f[5] = WH < rows - f[3] ? WH : rows - f[3];
}
struct TrialDev {
  const double* lin; const double* ang;   // ground-truth traction (H, W), float64
  int H, W;
  double xlo, ylo, res, dt, xgoal[2], tol, pxlim[2], pylim[2];
  float* u_cur;                           // (T, 2): u_cur[0] is applied, then the sequence is shifted by one
  float* x0_out;                          // RolloutArgs::p.x0 of this planner in the batch's device descriptors
  // stochastic trials: &RolloutWinArgs::WW of the planner in the batch's device descriptors (x0_out points into the
  // same record), whose window is recomputed from the new x0 (win_origin) over the map of the planner's TDMs; else null
  int* win;
  float win_pxl, win_pyl, win_res;
  int win_rows, win_cols;
};
struct TrialState {
  double x[3], cum_obj, cum_dist, dist;
  int steps, status;
};
struct PlantArgs {
  const TrialDev* trials; TrialState* state;
  int* active; int* active_count;
  double* xhist;                          // (K, max_steps+1, 3)
  float* uhist;                           // (K, max_steps, 2)
  int K, T, max_steps, step;
};
// [emu:end trial_args]
void launch_plant_step(const PlantArgs& a, cudaStream_t st);

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
