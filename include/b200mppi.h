/*
 * b200mppi.h -- C-ABI of the H100-native MPPI rollout-and-reduction engine.
 *
 * This is the drop-in boundary for the ONE hot path of mit-acl/mppi_numba:
 *   MPPI_Numba.solve()  (reference mppi_numba/mppi.py:186-211)  =
 *     TDM_Numba.sample_grids x2 (terrain.py:610-694) -> sample_noise_numba (mppi.py:1354-1370)
 *     -> rollout_numba / rollout_det_dyn_numba / rollout_det_dyn_w_speed_map_numba (mppi.py:613-1111)
 *     -> update_useq_numba (mppi.py:1113-1191) -> D2H of u_cur (T x 2 float32).
 *
 * The reference has no FFI of its own (it is pure Python + Numba-JIT kernels); the seam a maintainer
 * would bind is the set of Numba kernel launches and cuda.to_device / copy_to_host calls inside
 * MPPI_Numba and TDM_Numba.  Each entry point below names the reference code it replaces.
 * INTEGRATION.md shows the ctypes stub.
 *
 * Conventions: plain C types only; every function returns 0 on success or a negative B200MPPI_E*
 * code, b200mppi_last_error() returns the message of the last failure on the calling thread;
 * the caller owns all host buffers, the library owns all device buffers; handles are not
 * thread-safe (one host thread per handle, like the reference); all work is issued on the
 * handle's stream (b200mppi_*_set_stream; default: a private non-blocking stream).
 * There is NO CPU fallback: without a CUDA device every *_create fails with B200MPPI_ECUDA.
 */
#ifndef B200MPPI_H
#define B200MPPI_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200MPPI_VERSION 1

enum {
  B200MPPI_OK = 0,
  B200MPPI_EINVAL = -1,   /* bad argument / shape mismatch */
  B200MPPI_ESTATE = -2,   /* call order (e.g. solve before maps/params are set) */
  B200MPPI_ECUDA = -3,    /* CUDA runtime/driver error (text in last_error) */
  B200MPPI_ENOMEM = -4
};

/* Planner modes == the reference's mutually exclusive Config flags (config.py:41-47). */
enum {
  B200MPPI_MODE_TDM = 0,        /* use_tdm: M sampled traction maps, CVaR of the cost        */
  B200MPPI_MODE_DET_DYN = 1,    /* use_det_dynamics: one worst-case-expectation map          */
  B200MPPI_MODE_SPEED_MAP = 2,  /* use_nom_dynamics_with_speed_map: nominal map + speed map  */
  B200MPPI_MODE_BAREBONE = 3    /* map-free variant of barebone_mppi_numba.ipynb: quadratic cost,
                                   circular obstacles, no TDMs (set_obstacles instead of set_tdms) */
};

/* Fixed sizes, == Config (config.py:16-100) after its clamps. */
typedef struct {
  int32_t num_steps;              /* T = int(T_s/dt)                                  */
  int32_t num_control_rollouts;   /* N, GLOBAL count over all ranks                   */
  int32_t num_grid_samples;       /* M (only MODE_TDM uses more than map 0)           */
  int32_t max_map_rows;           /* cfg.max_map_dim[0]  (Rmax)                       */
  int32_t max_map_cols;           /* cfg.max_map_dim[1]  (Cmax)                       */
  int32_t tdm_thread_x;           /* cfg.tdm_sample_thread_dim[0] (RNG stream layout) */
  int32_t tdm_thread_y;           /* cfg.tdm_sample_thread_dim[1]                     */
  int32_t num_vis_state_rollouts; /* V                                                */
  int32_t mode;                   /* B200MPPI_MODE_*                                  */
  int32_t device;                 /* CUDA device ordinal                              */
  int32_t rank;                   /* this process' shard of the N rollouts ...        */
  int32_t world_size;             /* ... rollouts [rank*N/ws, (rank+1)*N/ws)          */
  uint64_t seed;                  /* cfg.seed (same seed for planner and both TDMs)   */
} b200mppi_config;

/* Per-solve task parameters, == the params dict uploaded by move_mppi_task_vars_to_device
 * (mppi.py:214-234), already cast to float32 as the reference casts them. */
typedef struct {
  float dt;
  float x0[3];
  float xgoal[2];
  float goal_tolerance;
  float v_post_rollout;
  float cvar_alpha;
  float lambda_weight;
  float u_std[2];
  float vrange[2];
  float wrange[2];
  float obs_penalty;      /* DEFAULT_OBS_COST 1e5  (mppi.py:33) */
  float unknown_penalty;  /* DEFAULT_UNKNOWN_COST 1e2 (mppi.py:32) */
  float dist_weight;      /* DEFAULT_DIST_WEIGHT 1.0 (mppi.py:36) */
  int32_t num_opt;
  double alpha_dyn;       /* passed to sample_grids (mppi.py:392-395); 1.0 when absent */
} b200mppi_params;

typedef struct b200mppi_tdm b200mppi_tdm;         /* == one TDM_Numba's device state  */
typedef struct b200mppi_planner b200mppi_planner; /* == one MPPI_Numba's device state */

const char* b200mppi_last_error(void);
int b200mppi_version(void);
/* Number of visible CUDA devices (0 on a GPU-less host); never fails. */
int b200mppi_device_count(void);

/* ------------------------------------------------------------------ traction distribution map */
/* TDM_Numba.init_device_vars_before_sampling (terrain.py:164-180): allocates the
 * (M|1, Rmax, Cmax) int8 sample buffer and the M*tx*ty (tx*ty in the deterministic modes)
 * xoroshiro128+ generators seeded with cfg.seed. */
int b200mppi_tdm_create(const b200mppi_config* cfg, b200mppi_tdm** out);
int b200mppi_tdm_destroy(b200mppi_tdm* tdm);
int b200mppi_tdm_set_stream(b200mppi_tdm* tdm, void* cuda_stream);

/* The H2D half of set_TDM_from_PMF_grid / set_TDM_from_semantic_grid (terrain.py:340-343,405-406,506):
 * padded PMF int8 (B, Hp, Wp) in percent, bin_values float32[B], bounds float32[2], plus the map
 * geometry the planner reads from lin_tdm (res, padded_xlimits, padded_ylimits; mppi.py:215-217). */
int b200mppi_tdm_set_pmf(b200mppi_tdm* tdm, const int8_t* pmf_padded, int32_t num_bins,
                         int32_t rows, int32_t cols, const float* bin_values,
                         const float bounds[2], float res, const float padded_xlimits[2],
                         const float padded_ylimits[2]);
/* The one-map modes' PMF preprocessing of set_TDM_from_PMF_grid ON THE DEVICE (terrain.py:408-495 fused with
 * the crop + zero-traction padding of :511-543): raw int8 PMF (B, H, W) in percent -> per cell the mean
 * (alpha == 1) or the expectation over the worst alpha tail -> one-hot PMF at the first bin >= it
 * (MODE_DET_DYN) or nominal PMF + int8 worst-case speed map (MODE_SPEED_MAP); the top-left keep_rows x
 * keep_cols cells are kept and surrounded by `pad` padding cells.  Ends like set_pmf (+ set_risk_map).
 * Optional host outputs: the padded PMF (B, keep_rows+2pad, keep_cols+2pad), the padded risk map, and the
 * number of raw columns that do not sum to 100 (the reference prints a warning for them). */
int b200mppi_tdm_set_pmf_collapsed(b200mppi_tdm* tdm, const int8_t* pmf_raw, int32_t num_bins, int32_t rows,
                                   int32_t cols, int32_t keep_rows, int32_t keep_cols, int32_t pad,
                                   const float* bin_values, const float bounds[2], float res,
                                   const float padded_xlimits[2], const float padded_ylimits[2], double alpha,
                                   int8_t* pmf_padded_out, int8_t* risk_padded_out, int32_t* bad_columns_out);
/* Override the int8 value written for each bin (default: terrain.py:689 evaluated with float32
 * bin values as set_TDM_from_PMF_grid uploads them).  set_TDM_from_semantic_grid uploads the
 * caller's bin_values UNCAST (terrain.py:331-332), so with float64 inputs Numba evaluates the same
 * expression in float64; the host mirror computes that variant and installs it here. */
int b200mppi_tdm_set_bin_quantisation(b200mppi_tdm* tdm, const int8_t* qvals, int32_t num_bins);
/* Raw device view of the sample buffer: base pointer and row pitch in bytes (rows are padded to a
 * multiple of 16 B; element (m, r, c) lives at base + (m*Rmax + r)*pitch + c). */
int b200mppi_tdm_sample_grid_view(b200mppi_tdm* tdm, void** dev_ptr, int32_t* pitch_bytes);
/* prepare_obstacle_and_unknown_map's H2D (terrain.py:370-371): padded int8 (Hp, Wp) masks. */
int b200mppi_tdm_set_masks(b200mppi_tdm* tdm, const int8_t* obstacle_padded,
                           const int8_t* unknown_padded, int32_t rows, int32_t cols);
/* risk_traction_map_d (terrain.py:308,495): padded int8 (Hp, Wp) worst-case speed map. */
int b200mppi_tdm_set_risk_map(b200mppi_tdm* tdm, const int8_t* risk_padded, int32_t rows,
                              int32_t cols);
/* TDM_Numba.sample_grids (terrain.py:610-622) == kernel sample_grids_numba (terrain.py:633-694):
 * bit-exact xoroshiro128+ stream layout (generator tid_x*(ty*M)+m*ty+tid_y walks its tile
 * row-major, one draw per cell). */
int b200mppi_tdm_sample_grids(b200mppi_tdm* tdm, double alpha_dyn);
/* sample_grid_batch_d.copy_to_host(): int8 (M|1, Rmax, Cmax), C order. */
int b200mppi_tdm_get_sample_grids(b200mppi_tdm* tdm, int8_t* out, size_t bytes);
/* Parity hook: overwrite the sample buffer with caller-provided grids (same shape). */
int b200mppi_tdm_set_sample_grids(b200mppi_tdm* tdm, const int8_t* in, size_t bytes);
/* rng_states_d.copy_to_host() / checkpoint-resume: uint64 (num_generators, 2) = (s0, s1),
 * the same 16-byte layout as numba's xoroshiro128p_dtype. */
int b200mppi_tdm_num_generators(b200mppi_tdm* tdm, int64_t* out);
int b200mppi_tdm_get_rng_states(b200mppi_tdm* tdm, uint64_t* out, size_t bytes);
int b200mppi_tdm_set_rng_states(b200mppi_tdm* tdm, const uint64_t* in, size_t bytes);

/* ------------------------------------------------------------------ planner */
/* MPPI_Numba.init_device_vars_before_solving (mppi.py:108-127): noise (N,T,2), u_cur/u_prev (T,2),
 * costs (N), weights (N), N*T xoroshiro128+ generators, vis buffer (V,T+1,3).  With
 * world_size > 1 the planner owns only its shard of N (generators n*T+t keep their GLOBAL index,
 * so results do not depend on world_size). */
int b200mppi_planner_create(const b200mppi_config* cfg, b200mppi_planner** out);
int b200mppi_planner_destroy(b200mppi_planner* pl);
int b200mppi_planner_set_stream(b200mppi_planner* pl, void* cuda_stream);
/* MPPI_Numba.set_tdm (mppi.py:152-155): the TDMs are BORROWED; obstacle/unknown/risk maps and
 * the map geometry are read from lin (mppi.py:266-270). */
int b200mppi_planner_set_tdms(b200mppi_planner* pl, b200mppi_tdm* lin, b200mppi_tdm* ang);
/* MODE_BAREBONE: the notebook's obstacle_positions (K,2) / obstacle_radius (K) (barebone_mppi_numba.ipynb
 * cell 3, move_mppi_task_vars_to_device); K = 0 clears them.  params.obs_penalty is the obstacle cost. */
int b200mppi_planner_set_obstacles(b200mppi_planner* pl, const float* positions_xy, const float* radius,
                                   int32_t count);
/* move_mppi_task_vars_to_device (mppi.py:214-234): one POD struct instead of 7 cuda.to_device. */
int b200mppi_planner_set_params(b200mppi_planner* pl, const b200mppi_params* p);
/* u_cur_d = cuda.to_device(u) (mppi.py:114,542) / u_cur_d.copy_to_host(): float32 (T,2). */
int b200mppi_planner_set_u(b200mppi_planner* pl, const float* u);
int b200mppi_planner_get_u(b200mppi_planner* pl, float* u_out);
/* shift_optimal_control_sequence (mppi.py:539-542) done on the device: u[:-s] = u[s:]. */
int b200mppi_planner_shift_u(b200mppi_planner* pl, int32_t num_shifts);

/* solve_det_dyn / solve_nom_dyn_w_speed_map / solve_stochastic (mppi.py:237-451), world_size 1:
 * sample both TDMs, then num_opt x (noise, rollout, CVaR, update); returns u_cur (T,2) in u_out. */
int b200mppi_planner_solve(b200mppi_planner* pl, float* u_out);

/* Multi-GPU, MODE_TDM (the M sampled maps are sharded: rank r owns maps [r*M/ws, (r+1)*M/ws), samples
 * only those -- bit-identical to the same maps of a single-rank run -- and rolls out ALL N control
 * sequences on them):
 *   solve_local  : noise, [first_iteration: sample this rank's maps], rollouts -> the device buffer
 *                  B200MPPI_BUF_COSTS_NM, map-major and already split by destination: (ws, M/ws, N/ws) float32,
 *                  block d = this rank's maps x the control sequences [d*N/ws, (d+1)*N/ws) that rank d reduces --
 *                  the send buffer of an all-to-all with equal contiguous blocks.
 *   solve_reduce : CVaR over all M maps for this rank's N/ws control sequences from the received buffer
 *                  (ws, M/ws, N/ws) float32 (block g = rank g's maps; i.e. the map-major (M, N/ws) array), then
 *                  this rank's softmax partial (2T+2 float32).
 *   solve_finish : as below.
 * Multi-GPU, deterministic modes (one map): the N control sequences are sharded, no solve_reduce. */
int b200mppi_planner_solve_reduce(b200mppi_planner* pl, const float* exchanged_costs_dev);

/* Multi-GPU (world_size > 1): one optimisation iteration split around the single exchange.
 *   solve_local : [first_iteration: sample both TDMs] noise, rollout, CVaR, and this rank's softmax
 *                 partial  (beta_r = min cost, S_r = sum exp(-(c-beta_r)/lambda), V_r[2T] = sum w*eps)
 *                 written as 2T+2 float32 to the buffer B200MPPI_BUF_PARTIAL (device).
 *   solve_finish: combine the world_size gathered partials (device pointer, world_size x (2T+2)
 *                 float32, e.g. the output of an NCCL all-gather) into the new u_cur and this
 *                 rank's normalised weights; u_out (host, may be NULL) receives u_cur. */
int b200mppi_planner_solve_local(b200mppi_planner* pl, int32_t first_iteration);
int b200mppi_planner_solve_finish(b200mppi_planner* pl, const float* gathered_partials_dev,
                                  float* u_out);
/* Peer-memory exchange (NVLink / NVSwitch): the same sharded solve with this library's own kernels doing
 * both exchanges -- plain stores into the peers' buffers + epoch flags -- instead of two collective calls
 * of a communication library.  world_size <= 16, all ranks on one node with peer access.
 *   p2p_export        : allocates this planner's exchange buffer and returns its CUDA IPC handle (64 bytes).
 *   p2p_import        : `handles` = the world_size exported handles in rank order (the caller all-gathers them
 *                       once, with any transport); opens the peers' buffers.
 *   p2p_connect_local : same for planners living in THIS process (peers[s] = rank s; devices may differ).
 *   p2p_push          : after solve_local (MODE_TDM): block d of the staged costs -> rank d, then signal.  A no-op
 *                       when the windowed rollout kernel ran: with peers connected it stores every cost straight
 *                       into the receive buffer of the rank that reduces it and raises the flags itself (the
 *                       all-to-all is the rollout kernel's epilogue).
 *   p2p_reduce        : wait for every rank's block, CVaR + softmax partial (as solve_reduce), store the
 *                       partial into every rank's gather buffer, signal.
 *   p2p_finish        : wait for every rank's partial, combine (as solve_finish); u_out may be NULL.
 *   solve_p2p         : num_opt x (solve_local, p2p_push, p2p_reduce, p2p_finish) -- the whole sharded solve()
 *                       in one call, no host synchronisation until the final copy of u.
 * A rank that never arrives does not hang the device: the waits give up after B200MPPI_P2P_TIMEOUT_MS
 * (environment, default 20000) and the call returns B200MPPI_ECUDA naming the missing rank. */
int b200mppi_planner_p2p_export(b200mppi_planner* pl, void* ipc_handle_out, size_t bytes);
int b200mppi_planner_p2p_import(b200mppi_planner* pl, const void* ipc_handles, size_t bytes);
int b200mppi_planner_p2p_connect_local(b200mppi_planner* pl, b200mppi_planner* const* peers, int32_t count);
int b200mppi_planner_p2p_push(b200mppi_planner* pl);
int b200mppi_planner_p2p_reduce(b200mppi_planner* pl);
int b200mppi_planner_p2p_finish(b200mppi_planner* pl, float* u_out);
int b200mppi_planner_solve_p2p(b200mppi_planner* pl, float* u_out);

/* Host-side reference combine of gathered partials (used by CPU tests of the N>1 logic; tiny). */
int b200mppi_combine_partials_host(const float* gathered, int32_t world_size, int32_t num_steps,
                                   float lambda_weight, const float* u_in, const float vrange[2],
                                   const float wrange[2], float* u_out);

/* ---- stage-level entry points (parity tests drive the kernels one at a time, like replaying the
 *      body of solve_* kernel by kernel; SURVEY.md 8c-iii) */
int b200mppi_planner_sample_noise(b200mppi_planner* pl);                 /* sample_noise_numba */
int b200mppi_planner_set_noise(b200mppi_planner* pl, const float* noise, size_t bytes);
/* rollout_* kernel + CVaR with the CURRENT noise, u_cur and TDM sample buffers. */
int b200mppi_planner_rollout(b200mppi_planner* pl);
/* only the CVaR reduction over M (mppi.py:718-755) on the CURRENT per-(n,m) cost buffer. */
int b200mppi_planner_cvar(b200mppi_planner* pl);
/* update_useq_numba on the current costs (or on `costs` if not NULL, N_local float32). */
int b200mppi_planner_update(b200mppi_planner* pl, const float* costs);
/* get_state_rollout (mppi.py:545-608): float32 (V, T+1, 3). */
int b200mppi_planner_get_state_rollout(b200mppi_planner* pl, float* out, size_t bytes);

enum {
  B200MPPI_BUF_NOISE = 0,     /* float32 (N_roll, T, 2)    noise_samples_d (N_roll = N when maps are sharded) */
  B200MPPI_BUF_U_CUR = 1,     /* float32 (T, 2)            u_cur_d                    */
  B200MPPI_BUF_COSTS = 2,     /* float32 (N_local)         costs_d (NOT clobbered)    */
  B200MPPI_BUF_WEIGHTS = 3,   /* float32 (N_local)         weights_d (normalised)     */
  B200MPPI_BUF_COSTS_NM = 4,  /* float32 per-(n,m) costs, MODE_TDM.  copy_out / copy_in: the logical (N_local, M_local)
                               * array [n][m].  Device buffer (planner_buffer): MAP-MAJOR (M, N) -- row m = all control
                               * sequences on sampled map m -- and for a map-sharded planner (ws, M/ws, N/ws) blocks by
                               * destination rank (see solve_local); not written when the rollout kernel stores
                               * straight into the peers (p2p_push) */
  B200MPPI_BUF_RNG = 5,       /* uint64  (N_local*T, 2)    rng_states_d               */
  B200MPPI_BUF_PARTIAL = 6,   /* float32 (2T+2)            this rank's softmax partial*/
  B200MPPI_BUF_U_PREV = 7,    /* float32 (T, 2)            u_prev_d                   */
  B200MPPI_BUF_STATE_ROLLOUT = 8 /* float32 (V, T+1, 3)    state_rollout_batch_d      */
};
int b200mppi_planner_buffer(b200mppi_planner* pl, int32_t buffer_id, void** dev_ptr,
                            size_t* bytes);
int b200mppi_planner_copy_out(b200mppi_planner* pl, int32_t buffer_id, void* dst, size_t bytes);
int b200mppi_planner_copy_in(b200mppi_planner* pl, int32_t buffer_id, const void* src,
                             size_t bytes);
int b200mppi_planner_synchronize(b200mppi_planner* pl);

/* Test hook (host only, no GPU needed): the sampler's threshold lookup q(draw) for raw 64-bit xoroshiro draws --
 * the same inline function and tables the kernel uses (terrain.py:682-684 restated as an integer table, see
 * csrc/common.cuh::sample_threshold_q).  q_cap = the smallest column total of the PMF (100 for a proper PMF).
 * B200MPPI_ESTATE if alpha_dyn is not representable (the sampler then uses its generic kernel). */
int b200mppi_debug_sample_threshold(double alpha_dyn, int32_t q_cap, const uint64_t* draws, int64_t n,
                                    uint8_t* q_out);

/* Debug hook: per-CTA start / end times (ns) and chunk shares of the windowed rollout kernel's launches that follow
 * (enable != 0), read back into out[6 * ctas]: start, end, share lo / hi (SM id in bits 40+ of lo), lane-steps on the slow
 * path, of which outside the staged window (bits 40+: warp-steps run) (tools/rollout_cta_times.py). */
int b200mppi_debug_rollout_cta_times(int32_t enable, int64_t* out, int32_t ctas);

/* Tracing: CUDA-event time of each stage of the last solve/solve_local+finish, milliseconds.
 * Enabled with b200mppi_planner_set_profiling(pl, 1) (adds event records, no syncs). */
enum {
  B200MPPI_T_SAMPLE_GRIDS = 0, B200MPPI_T_NOISE = 1, B200MPPI_T_ROLLOUT = 2, B200MPPI_T_CVAR = 3,
  B200MPPI_T_UPDATE = 4, B200MPPI_T_TOTAL = 5, B200MPPI_T_COUNT = 6
};
int b200mppi_planner_set_profiling(b200mppi_planner* pl, int32_t enable);
int b200mppi_planner_last_timings(b200mppi_planner* pl, float* ms_out /* [B200MPPI_T_COUNT] */);
/* Kernel launches issued by this handle since creation (bench.py's gpu_launches). */
int b200mppi_planner_launch_count(b200mppi_planner* pl, int64_t* out);
/* Reach-box map sampling (MODE_TDM solves only; the reference samples whole maps on every solve,
 * terrain.py:610-694 called from mppi.py:404-405).  A solve samples only the cells its rollouts can read -- the
 * box |x - x0| <= dt * max|traction| * S around the robot, S = sum_t |v_t| bounded by T * max|vrange| ("static")
 * or by the max over this solve's own N clipped control sequences ("dynamic", one 4-byte read-back per solve) --
 * and advances every generator by the draws of a whole-map walk (GF(2) jump), so costs, u and every RNG state are
 * those of whole-map sampling.  Readers of the sampled maps outside solve() (get_sample_grids, sample_grid_view,
 * get_state_rollout, planner_rollout) first complete the maps from the pre-solve states.  Whole maps are sampled
 * whenever the bound is not airtight (box not strictly inside the map, ill-formed PMF, generic rollout kernel).
 * Environment: B200MPPI_SAMPLE_BOX = off | static | dynamic (default).
 * out[5] = { mode used by the last solve (0 whole maps, 1 static, 2 dynamic), row_lo, row_hi, col_lo, col_hi }. */
int b200mppi_planner_sample_box(b200mppi_planner* pl, int32_t out[5]);

/* ------------------------------------------------------------------ batched one-map solves
 * K independent planners of the same shape solved with ONE launch per stage for the whole batch (noise, map sampling,
 * rollout, update; plus one descriptor upload and one D2H of all K control sequences), instead of K solve() calls of
 * four small launches, two copies and a host synchronisation each.  The planners are BORROWED (they must outlive the
 * batch) and keep every per-planner call (set_params, set_u, shift_u, copy_out, get_state_rollout, ...).
 *   create: planners on one device, world_size 1, one mode among MODE_DET_DYN / MODE_SPEED_MAP / MODE_BAREBONE (the
 *           stochastic MODE_TDM is not batched: its windowed rollout kernel already fills the GPU), equal num_steps and
 *           num_control_rollouts, no planner listed twice.  Anything else: B200MPPI_EINVAL naming the planner's index.
 *   solve : == b200mppi_planner_solve on planners[0], planners[1], ... in that order, bit for bit: u, u_prev, noise,
 *           costs, weights, the planners' and their TDMs' RNG states and the sampled maps all end up identical.  Needs
 *           equal params.num_opt and no TDM shared between two planners of the batch (B200MPPI_EINVAL; a planner whose
 *           lin == ang is fine); every planner must be ready to solve (the first that is not is reported with its
 *           index).  Rejections are decided before any work is issued.  The batch's work starts after all work already
 *           issued on the members' streams and has finished when the call returns.  Pairs of TDMs whose maps cannot
 *           be sampled with the batch's one sampler launch (other map geometry, ill-formed PMF, ...) are sampled by
 *           their own launches -- same results, more launches.
 *           u_out: float32 (count, T, 2), may be NULL.
 *   launch_count: kernel launches issued by this batch (per-planner launch counts and stage timings are not touched). */
typedef struct b200mppi_batch b200mppi_batch;
int b200mppi_batch_create(b200mppi_planner* const* planners, int32_t count, b200mppi_batch** out);
int b200mppi_batch_destroy(b200mppi_batch* b);
int b200mppi_batch_set_stream(b200mppi_batch* b, void* cuda_stream);
int b200mppi_batch_solve(b200mppi_batch* b, float* u_out);
int b200mppi_batch_launch_count(b200mppi_batch* b, int64_t* out);

#ifdef __cplusplus
}
#endif
#endif /* B200MPPI_H */
