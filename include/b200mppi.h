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

/* ------------------------------------------------------------------ ground-truth realisations on the device
 * The reference's real-world evaluation (confidence_score_example_vis.ipynb) drives the plant on realisations of a
 * ground-truth TDM pair: its sample_traction_grid(lin, ang) calls lin.sample_grids(), copies map 0 to the host and
 * converts it with q * (hi - lo) / 100.0 + lo, then does the same for ang, and wraps both in a TractionGrid on lin's
 * padded limits and resolution.  A realisation set holds such grids in device memory, where trial calls read them in
 * place (b200mppi_trial_desc).
 *   draw_realisations: realisation i is what the helper's i-th call returns: b200mppi_tdm_sample_grids(lin, 1.0), then
 *           b200mppi_tdm_sample_grids(ang, 1.0) (the same sampling path), map 0 of each converted into the set.  lin ==
 *           ang is allowed and follows that order (the lin plane from the first sampling, the ang plane from the
 *           second).  Afterwards both TDMs are exactly as after those 2 * count calls: generator states and sampled
 *           maps.  Each plane is float64 (height, width) = (max_map_rows, max_map_cols) row-major on the TDMs' device
 *           -- the whole sample plane, as copy_to_host()[0] -- with each cell float64(((float)q * (hi - lo)) / 100 + lo)
 *           evaluated in float32, every operation rounded to nearest on its own (no flush to zero, no contraction), hi
 *           and lo the bounds of that plane's TDM: what NumPy 2 computes for the helper (float32 bounds keep the result
 *           float32), widened exactly.  One conversion launch per realisation for both planes (two when lin == ang).
 *           Refused: count < 1, a PMF not set (B200MPPI_ESTATE), TDMs on different devices or of different
 *           max_map_dim.
 *   info  : count, height, width, and lin's res and padded limits (as the TDM holds them, float32) and the device.
 *   planes: the device pointers of realisation i's lin and ang planes, for b200mppi_trial_desc.
 *   copy_out: realisation i's planes into host float64 (height, width) arrays.
 * The library keeps a registry of live sets; destroy removes a set from it and frees its memory. */
typedef struct b200mppi_realisations b200mppi_realisations;
int b200mppi_tdm_draw_realisations(b200mppi_tdm* lin, b200mppi_tdm* ang, int32_t count, b200mppi_realisations** out);
int b200mppi_realisations_destroy(b200mppi_realisations* set);
int b200mppi_realisations_info(const b200mppi_realisations* set, int32_t* count, int32_t* height, int32_t* width,
                               double* res, double xlimits[2], double ylimits[2], int32_t* device);
int b200mppi_realisations_planes(const b200mppi_realisations* set, int32_t i, const double** lin, const double** ang);
int b200mppi_realisations_copy_out(const b200mppi_realisations* set, int32_t i, double* lin, double* ang);

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

/* Test hook (needs a GPU): out[i] = op(a[i]) or op(a[i], b[i]) for n host floats, evaluated on the device by the
 * approximate operations the kernels use -- sin.approx / cos.approx / sqrt.approx / div.approx / div.full (.ftz) of
 * csrc/common.cuh and the libdevice logf / cosf of the Box-Muller noise -- so that a host oracle can reproduce every
 * rollout cost and noise value exactly.  b is read only by the two divisions.  B200MPPI_EINVAL for an unknown op,
 * n < 0 or a missing array. */
enum {
  B200MPPI_MATH_SIN_APPROX = 0, B200MPPI_MATH_COS_APPROX = 1, B200MPPI_MATH_SQRT_APPROX = 2,
  B200MPPI_MATH_DIV_APPROX = 3, B200MPPI_MATH_DIV_FULL = 4, B200MPPI_MATH_LOGF = 5, B200MPPI_MATH_COSF = 6
};
int b200mppi_debug_device_math(int32_t op, const float* a, const float* b, float* out, int64_t n);

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
 * Window-first (the default): a single-rank solve() of one iteration with the windowed rollout samples only the
 * window the rollout kernel stages around the robot plus a ring of 8 cells, with no host wait; the rollout flags the
 * maps whose rollouts read outside that rectangle, and two launches gated on the flags complete those maps from the
 * pre-solve states and rerun their rollouts, so results are again those of whole-map sampling.  sample_box() then
 * reports the reach box the solve would have sampled (decided on the device, copied back with u).  Sharded solves,
 * num_opt != 1, batches and trials sample their reach box.
 * Environment: B200MPPI_SAMPLE_BOX = off | static | dynamic | window (unset: window; any other value: dynamic).
 * out[5] = { mode used by the last solve (0 whole maps, 1 static, 2 dynamic), row_lo, row_hi, col_lo, col_hi }. */
int b200mppi_planner_sample_box(b200mppi_planner* pl, int32_t out[5]);
/* Window-first sampling of the last solve(): out[6] = { 1 if it sampled window-first (else 0 and zeros), row_lo,
 * row_hi, col_lo, col_hi of the rectangle sampled up front, number of maps whose rollouts read outside it (completed
 * and rerun) }. */
int b200mppi_planner_sample_window(b200mppi_planner* pl, int32_t out[6]);

/* ------------------------------------------------------------------ batched one-map solves
 * K independent planners of the same shape solved with ONE launch per stage for the whole batch (noise, map sampling,
 * rollout, update; plus one descriptor upload and one D2H of all K control sequences), instead of K solve() calls of
 * four small launches, two copies and a host synchronisation each.  The planners are BORROWED (they must outlive the
 * batch) and keep every per-planner call (set_params, set_u, shift_u, copy_out, get_state_rollout, ...).
 *   create: planners on one device, world_size 1, one mode among MODE_DET_DYN / MODE_SPEED_MAP / MODE_BAREBONE
 *           (MODE_TDM planners: b200mppi_batch_create_stochastic below), equal num_steps and
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

/* ------------------------------------------------------------------ batched stochastic solves
 * K independent MODE_TDM (CVaR-cost) planners of one shape solved together: per optimisation iteration ONE launch each
 * of noise + controls, windowed rollout (all K*M (planner, map) units on the persistent grid), CVaR and update.  The map
 * sampling of the first iteration stays per planner (each planner's reach box is its own: 1 or 2 launches each), with
 * one host wait for all K reach statistics.  The result is a b200mppi_batch: batch_solve, set_stream, launch_count and
 * destroy work on it as above; b200mppi_batch_run_trials refuses it (b200mppi_batch_run_stochastic_trials below runs
 * its closed-loop trials).
 *   create: planners on one device, MODE_TDM, world_size 1, equal num_steps, num_control_rollouts and
 *           num_grid_samples (any M a MODE_TDM planner takes, up to 16384), no planner listed twice.  Anything else:
 *           B200MPPI_EINVAL naming the planner.
 *   solve : == b200mppi_planner_solve on planners[0], planners[1], ... in that order, bit for bit: u, noise, per-(m, n)
 *           costs, costs, weights, the planners' and their TDMs' RNG states, the sampled maps (boxed or whole), the
 *           reach-box decisions (b200mppi_planner_sample_box) and the host-side solve state.  Refused before any work is
 *           issued (B200MPPI_EINVAL or the planner's own error, naming the planner): what batch_solve refuses, and a
 *           planner that would not take the windowed rollout kernel (B200MPPI_NO_WINDOW, a window that does not fit,
 *           tensor maps that cannot be encoded).  u_prev is not touched (a stochastic solve does not alias it). */
int b200mppi_batch_create_stochastic(b200mppi_planner* const* planners, int32_t count, b200mppi_batch** out);

/* ------------------------------------------------------------------ planners sharing TDM pairs
 * b200mppi_batch_share_tdms(b, 1) lets planners of a one-map or stochastic batch share a lin/ang TDM pair (many robots
 * on one map, or one environment solved at several cvar_alpha): each shared pair is sampled ONCE per call instead of
 * once per planner.  Off (the default, enable = 0) the batch behaves exactly as described above.  Barebone batches
 * have no TDMs and accept the call as a no-op.  It applies to batch_solve and to every trial call.
 *   groups: planners with the same (lin, ang) objects form one group.  Refused before any work (B200MPPI_EINVAL, naming
 *           both planners): a TDM that is lin of one planner and ang of another, two planners sharing lin but not ang,
 *           and, in a stochastic batch, members of one group with unequal params.alpha_dyn.
 *   solve : each group's pair is sampled once, in the first iteration after the noise launch.  Afterwards every planner
 *           is byte for byte as after its own b200mppi_planner_solve on a PRIVATE copy of its pair taken before the call
 *           (same PMF, masks, risk map and generator states): u (and the u_prev alias of one-map planners), noise,
 *           per-(m, n) and CVaR costs, weights and its RNG streams.  The shared TDMs end with the generator states of
 *           every copy, and their completed maps equal every copy's.  This is not "K solves in order": sequential
 *           solves would sample a shared pair K times.
 *   box   : a stochastic group samples one box.  One member: exactly its own reach-box decision, disc included.  Two or
 *           more: the rectangle hull of the members' boxes without a disc, or whole maps if any member decides whole
 *           maps or the hull's sampler launch does not fit; the mode is the largest of the members'.
 *           b200mppi_planner_sample_box of every member reports the box its group sampled -- the one piece of planner
 *           state that may differ from the private copy's.
 *   trials: a group's pair is sampled once per step while any member runs and not at all once every member has
 *           stopped.  Every planner ends as after its own episode on a private copy (planner state as above, histories,
 *           steps, status, logs and records); the shared TDMs end as the copy of the group's longest-running member.
 *           sample_box is the box of the planner's own last step.
 *   A planner alone in its group behaves exactly as without sharing, sample_box included. */
int b200mppi_batch_share_tdms(b200mppi_batch* b, int32_t enable);

/* ------------------------------------------------------------------ visualisation rollouts of a batch
 * b200mppi_planner_get_state_rollout of every planner of a batch (either kind) with ONE launch: for MODE_TDM planners
 * u_cur over the first V sampled maps, for the others u_cur and V-1 clipped u_prev + noise rollouts (MODE_BAREBONE
 * without a map).  MODE_TDM planners whose last sampling was boxed first get their maps completed, as the single call
 * does.  Each planner's own state-rollout buffer (B200MPPI_BUF_STATE_ROLLOUT) is written, then copied into out with one
 * synchronisation: afterwards every planner is exactly as after get_state_rollout on planners[0], planners[1], ... in
 * that order, bit for bit (per-planner launch counts are not touched; the batch's count grows by one).
 *   out: float32 (count, V, T+1, 3), bytes its size.
 * Refused (B200MPPI_EINVAL or the planner's own error, naming the planner) before any work is issued: a planner that is
 * not ready (params not set, ...), unequal num_vis_state_rollouts, and V larger than a planner's M (MODE_TDM) or N. */
int b200mppi_batch_get_state_rollout(b200mppi_batch* b, float* out, size_t bytes);

/* ------------------------------------------------------------------ closed-loop trials of a batch
 * Every planner of a MODE_DET_DYN or MODE_SPEED_MAP batch drives a unicycle through one receding-horizon episode on
 * its own ground-truth traction grid, entirely on the device: per step ONE launch each of noise, rollout and update for
 * the whole batch (num_opt > 1 repeats them) and one map-sampling launch per launch class, then the plant step:
 * 3*num_opt + 1 + C launches for C classes.  The planners' maps may differ in size, resolution and bin count; a launch
 * class holds the TDM pairs that share the padded bin count of both TDMs, the thread tile and the number of maps, so a
 * batch on one map geometry is one class (5 launches at num_opt = 1).
 * The plant step is the benchmark loop's: u = u_cur[0]; (lt, at) = grid value of the cell holding (x, y), (0, 0)
 * outside the grid; x += dt*lt*cos(theta)*v, y += dt*lt*sin(theta)*v, theta += dt*at*w in float64; u_cur shifted by
 * one (the last row kept); d = |(x, y) - xgoal| - goal_tolerance, cum_obj += dt + d, cum_dist_to_goal += d.  A planner
 * stops once d <= 0 (GOAL), once its pose leaves the padded map limits (LEFT_MAP: its next solve would be refused) or
 * after max_steps steps (MAX_STEPS).  Stopped planners' CTAs return at once; the host polls the count of running
 * planners every few steps and issues nothing more once it is zero.
 * Afterwards every planner, its TDMs (RNG states, sampled maps) and its params are exactly as `steps` rounds of
 * solve() -> plant step -> set_u(shifted u) -> set_params(x0 = float32(new pose)) would leave them, except that the
 * C-side params keep the x0 of the last solve (as in that loop, where the new pose is uploaded by the next solve).
 * Refused (B200MPPI_EINVAL naming the planner) before any work is issued: what batch_solve refuses, MODE_BAREBONE,
 * max_steps < 1, num_opt < 1, a grid or limit that is not usable, a start pose outside the padded limits, and a TDM
 * pair that the batched sampler cannot take (diverged lin / ang streams, a PMF the staged sampler cannot take).
 *   trials  : count descriptors, in planner order; the grids are uploaded and freed by the call.
 *   xhist   : float64 (count, max_steps+1, 3), NaN after a planner's last step;  uhist: float32 (count, max_steps, 2),
 *             NaN after it;  results: count records;  steps_issued (may be NULL): steps the batch issued. */
enum { B200MPPI_TRIAL_GOAL = 1, B200MPPI_TRIAL_MAX_STEPS = 2, B200MPPI_TRIAL_LEFT_MAP = 3,
       B200MPPI_TRIAL_NOT_RUN = 4 /* an episode of a trial sequence that never started */ };
/* Grids: lin and ang are host arrays, uploaded by the call, or both the planes of one realisation of a live
 * b200mppi_realisations set on the batch's device (b200mppi_realisations_planes), which the call reads in place: no copy
 * and no device grid section for that slot; height and width must be the set's.  Both kinds may be mixed in one call.
 * The call checks every pointer with cudaPointerGetAttributes and the set registry before any work: device memory that
 * is not the start of a plane of a live set (another allocation, a destroyed set, the middle of a plane), a set on
 * another device, lin and ang from different sets or of different kinds are refused (B200MPPI_EINVAL naming the planner
 * and, for sequences, the episode).  The grid's position and resolution are the descriptor's (xlo, ylo, res), as for
 * host grids. */
typedef struct {
  const double* lin;            /* ground-truth linear traction, (height, width) row-major: host, or a realisation plane */
  const double* ang;            /* ground-truth angular traction, same shape and kind */
  int32_t height, width;
  double xlo, ylo, res;         /* the grid's xlimits[0], ylimits[0] and cell size: cell = floor((x - xlo) / res) */
  double x0[3];                 /* start pose */
  double xgoal[2];
  double goal_tolerance, v_post_rollout, dt;
  double pxlim[2], pylim[2];    /* the planner's padded map limits */
} b200mppi_trial_desc;
typedef struct {
  double cum_obj;               /* sum over steps of dt + d (the caller adds the benchmark's d / v_post_rollout tail) */
  double cum_dist_to_goal;      /* sum over steps of d */
  double dist_to_goal;          /* d of the last step */
  int32_t steps, status;        /* steps run, B200MPPI_TRIAL_* */
} b200mppi_trial_result;
int b200mppi_batch_run_trials(b200mppi_batch* b, const b200mppi_trial_desc* trials, int32_t max_steps, double* xhist,
                              float* uhist, b200mppi_trial_result* results, int32_t* steps_issued);

/* ------------------------------------------------------------------ closed-loop trials of a stochastic batch
 * The same episodes, plant step, stop rules, descriptors and results as b200mppi_batch_run_trials, for a batch made by
 * b200mppi_batch_create_stochastic (MODE_TDM, CVaR cost).  Each planner's map-sampling reach box is decided on the device
 * by the function the host-side solve uses, from the pose the plant step wrote and the reach of the controls just drawn,
 * so no step waits for the host.  Per step 4*num_opt + 1 + 2*C launches for the whole batch and C launch classes (as in
 * b200mppi_batch_run_trials; 7 at num_opt = 1 on one map geometry): num_opt x (noise + controls, windowed rollout, CVaR,
 * update), per class one boxed map sampling of its pairs and one state advance of its pairs, and the plant step, which
 * also moves each planner's rollout window.
 * Afterwards every planner is exactly as `steps` rounds of batch_solve (b200mppi_batch_solve on this batch) -> plant step
 * -> set_u(shifted u) -> set_params(x0 = float32(new pose)) would leave it, bit for bit: u, noise, per-(m, n) costs,
 * costs, weights, the planners' and their TDMs' RNG states, the sampled maps, b200mppi_planner_sample_box and the host-side
 * solve state; the C-side params keep the x0 of the last solve.
 * Refused (B200MPPI_EINVAL naming the planner) before any work is issued: what b200mppi_batch_run_trials and the
 * stochastic batch_solve refuse, and a TDM pair that the batched sampler cannot take (lin == ang, diverged lin / ang
 * streams, a PMF the staged sampler cannot take at the planner's alpha_dyn), or a launch class whose boxed sampler
 * launch does not fit a CTA (naming its first planner).  A batch made by
 * b200mppi_batch_create is refused, naming planner 0's mode. */
int b200mppi_batch_run_stochastic_trials(b200mppi_batch* b, const b200mppi_trial_desc* trials, int32_t max_steps,
                                         double* xhist, float* uhist, b200mppi_trial_result* results,
                                         int32_t* steps_issued);

/* ------------------------------------------------------------------ closed-loop trials of a barebone batch
 * The episodes of the barebone notebook's closed loop for a MODE_BAREBONE batch made by b200mppi_batch_create, entirely
 * on the device: per step 3*num_opt + 1 launches for the whole batch, num_opt x (noise, rollout, update), then the
 * plant step.  The plant step is the notebook's nominal unicycle in float64: u = u_cur[0]; x += dt*cos(theta)*v,
 * y += dt*sin(theta)*v, theta += dt*w; u_cur shifted by one (the last row kept); d = |(x, y) - xgoal| - goal_tolerance,
 * cum_obj += dt + d, cum_dist_to_goal += d.  A planner stops once d <= 0 (GOAL) or after max_steps steps (MAX_STEPS);
 * there is no map to leave.  Every new pose is checked against the planner's obstacles (b200mppi_planner_set_obstacles):
 * it touches obstacle (ox, oy, r) when (x - ox)^2 + (y - oy)^2 <= r^2 in float64 (each operation rounded on its own),
 * the rollout's rule, and contact_steps[k] counts the steps whose new pose touches at least one.  An episode does not
 * stop on contact.  Polling, stop gating and the state left behind are those of b200mppi_batch_run_trials: every
 * planner is exactly as `steps` rounds of batch_solve -> plant step -> set_u(shifted u) -> set_params(x0 = float32(new
 * pose)) would leave it, and the C-side params keep the x0 of the last solve.
 *   trials       : count descriptors; the call reads x0, xgoal, goal_tolerance and dt.  lin and ang must be NULL; the
 *                  grid fields, the padded limits and v_post_rollout are ignored.
 *   contact_steps: int32 (count).  xhist, uhist, results and steps_issued as in b200mppi_batch_run_trials.
 * Refused (B200MPPI_EINVAL naming the planner) before any work is issued: what batch_solve refuses, a batch that is not
 * MODE_BAREBONE (naming planner 0's mode), max_steps < 1, num_opt < 1, non-NULL grids, a non-finite x0, xgoal or
 * goal_tolerance, and a dt that is not finite and positive.  b200mppi_batch_run_trials and
 * b200mppi_batch_run_stochastic_trials refuse MODE_BAREBONE batches. */
int b200mppi_batch_run_barebone_trials(b200mppi_batch* b, const b200mppi_trial_desc* trials, int32_t max_steps,
                                       double* xhist, float* uhist, b200mppi_trial_result* results,
                                       int32_t* contact_steps, int32_t* steps_issued);

/* ------------------------------------------------------------------ closed-loop trials with visualisation records
 * One of the trial calls above (kind: B200MPPI_TRIALS_MAP = b200mppi_batch_run_trials, _STOCHASTIC =
 * b200mppi_batch_run_stochastic_trials, _BAREBONE = b200mppi_batch_run_barebone_trials, _MIXED =
 * b200mppi_batch_run_mixed_trials below; contact_steps as that call takes it, NULL for all but barebone) that also records the visualisation rollouts of every step s with
 * s % record_every == 0, as a host loop calling b200mppi_planner_get_state_rollout after solve() and the plant step and
 * before shift_and_update records them: u_cur and x0 of that step's solve.  Everything else -- episodes, results,
 * histories and the state every planner is left in -- is that call's, bit for bit; in addition each planner's
 * state-rollout buffer holds its last record.
 *   rollouts: float32 (count, R, V, T+1, 3), R = ceil(max_steps / record_every), rollout_bytes its size.  Record r
 *             belongs to step r * record_every; it is NaN when that step is >= the planner's steps.  The records stay
 *             in device memory during the call; at the end each written record is copied into rollouts once, and the
 *             rest are set to NaN on the host.
 * Launches: one more per recorded step (the batched visualisation rollouts, before the plant step), and for a
 * batch holding MODE_TDM planners one more per stochastic launch class: a whole-map sampling of maps [0, V) for every pair whose step sampled a
 * reach box,
 * from that step's pre-call generator states (the maps the rollouts read; no generator state changes, maps >= V keep
 * their box and are completed by any later reader, as after the host loop).
 * Refused (B200MPPI_EINVAL naming the planner) before any work is issued: what the chosen call refuses, an unknown kind,
 * record_every < 1, a NULL rollouts or a wrong rollout_bytes, unequal num_vis_state_rollouts and V larger than a
 * planner's M (MODE_TDM) or N. */
enum { B200MPPI_TRIALS_MAP = 0, B200MPPI_TRIALS_STOCHASTIC = 1, B200MPPI_TRIALS_BAREBONE = 2, B200MPPI_TRIALS_MIXED = 3 };
int b200mppi_batch_run_trials_recorded(b200mppi_batch* b, int32_t kind, const b200mppi_trial_desc* trials,
                                       int32_t max_steps, double* xhist, float* uhist, b200mppi_trial_result* results,
                                       int32_t* contact_steps, int32_t record_every, float* rollouts,
                                       size_t rollout_bytes, int32_t* steps_issued);

/* ------------------------------------------------------------------ trial sequences
 * Several episodes per planner, back to back on the same planners with no reset in between, as the reference benchmark
 * runs trials_per_env ground-truth realisations after one setup().  Planner k runs episodes[k] episodes; episode e uses
 * descriptor trials[first[k] + e], first[k] = episodes[0] + ... + episodes[k-1] (planner-major slots).  Each episode is
 * one episode of b200mppi_batch_run_trials (kind B200MPPI_TRIALS_MAP) or b200mppi_batch_run_stochastic_trials (kind
 * B200MPPI_TRIALS_STOCHASTIC) on its descriptor: its plant starts at the descriptor's x0, with its grid, goal, dt, stop
 * rules and metrics.  Between episodes the planner keeps u_cur, its RNG streams and its TDMs' streams and maps.
 *   reset_x0 = 0: the benchmark's loop.  The first solve of an episode e > 0 plans from the final pose of episode e-1
 *                 (the planner's params x0 is never reset there).  An episode that ends LEFT_MAP ends the sequence (the
 *                 next solve would be refused); its later episodes are B200MPPI_TRIAL_NOT_RUN.
 *   reset_x0 = 1: the first solve of every episode plans from float32 of the episode's x0, as after set_params with
 *                 x0 = start before each episode; every episode runs.
 * The step loop is that of b200mppi_batch_run_trials: the same launches per step, up to max_k episodes[k] * max_steps
 * steps, stopped once every planner's sequence has ended.  An episode boundary costs no launch and no host round trip.
 * Afterwards every planner, its TDMs and its params are as after that host loop of all its run episodes: the reach
 * slots, sample box and the samplings of shared pairs follow its total steps, and the C-side params keep the x0 of the
 * last solve.
 *   kind        : B200MPPI_TRIALS_MAP, B200MPPI_TRIALS_STOCHASTIC or B200MPPI_TRIALS_MIXED, for the batches those
 *                 calls take.
 *   trials      : sum_k episodes[k] descriptors, the grids uploaded and freed by the call.  episodes: int32 (count).
 *   xhist       : float64 (slots, max_steps+1, 3); uhist: float32 (slots, max_steps, 2); results: slots records; NaN
 *                 after an episode's last step and in every row of an episode that never ran, whose record has steps 0
 *                 and status B200MPPI_TRIAL_NOT_RUN.  steps_issued (may be NULL): steps the batch issued.
 * Refused (B200MPPI_EINVAL naming the planner and episode) before any work is issued: what the call of that kind
 * refuses (for every descriptor), another kind, a NULL episodes, an episode count < 1. */
int b200mppi_batch_run_trial_sequences(b200mppi_batch* b, int32_t kind, const b200mppi_trial_desc* trials,
                                       const int32_t* episodes, int32_t max_steps, int32_t reset_x0, double* xhist,
                                       float* uhist, b200mppi_trial_result* results, int32_t* steps_issued);

/* b200mppi_batch_run_trial_sequences with every option: b200mppi_batch_run_trial_sequences_ex(..., contact_steps,
 * record_every, rollouts, rollout_bytes, steps_issued) with contact_steps NULL and record_every 0 is
 * b200mppi_batch_run_trial_sequences for kinds MAP, STOCHASTIC and MIXED: the same launches, buffers and results.
 *   kind          : also B200MPPI_TRIALS_BAREBONE: episodes of b200mppi_batch_run_barebone_trials back to back on a
 *                   MODE_BAREBONE batch, with reset_x0 as above.  Its plant has no map to leave, so every episode runs.
 *   contact_steps : int32 (slots), per episode the steps whose new pose touched an obstacle: required for barebone
 *                   sequences, NULL for the other kinds.
 *   record_every  : 0, or n >= 1: each run episode records at each of its own steps t with t % n == 0 what
 *                   b200mppi_batch_run_trials_recorded records there.  rollouts: float32 (K, Emax, R, V, T+1, 3),
 *                   Emax = max_k episodes[k], R = ceil(max_steps / n), rollout_bytes its size; record r of (k, e)
 *                   belongs to step r n of planner k's episode e, NaN after its last step and everywhere for an
 *                   episode that did not run or that planner k does not have (e >= episodes[k]).  Each planner's
 *                   state_rollout ends with the last record of its last run episode.  Whether a planner records at a
 *                   step is decided on the device, so a recorded sequence issues the record launches (1 + C2, C2 the
 *                   stochastic sampler launch classes) at every step; everything else is as without recording.
 * Refused (B200MPPI_EINVAL) before any work is issued: what b200mppi_batch_run_trial_sequences refuses (bar the
 * barebone kind), record_every < 0, contact_steps missing for barebone or given for another kind, a wrong
 * rollout_bytes, unequal num_vis_state_rollouts when recording.  A record buffer that cannot be allocated:
 * B200MPPI_ECUDA, nothing issued. */
int b200mppi_batch_run_trial_sequences_ex(b200mppi_batch* b, int32_t kind, const b200mppi_trial_desc* trials,
                                          const int32_t* episodes, int32_t max_steps, int32_t reset_x0, double* xhist,
                                          float* uhist, b200mppi_trial_result* results, int32_t* contact_steps,
                                          int32_t record_every, float* rollouts, size_t rollout_bytes,
                                          int32_t* steps_issued);

/* ------------------------------------------------------------------ mixed batches
 * The planners of a method comparison -- MODE_DET_DYN, MODE_SPEED_MAP and MODE_TDM planners on the same environments and
 * realisations -- solved and run through closed-loop trials in ONE batch, with one step loop, one host poll and one
 * grid upload per call instead of one per kind.
 *   create: the one-map planners (MODE_DET_DYN and MODE_SPEED_MAP, in any order) first, then the MODE_TDM planners; one
 *           device, world_size 1, equal num_steps and num_control_rollouts, equal num_grid_samples among the MODE_TDM
 *           planners, no planner listed twice.  MODE_BAREBONE planners (b200mppi_batch_run_barebone_trials), a
 *           one-map planner after a MODE_TDM one and anything batch_create or batch_create_stochastic refuse:
 *           B200MPPI_EINVAL naming the planner.  Messages name planners by their index in this order.
 *   Each planner's results and the state it is left in (u, u_prev, noise, costs, weights, RNG streams, its TDMs'
 *   streams and maps, b200mppi_planner_sample_box, the C-side x0) are, bit for bit, those of the same call on the
 *   batch of its kind: b200mppi_batch_create of the MODE_DET_DYN planners, of the MODE_SPEED_MAP planners, and
 *   b200mppi_batch_create_stochastic of the MODE_TDM planners, with the same b200mppi_batch_share_tdms setting.  A TDM
 *   pair shared by a one-map and a MODE_TDM planner is refused (B200MPPI_EINVAL naming both) before any work.
 *   b200mppi_batch_solve, get_state_rollout, set_stream, launch_count, share_tdms and destroy take a mixed batch;
 *   its trials run through b200mppi_batch_run_mixed_trials, b200mppi_batch_run_trials_recorded and
 *   b200mppi_batch_run_trial_sequences with kind B200MPPI_TRIALS_MIXED.  The other trial calls refuse it, naming
 *   b200mppi_batch_run_mixed_trials, and the mixed calls refuse every other batch.
 *   Launches: a batch of one kind issues exactly the launches of the batch of that kind.  Holding both, a trial step at
 *   num_opt n issues 6 n + 1 + C1 + 2 C2 launches, C1 and C2 the one-map and stochastic sampler launch classes: per
 *   iteration the one-map noise, noise + controls, one-map rollout, windowed rollout, CVaR and ONE update over all
 *   planners; per step the sampler classes and ONE plant step.  A recorded step adds 1 + C2.  A solve issues each
 *   kind's launches and one update per iteration.
 * b200mppi_batch_run_mixed_trials: b200mppi_batch_run_trials / b200mppi_batch_run_stochastic_trials of every planner
 * of a mixed batch in one call, one descriptor per planner in the batch's order, with the same outputs and refusals
 * (those of each planner's kind, a batch that is not mixed). */
int b200mppi_batch_create_mixed(b200mppi_planner* const* planners, int32_t count, b200mppi_batch** out);
int b200mppi_batch_run_mixed_trials(b200mppi_batch* b, const b200mppi_trial_desc* trials, int32_t max_steps,
                                    double* xhist, float* uhist, b200mppi_trial_result* results,
                                    int32_t* steps_issued);

/* ------------------------------------------------------------------ device loops
 * A receding-horizon loop whose plant is the caller's: a simulator, a learned model or the robot's own state estimate in
 * GPU memory.  A loop opened on a batch enqueues each solve and each shift_and_update on the batch's stream
 * (b200mppi_batch_set_stream); they read poses from and write controls to device memory, and no call waits on the host.
 * Per planner the loop is the host loop of the same calls, bit for bit:
 *   b200mppi_loop_solve              == batch_solve of that planner (its trial kind's batch solve);
 *   b200mppi_loop_shift_and_update   == set_u(u_cur shifted by one row, the last row kept) and set_params with x0 =
 *                                      float32 of the pose, as shift_and_update(pose, u, 1) after that solve.
 * The calls may come in any order (two solves, two shifts, a close right after a solve).  One planner: a batch of one.
 * A loop issues what the trial of its kind issues, without the plant step: a solve issues one trial step's launches
 * (num_opt x the solve stages, the sampler classes) and one export; a shift and a stop one launch each.
 * CUDA graphs: the loop counts its solves on the device (the export that ends a solve prepares the next one's sampler
 * parity and reach slots), so no launch depends on how many solves came before.  Solve, shift_and_update and stop may
 * be captured (cudaStreamCaptureModeGlobal included) on the batch's stream and replayed any number of times, mixed
 * with eager calls: each replay is those calls at that point of the loop, bit for bit, reading the arrays captured.
 * Launches count where they are issued from the host: a capture counts once, a replay adds nothing.
 * Task updates: b200mppi_loop_set_goals and (barebone loops) b200mppi_loop_set_obstacles give every running planner a new
 * goal or obstacle set from device memory between solves, one launch each and capturable like the other calls.  Per
 * planner they are set_params with that goal and set_obstacles with that set before its later solves, bit for bit.
 *
 * b200mppi_batch_loop_open: kind as in b200mppi_batch_run_trials_recorded (the batch's own kind).  padded_limits: float64
 * (count, 4) = padded x lo, x hi, y lo, y hi of each planner's map (the limits of the host's solve check; NULL for
 * barebone).  rows: int32 (count), planner i's row in the caller's controls, poses and stop mask (a permutation of
 * 0 .. count-1; NULL: row i).  The batch's descriptors are built from each planner's params as set now.  Refused
 * (B200MPPI_EINVAL naming the planner) before any work: what batch_solve refuses, num_opt < 1, another kind, a NaN limit,
 * bad rows, a loop already open; and what the trial of that kind refuses of the TDM pairs.
 * b200mppi_batch_loop_open_ex: the same with an obstacle capacity O = max(max_obstacles, the largest obstacle count of
 *   the batch's planners) per planner, allocated at open (a barebone loop can always set as many obstacles as it started
 *   with).  max_obstacles outside [0, 2^24], or above 0 for a loop that is not barebone: B200MPPI_EINVAL.  A barebone
 *   loop's rollouts read each planner's obstacles from its slice of the loop's buffer, filled at open with the planner's
 *   current ones.  b200mppi_batch_loop_open is b200mppi_batch_loop_open_ex with max_obstacles 0.
 * b200mppi_loop_obstacle_capacity: O.
 * While a loop is open, every planner and batch call that touches the state of the batch or its planners (solve, set_*,
 * get_u, shift_u, copy_in / copy_out, the stage calls, get_state_rollout, the trial calls, share_tdms, set_stream and
 * destroy) returns B200MPPI_EINVAL.
 * b200mppi_loop_controls: the loop's own (count, T, 2) float32 device buffer, and the batch's stream.
 * b200mppi_loop_solve: one solve of every running planner; row rows[i] of u_dev ((count, T, 2) float32 in device memory
 *   of the batch's device) gets planner i's new u_cur, NaN for a planner that no longer runs.
 * b200mppi_loop_shift_and_update: pose of planner i = row rows[i] of x_dev: 3 contiguous elements of dtype
 *   B200MPPI_POSE_F64 or _F32 (widened exactly), rows row_stride_bytes apart.  Every running planner shifts u_cur by one
 *   row and plans its next solve from float32 of the pose (a stochastic planner's rollout window moves with it).  A pose
 *   outside its padded limits (float64 lo <= v <= hi for x and y; NaN fails), where the host's next solve would be
 *   refused, stops that planner for good with status B200MPPI_TRIAL_LEFT_MAP (not for barebone planners: no map).
 * b200mppi_loop_stop: mask_dev (count) of elem_bytes 4 (int32) or 1 (bool / uint8), indexed by row: a running planner
 *   whose entry is nonzero stops for good (B200MPPI_LOOP_STOPPED).  A stopped planner never runs again, so every running
 *   planner has solved equally often and one sampler parity serves them all.
 * b200mppi_loop_set_goals: goal of planner i = row rows[i] of g_dev: 2 contiguous elements of dtype B200MPPI_POSE_F64 or
 *   _F32 (widened exactly), rows row_stride_bytes apart.  Every running planner's later solves plan toward float32 of
 *   it, as set_params with that goal.  Not checked, as set_params does not check the goal (NaN and inf pass).
 * b200mppi_loop_set_obstacles: barebone loops only.  obs_dev: rows of count (O' <= O) triples [x, y, r], contiguous, of
 *   dtype B200MPPI_POSE_F64 or _F32, rows row_stride_bytes apart (may be NULL when count is 0).  counts_dev: int32 (count)
 *   by row, or NULL for O' each.  Every running planner's later solves take the first counts[rows[i]] triples of its
 *   row as float32, as set_obstacles with that set (0: no obstacles).  A count outside [0, O'], which set_obstacles
 *   refuses, stops that planner for good with status B200MPPI_LOOP_BAD_OBSTACLES; it keeps its last set.
 *   Refused with B200MPPI_EINVAL before any work: a loop that is not barebone, O' > O, a null pointer, a bad dtype,
 *   stride or alignment, an array outside the batch's device.
 * b200mppi_loop_wait_stream: the batch's stream waits (an event, not the host) for the work issued so far on stream.
 *   While the batch's stream captures a graph, B200MPPI_EINVAL unless stream is part of the same capture (an event
 *   recorded outside it would invalidate the capture).
 * b200mppi_loop_active: the device's int32 (count) running flags, in the batch's order.
 * b200mppi_loop_close: waits for the stream, commits and frees the loop (also on an error).  Every planner and TDM pair is
 *   left as after the host loop: the reach slots, sample boxes and the samplings of shared pairs follow each planner's
 *   solves (a pair's group: its longest-running member), and the C-side params keep the x0 of the last solve.
 *   per_planner (may be NULL): count summaries in the batch's order.
 *   While the batch's stream captures a graph: B200MPPI_EINVAL before any work, the loop left open and usable (close
 *   waits for the stream).  More than 2^31 - 1 solves issued: B200MPPI_ESTATE, the loop freed and the planners' counts
 *   not committed.  Any other error: the loop is freed.
 * b200mppi_loop_close_ex: b200mppi_loop_close that also commits the task updates and returns them per planner in the
 *   batch's order (tasks, obstacles: may be NULL).  A planner that took a goal keeps its float32 in the C-side params; one
 *   that took an obstacle set keeps that set (float32) as its own obstacles, the buffer grown if needed.  tasks[i]: what
 *   planner i took; obstacles: (count, O, 3) float64, planner i's last set in its first tasks[i].num_obstacles triples.
 *   A planner that never took a call is left as it was. */
typedef struct b200mppi_loop b200mppi_loop;
enum { B200MPPI_POSE_F64 = 0, B200MPPI_POSE_F32 = 1 };
enum { B200MPPI_LOOP_RUNNING = 0, B200MPPI_LOOP_STOPPED = 5, B200MPPI_LOOP_BAD_OBSTACLES = 6 };   /* and B200MPPI_TRIAL_LEFT_MAP */
typedef struct {
  int32_t solves, shifts;       /* solves and shifts the planner took */
  int32_t status;               /* B200MPPI_LOOP_RUNNING, B200MPPI_TRIAL_LEFT_MAP, B200MPPI_LOOP_STOPPED or
                                   B200MPPI_LOOP_BAD_OBSTACLES */
  int32_t pad_;
  double x[3];                  /* the last pose shift_and_update took (the params' x0 before the loop: shifts 0) */
} b200mppi_loop_summary;
typedef struct {
  int32_t took_goal;            /* 1: the planner took a goal (b200mppi_loop_set_goals) */
  int32_t took_obstacles;       /* 1: it took an obstacle set (b200mppi_loop_set_obstacles) */
  int32_t num_obstacles;        /* the count of the last set it took */
  int32_t pad_;
  double goal[2];               /* the last goal it took, float64 (a float32 goal widened) */
} b200mppi_loop_task;
int b200mppi_batch_loop_open(b200mppi_batch* b, int32_t kind, const double* padded_limits, const int32_t* rows,
                             b200mppi_loop** out);
int b200mppi_batch_loop_open_ex(b200mppi_batch* b, int32_t kind, const double* padded_limits, const int32_t* rows,
                                int32_t max_obstacles, b200mppi_loop** out);
int b200mppi_loop_obstacle_capacity(b200mppi_loop* loop, int32_t* capacity);
int b200mppi_loop_controls(b200mppi_loop* loop, float** u_dev, void** stream);
int b200mppi_loop_solve(b200mppi_loop* loop, float* u_dev);
int b200mppi_loop_shift_and_update(b200mppi_loop* loop, const void* x_dev, int32_t dtype, int64_t row_stride_bytes);
int b200mppi_loop_stop(b200mppi_loop* loop, const void* mask_dev, int32_t elem_bytes);
int b200mppi_loop_set_goals(b200mppi_loop* loop, const void* g_dev, int32_t dtype, int64_t row_stride_bytes);
int b200mppi_loop_set_obstacles(b200mppi_loop* loop, const void* obs_dev, int32_t dtype, int32_t count,
                                int64_t row_stride_bytes, const int32_t* counts_dev);
int b200mppi_loop_wait_stream(b200mppi_loop* loop, void* stream);
int b200mppi_loop_active(b200mppi_loop* loop, const int32_t** dev);
int b200mppi_loop_close(b200mppi_loop* loop, b200mppi_loop_summary* per_planner);
int b200mppi_loop_close_ex(b200mppi_loop* loop, b200mppi_loop_summary* per_planner, b200mppi_loop_task* tasks,
                           double* obstacles);

#ifdef __cplusplus
}
#endif
#endif /* B200MPPI_H */
