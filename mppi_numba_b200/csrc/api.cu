// api.cu -- the C-ABI of include/b200mppi.h: handles, device buffers, and the per-solve launch
// sequence that replaces the bodies of MPPI_Numba.solve_* (mppi_numba/mppi.py:237-451) and
// TDM_Numba.sample_grids (terrain.py:610-622).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b200mppi.h"
#include "kernels.h"

using namespace b200;

// --------------------------------------------------------------------------------------------- errors
static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
#define CU(call)                                                                          \
  do {                                                                                    \
    cudaError_t e__ = (call);                                                             \
    if (e__ != cudaSuccess)                                                               \
      return fail(B200MPPI_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e__));   \
  } while (0)
#define CHECK_LAUNCH() CU(cudaGetLastError())

extern "C" const char* b200mppi_last_error(void) { return g_err.c_str(); }
extern "C" int b200mppi_version(void) { return B200MPPI_VERSION; }
extern "C" int b200mppi_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

static inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

// --------------------------------------------------------------------------------------------- TDM
struct b200mppi_tdm {
  b200mppi_config cfg{};
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  bool det_dyn = false;
  int num_maps = 1;           // M or 1
  int pitch = 0;              // bytes per sample-grid row
  int8_t* grid = nullptr;     // (num_maps, Rmax, pitch)
  uint64_t* states = nullptr; // (num_gen, 2)  current generator states
  uint64_t* states_alt = nullptr;   // double buffer for the segmented sampler
  uint64_t* jump_d = nullptr;       // jump-ahead matrices of the current tile geometry
  uint64_t* jump_tile_d = nullptr;  // [4][128][2]: whole-tile advance per tile class (sample_tile_draws)
  uint64_t* jump_box_d = nullptr;   // segment jumps of a boxed launch (finer row segments: fewer tile rows to spread)
  int box_segs = 1, box_seg_rows = 1;
  int jump_segs = 0, jump_seg_rows = 0, jump_rows = 0, jump_cols = 0;
  // reach-box sampling (solve() only): the sampled maps hold fresh values inside the box of the last solve and
  // stale ones outside; states_alt still holds the pre-solve generator states, so the whole maps of that very
  // sampling call can be produced on demand (tdm_complete_grid) -- every reader of `grid` outside solve() does
  bool grid_partial = false;
  double partial_alpha = 1.0;
  float tr_abs_max = 0.0f;          // max |traction| a sampled byte can decode to: max_b |lo + 0.01*(hi-lo)*q_b|
  int64_t num_gen = 0;
  // map
  bool pmf_set = false, masks_set = false, risk_set = false;
  int B = 0, bpad = 0, rows = 0, cols = 0;
  int8_t* pmf = nullptr; int8_t* cum = nullptr; int8_t* qvals = nullptr;
  size_t pmf_cap = 0, cum_cap = 0;
  float bounds[2] = {0, 1};
  float res = 1, pxl[2] = {0, 0}, pyl[2] = {0, 0};
  int8_t* obstacle = nullptr; int8_t* unknown = nullptr; int8_t* risk = nullptr;
  bool masks01 = true;            // every obstacle / unknown byte is 0 or 1 (b200mppi_tdm_set_masks checks the host arrays)
  size_t mask_cap = 0, risk_cap = 0;
  int mask_rows = 0, mask_cols = 0, mask_pitch = 0;
  // fast sampler eligibility (sample.cu v2): entries in [0,127], monotone sums <= 127
  bool pmf_valid = false;
  int min_total = 0;            // smallest column total (q above it would leave a cell unwritten)
  uint64_t* thr_d = nullptr;    // device copy of the q(v) breakpoints for thr_alpha
  double thr_alpha = -1.0;
  bool thr_ok = false;
  uint64_t sig = 0;             // identifies the generator-state history (equal sig <=> equal states)
};

static inline uint64_t mix_sig(uint64_t h, uint64_t v) {
  h ^= v + 0x9E3779B97F4A7C15ULL + (h << 6) + (h >> 2);
  h *= 0xBF58476D1CE4E5B9ULL;
  return h ^ (h >> 29);
}

static int tdm_prepare_thresholds(b200mppi_tdm* t, double alpha, cudaStream_t st) {
  if (t->thr_alpha == alpha && t->thr_d) return B200MPPI_OK;
  uint64_t T[SAMPLE_TABLE_WORDS];
  t->thr_ok = t->pmf_valid && build_sample_thresholds(alpha, t->min_total, T);
  t->thr_alpha = alpha;
  if (!t->thr_d) CU(cudaMalloc(&t->thr_d, sizeof(T)));
  if (t->thr_ok) {
    // pageable source: the copy is staged by the driver before the call returns
    CU(cudaMemcpyAsync(t->thr_d, T, sizeof(T), cudaMemcpyHostToDevice, st));
  }
  return B200MPPI_OK;
}

static void tdm_advance_sig(b200mppi_tdm* t) {
  t->sig = mix_sig(mix_sig(t->sig, ((uint64_t)t->rows << 32) | (uint32_t)t->cols), 0x5a);
}

// Row segments per generator tile: enough CTAs to fill the GPU (the stream of a generator is sequential,
// so parallelism beyond M*tx*ty generators comes from GF(2) jump-ahead), at most SAMPLE_MAX_SEGS.
constexpr int SAMPLE_MAX_SEGS = 33;
constexpr int SAMPLE_BOX_MAX_SEGS = 128;   // boxed launches of a rank holding few maps go down to one-row segments
static int tdm_prepare_jump(b200mppi_tdm* t, cudaStream_t st) {
  const int tx = t->cfg.tdm_thread_x, ty = t->cfg.tdm_thread_y;
  const int nrow = (t->rows + tx - 1) / tx, ncol = (t->cols + ty - 1) / ty;
  const int groups = (t->num_maps + 7) / 8;
  // enough CTAs (~4k, i.e. several waves of the 5 resident CTAs per SM) to keep every SM busy through the
  // tail; a rank holding M/8 = 32 maps (8 GPUs) gets 2-row segments (33 of them; sweep: tools/sampler_segs.py)
  int segs = (4096 + tx * groups - 1) / (tx * groups);
  if (const char* e = getenv("B200MPPI_SAMPLE_SEGS")) segs = atoi(e);      // tuning / test hook
  if (segs > SAMPLE_MAX_SEGS) segs = SAMPLE_MAX_SEGS;
  if (segs > nrow) segs = nrow;
  if (segs < 1) segs = 1;
  const int seg_rows = (nrow + segs - 1) / segs;
  if (t->jump_d && t->jump_segs == segs && t->jump_seg_rows == seg_rows && t->jump_rows == t->rows &&
      t->jump_cols == t->cols)
    return B200MPPI_OK;
  if (!t->jump_d) CU(cudaMalloc(&t->jump_d, (size_t)(SAMPLE_MAX_SEGS - 1) * 2 * 256 * sizeof(uint64_t)));
  if (!t->jump_tile_d) CU(cudaMalloc(&t->jump_tile_d, (size_t)4 * 256 * sizeof(uint64_t)));
  {
    int64_t ks[4];
    sample_tile_draws(t->rows, t->cols, tx, ty, ks);
    std::vector<uint64_t> h(4 * 256);
    build_jump_matrices(ks, 4, h.data());
    CU(cudaMemcpyAsync(t->jump_tile_d, h.data(), h.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));            // h is a temporary
  }
  // width classes: 0 = full tile column (ncol cells), 1 = the last, narrower column
  int last_w = t->cols - (ty - 1) * ncol;
  for (int iy = ty - 1; iy >= 0 && last_w <= 0; --iy) last_w = t->cols - iy * ncol;   // first non-empty from the right
  if (last_w > ncol) last_w = ncol;
  if (last_w < 0) last_w = 0;
  auto upload_set = [&](uint64_t* dst, int nsegs, int rows_per_seg) -> int {
    if (nsegs <= 1) return B200MPPI_OK;
    std::vector<uint64_t> h((size_t)(nsegs - 1) * 2 * 256);
    build_jump_series((int64_t)rows_per_seg * ncol, (int64_t)rows_per_seg * last_w, nsegs, h.data());
    CU(cudaMemcpyAsync(dst, h.data(), h.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));            // h is a temporary
    return B200MPPI_OK;
  };
  int rc = upload_set(t->jump_d, segs, seg_rows);
  if (rc) return rc;
  // a boxed launch covers a few tile rows only: finer row segments keep every SM busy through several waves
  // (with whole-map segment sizes a large share of the SM-cycles sits idle in the tail)
  // ~6 waves of the ~6 resident CTAs per SM, for a box of ~8 tile rows sampled ~14 maps per CTA (the segment count
  // only splits the work: every segment starts from its generator's jumped state, the draws are the same).  At
  // config 5 on an H100 that is 32 segments; 16 (3 waves) left the boxed kernel ~5 % slower, 64 ~4 % slower.
  int bsegs = (6 * 6 * device_sm_count() + 8 * ((t->num_maps + 13) / 14) - 1) / (8 * ((t->num_maps + 13) / 14));
  if (const char* e = getenv("B200MPPI_SAMPLE_BOX_SEGS")) bsegs = atoi(e);
  if (bsegs > SAMPLE_BOX_MAX_SEGS) bsegs = SAMPLE_BOX_MAX_SEGS;
  if (bsegs > nrow) bsegs = nrow;
  if (bsegs < segs) bsegs = segs;
  if (bsegs < 1) bsegs = 1;
  const int bseg_rows = (nrow + bsegs - 1) / bsegs;
  if (!t->jump_box_d) CU(cudaMalloc(&t->jump_box_d, (size_t)(SAMPLE_BOX_MAX_SEGS - 1) * 2 * 256 * sizeof(uint64_t)));
  if ((rc = upload_set(t->jump_box_d, bsegs, bseg_rows))) return rc;
  t->box_segs = bsegs; t->box_seg_rows = bseg_rows;
  t->jump_segs = segs; t->jump_seg_rows = seg_rows; t->jump_rows = t->rows; t->jump_cols = t->cols;
  return B200MPPI_OK;
}

static void fill_v2(const b200mppi_tdm* t, SampleGridsV2Args& a, int slot) {
  a.t[slot].grid = t->grid; a.t[slot].cum = t->cum; a.t[slot].states = t->states;
  a.t[slot].states_out = t->states_alt;
  a.t[slot].qvals = t->qvals; a.t[slot].bpad = t->bpad;
  if (slot == 0) {
    a.thresholds = t->thr_d; a.jump = t->jump_d;
    a.rows = t->rows; a.cols = t->cols; a.grid_rows = t->cfg.max_map_rows; a.pitch = t->pitch;
    a.tx = t->cfg.tdm_thread_x; a.ty = t->cfg.tdm_thread_y; a.num_maps = t->num_maps;
    a.segs = t->jump_segs; a.seg_rows = t->jump_seg_rows;
    sample_box_full(a);
    if (a.ty * a.gm > 256) a.gm = 256 / a.ty;          // wide thread tiles: fewer maps per CTA (0: does not fit)
  }
}

// Restrict a whole-map launch description to the tile rows / row range / tile columns covering the reach box `b`
// (reach_box_decide, kernels.h).
static void apply_box(const b200mppi_tdm* t, SampleGridsV2Args& a, const ReachBox& b) {
  const int nrow = (a.rows + a.tx - 1) / a.tx, ncol = (a.cols + a.ty - 1) / a.ty;
  a.segs = t->box_segs; a.seg_rows = t->box_seg_rows; a.jump = t->jump_box_d;
  a.row_lo = b.row_lo; a.row_hi = b.row_hi;
  a.tix_lo = b.row_lo / nrow;
  a.tiy_lo = b.col_lo / ncol;
  a.nact = (b.col_hi - 1) / ncol - a.tiy_lo + 1;
  int gm = 128 / a.nact;                                // ~4 warps per CTA whatever the number of active tile columns
  if (gm > SG_GM_MAX) gm = SG_GM_MAX;
  if (gm > a.num_maps) gm = a.num_maps;
  if (gm < 1) gm = 1;
  a.gm = gm;
  a.write_states = 0;
  a.disc_cx = b.cx; a.disc_cy = b.cy; a.disc_r = b.r;
}

// Two distinct TDMs whose generators are in identical states over identical tiles: one stream of draws samples both.
static bool tdm_same_stream(const b200mppi_tdm* l, const b200mppi_tdm* g) {
  return l != g && l->sig == g->sig && l->rows == g->rows && l->cols == g->cols && l->num_maps == g->num_maps &&
         l->pitch == g->pitch && l->cfg.tdm_thread_x == g->cfg.tdm_thread_x &&
         l->cfg.tdm_thread_y == g->cfg.tdm_thread_y && l->cfg.max_map_rows == g->cfg.max_map_rows;
}

// How one sampling call samples one TDM or a lin/ang pair.  Fused: the pair's generator states are identical (same
// seed, same history: the reference seeds both with cfg.seed), so ONE staged launch (nt = 2, args a[0]) draws each
// uniform once and samples both maps.  Otherwise each TDM on its own, one after the other: the staged sampler (nt = 1,
// args a[i]) when its PMF is well-formed at this alpha and the launch fits, else the generic per-generator kernel.
// boxed[i]: a[i] samples only the reach box (plan_box); generator states still advance as for whole maps.
struct SamplePlan {
  b200mppi_tdm* t[2] = {};
  int nt = 1;
  bool fused = false;
  bool v2[2] = {};
  bool boxed[2] = {};
  double alpha = 1.0;
  SampleGridsV2Args a[2] = {};
};

// Host preparation (threshold tables; jump tables where the staged sampler may run) and the whole-map plan of TDM l,
// or of the pair l, g.  g may be l: that TDM is then sampled twice.
static int plan_sampling(b200mppi_tdm* l, b200mppi_tdm* g, double alpha, cudaStream_t st, SamplePlan* pl) {
  *pl = SamplePlan{};
  pl->t[0] = l; pl->t[1] = g; pl->nt = g ? 2 : 1; pl->alpha = alpha;
  int rc;
  for (int i = 0; i < pl->nt; ++i) {
    if (!pl->t[i]->pmf_set) return fail(B200MPPI_ESTATE, "sample_grids: PMF grid not set");
    if ((rc = tdm_prepare_thresholds(pl->t[i], alpha, st))) return rc;
  }
  if (l->thr_ok && (rc = tdm_prepare_jump(l, st))) return rc;
  if (g && tdm_same_stream(l, g) && l->thr_ok && g->thr_ok) {      // the fused launch runs on l's jump tables
    fill_v2(l, pl->a[0], 0);
    fill_v2(g, pl->a[0], 1);
    if (sample_grids_v2_fits(pl->a[0], 2)) { pl->fused = pl->v2[0] = pl->v2[1] = true; return B200MPPI_OK; }
    pl->a[0] = SampleGridsV2Args{};
  }
  if (g && g->thr_ok && (rc = tdm_prepare_jump(g, st))) return rc;
  for (int i = 0; i < pl->nt; ++i) {
    if (!pl->t[i]->thr_ok) continue;
    fill_v2(pl->t[i], pl->a[i], 0);
    pl->v2[i] = sample_grids_v2_fits(pl->a[i], 1);
  }
  return B200MPPI_OK;
}

// Narrow a plan's staged launches to `b` where the narrowed launch fits; the others (and the generic kernel) keep
// sampling whole maps.
static void plan_box(SamplePlan* pl, const ReachBox& b) {
  for (int i = 0; i < (pl->fused ? 1 : pl->nt); ++i) {
    if (!pl->v2[i]) continue;
    SampleGridsV2Args bx = pl->a[i];
    apply_box(pl->t[i], bx, b);
    if (sample_grids_v2_fits(bx, pl->fused ? 2 : 1)) { pl->a[i] = bx; pl->boxed[i] = true; }
  }
  if (pl->fused) pl->boxed[1] = pl->boxed[0];
}

// The state advance of a boxed staged launch (which stores no states) for TDM i, or for the fused pair: every generator
// jumped over its whole tile into the other buffer.  It does not depend on the box.
static void launch_plan_advance(const SamplePlan& pl, int i, cudaStream_t st) {
  const b200mppi_tdm* t = pl.t[i];
  launch_advance_states(t->states, t->states_alt, pl.fused ? pl.t[1]->states_alt : nullptr, t->jump_tile_d, t->rows,
                        t->cols, t->cfg.tdm_thread_x, t->cfg.tdm_thread_y, t->num_maps, st);
}

// After TDM i's sampling: the staged sampler left the advanced states in the other buffer (the generic kernel advances
// them in place), the maps are fresh inside the box only, if boxed, and the signature moves on.
static void plan_commit(const SamplePlan& pl, int i) {
  b200mppi_tdm* t = pl.t[i];
  if (pl.v2[i]) std::swap(t->states, t->states_alt);
  t->grid_partial = pl.boxed[i];
  t->partial_alpha = pl.alpha;
  tdm_advance_sig(t);
}

// Issue a plan's launches -- each sampler launch followed, if boxed, by its state advance unless `advanced` (the fused
// pair's advance is already queued: stage_sample_tdms) -- add their number to *launches, and commit every TDM.
static int plan_launch(SamplePlan& pl, bool advanced, cudaStream_t st, int64_t* launches) {
  for (int i = 0; i < (pl.fused ? 1 : pl.nt); ++i) {
    b200mppi_tdm* t = pl.t[i];
    if (pl.v2[i]) {
      // the states as they are now: when lin == ang the first sampling has swapped the buffers
      pl.a[i].t[0].states = t->states; pl.a[i].t[0].states_out = t->states_alt;
      launch_sample_grids_v2(pl.a[i], pl.fused ? 2 : 1, st);
      if (pl.boxed[i] && !advanced) launch_plan_advance(pl, i, st);
    } else {
      SampleGridsArgs a{};
      a.grid = t->grid; a.cum = t->cum; a.states = t->states; a.qvals = t->qvals;
      a.num_bins = t->B; a.bpad = t->bpad; a.rows = t->rows; a.cols = t->cols;
      a.grid_rows = t->cfg.max_map_rows; a.pitch = t->pitch;
      a.tx = t->cfg.tdm_thread_x; a.ty = t->cfg.tdm_thread_y; a.num_maps = t->num_maps;
      a.alpha_dyn = pl.alpha;
      launch_sample_grids(a, st);
    }
    CHECK_LAUNCH();
    *launches += pl.boxed[i] && !advanced ? 2 : 1;
    plan_commit(pl, i);
    if (pl.fused) plan_commit(pl, 1);
  }
  return B200MPPI_OK;
}

// The whole maps of the last (boxed) sampling call, on demand: re-walk every tile from the pre-call states the
// double buffer still holds; the advanced states the walk stores are the ones `states` already holds.
static int tdm_complete_grid(b200mppi_tdm* t, cudaStream_t st) {
  if (!t->grid_partial) return B200MPPI_OK;
  SamplePlan pl;
  const int rc = plan_sampling(t, nullptr, t->partial_alpha, st, &pl);
  if (rc) return rc;
  if (!pl.v2[0]) return fail(B200MPPI_ESTATE, "complete_grid: sampler state changed");
  pl.a[0].t[0].states = t->states_alt; pl.a[0].t[0].states_out = t->states;
  launch_sample_grids_v2(pl.a[0], 1, st);
  CHECK_LAUNCH();
  t->grid_partial = false;
  return B200MPPI_OK;
}

static int tdm_init(b200mppi_tdm* t, const b200mppi_config* cfg) {
  t->cfg = *cfg;
  t->det_dyn = cfg->mode != B200MPPI_MODE_TDM;
  // MODE_TDM with world_size > 1: the M sampled maps are sharded over the ranks (rank r owns maps
  // [r*M/ws, (r+1)*M/ws)); generator (tid_x, m, tid_y) keeps its GLOBAL index, so the union of the ranks'
  // maps is bit-identical to a single-rank run
  const int ws = cfg->world_size < 1 ? 1 : cfg->world_size;
  if (!t->det_dyn && ws > 1 && cfg->num_grid_samples % ws != 0)
    return fail(B200MPPI_EINVAL, "tdm_create: num_grid_samples must be divisible by world_size");
  t->num_maps = t->det_dyn ? 1 : cfg->num_grid_samples / ws;
  const int m_total = t->det_dyn ? 1 : cfg->num_grid_samples;
  const int m_begin = t->det_dyn ? 0 : cfg->rank * t->num_maps;
  t->pitch = round_up(cfg->max_map_cols, 16);
  CU(cudaStreamCreateWithFlags(&t->stream, cudaStreamNonBlocking));
  t->own_stream = true;
  const size_t gbytes = (size_t)t->num_maps * cfg->max_map_rows * t->pitch;
  CU(cudaMalloc(&t->grid, gbytes));
  CU(cudaMemsetAsync(t->grid, 0, gbytes, t->stream));
  t->num_gen = (int64_t)cfg->tdm_thread_x * cfg->tdm_thread_y * t->num_maps;
  t->sig = mix_sig(mix_sig(mix_sig(cfg->seed, (uint64_t)t->num_gen), 0x71), (uint64_t)m_begin);
  std::vector<uint64_t> h((size_t)t->num_gen * 2);
  {
    // global generator index tid_x*(ty*M) + m*ty + tid_y (terrain.py:657-658); local storage uses the
    // same formula with the local map count
    const int64_t all = (int64_t)cfg->tdm_thread_x * cfg->tdm_thread_y * m_total;
    std::vector<uint64_t> g((size_t)all * 2);
    create_xoroshiro_states(g.data(), 0, all, cfg->seed);
    const int ty = cfg->tdm_thread_y;
    for (int ix = 0; ix < cfg->tdm_thread_x; ++ix)
      for (int ml = 0; ml < t->num_maps; ++ml)
        for (int iy = 0; iy < ty; ++iy) {
          const int64_t src = (int64_t)ix * ((int64_t)ty * m_total) + (int64_t)(m_begin + ml) * ty + iy;
          const int64_t dst = (int64_t)ix * ((int64_t)ty * t->num_maps) + (int64_t)ml * ty + iy;
          h[2 * dst] = g[2 * src]; h[2 * dst + 1] = g[2 * src + 1];
        }
  }
  CU(cudaMalloc(&t->states, h.size() * sizeof(uint64_t)));
  CU(cudaMalloc(&t->states_alt, h.size() * sizeof(uint64_t)));
  CU(cudaMemcpyAsync(t->states, h.data(), h.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, t->stream));
  // both halves of the double buffer start alike: a whole-map sampling writes only the generators whose tile holds map
  // cells, the others (tiles below / right of the map) keep their states across the swap, as in the reference
  CU(cudaMemcpyAsync(t->states_alt, h.data(), h.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, t->stream));
  CU(cudaStreamSynchronize(t->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_destroy(b200mppi_tdm* t);

extern "C" int b200mppi_tdm_create(const b200mppi_config* cfg, b200mppi_tdm** out) {
  if (!cfg || !out) return fail(B200MPPI_EINVAL, "tdm_create: null argument");
  if (cfg->max_map_rows < 1 || cfg->max_map_cols < 1 || cfg->tdm_thread_x < 1 || cfg->tdm_thread_y < 1 ||
      cfg->num_grid_samples < 1)
    return fail(B200MPPI_EINVAL, "tdm_create: bad sizes");
  if (b200mppi_device_count() < 1) return fail(B200MPPI_ECUDA, "tdm_create: no CUDA device (no CPU fallback)");
  CU(cudaSetDevice(cfg->device));
  b200mppi_tdm* t = new b200mppi_tdm();
  const int rc = tdm_init(t, cfg);
  if (rc) {                                   // release whatever was allocated before the failure
    const std::string keep = g_err;
    b200mppi_tdm_destroy(t);
    g_err = keep;
    return rc;
  }
  *out = t;
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_destroy(b200mppi_tdm* t) {
  if (!t) return B200MPPI_OK;
  cudaSetDevice(t->cfg.device);
  cudaFree(t->grid); cudaFree(t->states); cudaFree(t->pmf); cudaFree(t->cum); cudaFree(t->qvals);
  cudaFree(t->obstacle); cudaFree(t->unknown); cudaFree(t->risk); cudaFree(t->thr_d); cudaFree(t->states_alt); cudaFree(t->jump_d); cudaFree(t->jump_tile_d); cudaFree(t->jump_box_d);
  if (t->own_stream && t->stream) cudaStreamDestroy(t->stream);
  delete t;
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_set_stream(b200mppi_tdm* t, void* s) {
  if (!t) return fail(B200MPPI_EINVAL, "null tdm");
  if (t->own_stream && t->stream) { cudaStreamSynchronize(t->stream); cudaStreamDestroy(t->stream); }
  t->stream = (cudaStream_t)s;
  t->own_stream = false;
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_set_pmf(b200mppi_tdm* t, const int8_t* pmf, int32_t B, int32_t rows, int32_t cols,
                                    const float* bin_values, const float bounds[2], float res,
                                    const float pxl[2], const float pyl[2]) {
  if (!t || !pmf || !bin_values || !bounds || !pxl || !pyl) return fail(B200MPPI_EINVAL, "set_pmf: null argument");
  if (B < 1 || B > 127 || rows < 1 || cols < 1) return fail(B200MPPI_EINVAL, "set_pmf: bad shape");
  if (rows > t->cfg.max_map_rows || cols > t->cfg.max_map_cols)
    return fail(B200MPPI_EINVAL, "set_pmf: padded PMF larger than max_map_dim (crop on the host first, terrain.py:562-583)");
  CU(cudaSetDevice(t->cfg.device));
  const int bpad = round_up(B, 4);
  const size_t pbytes = (size_t)B * rows * cols, cbytes = (size_t)bpad * rows * cols;
  if (pbytes > t->pmf_cap) { cudaFree(t->pmf); t->pmf = nullptr; CU(cudaMalloc(&t->pmf, pbytes)); t->pmf_cap = pbytes; }
  if (cbytes > t->cum_cap) { cudaFree(t->cum); t->cum = nullptr; CU(cudaMalloc(&t->cum, cbytes)); t->cum_cap = cbytes; }
  if (!t->qvals) CU(cudaMalloc(&t->qvals, 128));
  CU(cudaMemcpyAsync(t->pmf, pmf, pbytes, cudaMemcpyHostToDevice, t->stream));
  {  // well-formed PMF? (entries in [0,127], running sums <= 127) and the smallest column total
    const size_t cells = (size_t)rows * cols;
    std::vector<int16_t> acc(cells, 0);
    bool ok = true;
    for (int b = 0; b < B && ok; ++b) {
      const int8_t* plane = pmf + (size_t)b * cells;
      for (size_t i = 0; i < cells; ++i) {
        const int v = plane[i];
        const int s2 = acc[i] + v;
        if (v < 0 || s2 > 127) { ok = false; break; }
        acc[i] = (int16_t)s2;
      }
    }
    int mn = 127;
    if (ok) for (size_t i = 0; i < cells; ++i) mn = acc[i] < mn ? acc[i] : mn;
    t->pmf_valid = ok;
    t->min_total = ok ? mn : 0;
    t->thr_alpha = -1.0;          // force a rebuild of the threshold table
  }
  // quantised bin values, terrain.py:689 as compiled: int8(100.*(f32-f32)/f64(f32 range)), truncation
  int8_t q[128];
  std::memset(q, 0, sizeof(q));
  const float range = bounds[1] - bounds[0];
  for (int b = 0; b < B; ++b) {
    const float d = bin_values[b] - bounds[0];
    const double v = ((double)d * 100.0) / (double)range;
    q[b] = (int8_t)(int16_t)std::trunc(v);
  }
  CU(cudaMemcpyAsync(t->qvals, q, 128, cudaMemcpyHostToDevice, t->stream));
  {
    const double ratio = 0.01 * (double)range;            // as the rollout kernels decode a byte (mppi.py:674-684)
    double mx = 0.0;
    for (int b = 0; b < B; ++b) mx = std::fmax(mx, std::fabs((double)bounds[0] + ratio * (double)q[b]));
    t->tr_abs_max = (float)mx;
  }
  t->grid_partial = false;                                // a new PMF: nothing left to complete
  launch_build_cum(t->pmf, t->cum, B, bpad, rows, cols, t->stream);
  CHECK_LAUNCH();
  CU(cudaStreamSynchronize(t->stream));
  t->B = B; t->bpad = bpad; t->rows = rows; t->cols = cols;
  t->bounds[0] = bounds[0]; t->bounds[1] = bounds[1];
  t->res = res; t->pxl[0] = pxl[0]; t->pxl[1] = pxl[1]; t->pyl[0] = pyl[0]; t->pyl[1] = pyl[1];
  t->pmf_set = true;
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_set_pmf_collapsed(b200mppi_tdm* t, const int8_t* raw, int32_t B, int32_t H, int32_t W,
                                              int32_t keep_r, int32_t keep_c, int32_t pad, const float* bin_values,
                                              const float bounds[2], float res, const float pxl[2], const float pyl[2],
                                              double alpha, int8_t* pmf_out, int8_t* risk_out, int32_t* bad_out) {
  if (!t || !raw || !bin_values || !bounds || !pxl || !pyl) return fail(B200MPPI_EINVAL, "set_pmf_collapsed: null argument");
  if (t->cfg.mode != B200MPPI_MODE_DET_DYN && t->cfg.mode != B200MPPI_MODE_SPEED_MAP)
    return fail(B200MPPI_ESTATE, "set_pmf_collapsed: only for the one-map modes");
  if (B < 1 || B > 127 || H < 1 || W < 1 || keep_r < 1 || keep_c < 1 || keep_r > H || keep_c > W || pad < 0 ||
      !(alpha > 0.0 && alpha <= 1.0))
    return fail(B200MPPI_EINVAL, "set_pmf_collapsed: bad shape / alpha");
  const int Hp = keep_r + 2 * pad, Wp = keep_c + 2 * pad;
  if (Hp > t->cfg.max_map_rows || Wp > t->cfg.max_map_cols)
    return fail(B200MPPI_EINVAL, "set_pmf_collapsed: padded map larger than max_map_dim");
  CU(cudaSetDevice(t->cfg.device));
  const bool speed = t->cfg.mode == B200MPPI_MODE_SPEED_MAP;
  const size_t raw_bytes = (size_t)B * H * W, out_bytes = (size_t)B * Hp * Wp;
  int8_t* raw_d = nullptr; float* bv_d = nullptr; int* bad_d = nullptr;
  std::vector<int8_t> host_out(out_bytes);
  int rc = B200MPPI_OK;
  do {
    if (cudaMalloc(&raw_d, raw_bytes) != cudaSuccess || cudaMalloc(&bv_d, (size_t)B * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&bad_d, sizeof(int)) != cudaSuccess) {
      (void)cudaGetLastError();
      rc = fail(B200MPPI_ENOMEM, "set_pmf_collapsed: cudaMalloc");
      break;
    }
    if (out_bytes > t->pmf_cap) { cudaFree(t->pmf); t->pmf = nullptr; if (cudaMalloc(&t->pmf, out_bytes) != cudaSuccess) { rc = fail(B200MPPI_ENOMEM, "set_pmf_collapsed: cudaMalloc"); break; } t->pmf_cap = out_bytes; }
    const int rpitch = round_up(Wp, 16);
    if (speed) {
      const size_t rbytes = (size_t)Hp * rpitch;
      if (rbytes > t->risk_cap) { cudaFree(t->risk); t->risk = nullptr; if (cudaMalloc(&t->risk, rbytes) != cudaSuccess) { rc = fail(B200MPPI_ENOMEM, "set_pmf_collapsed: cudaMalloc"); break; } t->risk_cap = rbytes; }
      cudaMemsetAsync(t->risk, 0, rbytes, t->stream);
    }
    cudaMemcpyAsync(raw_d, raw, raw_bytes, cudaMemcpyHostToDevice, t->stream);
    cudaMemcpyAsync(bv_d, bin_values, (size_t)B * sizeof(float), cudaMemcpyHostToDevice, t->stream);
    cudaMemsetAsync(bad_d, 0, sizeof(int), t->stream);
    launch_collapse_pad(raw_d, t->pmf, speed ? t->risk : nullptr, bad_d, bv_d, B, H, W, keep_r, keep_c, pad, rpitch, alpha,
                        bounds[0], bounds[1] - bounds[0], t->cfg.mode, t->stream);
    int bad = 0;
    cudaMemcpyAsync(&bad, bad_d, sizeof(int), cudaMemcpyDeviceToHost, t->stream);
    cudaMemcpyAsync(host_out.data(), t->pmf, out_bytes, cudaMemcpyDeviceToHost, t->stream);
    if (speed && risk_out)
      cudaMemcpy2DAsync(risk_out, Wp, t->risk, rpitch, Wp, Hp, cudaMemcpyDeviceToHost, t->stream);
    if (cudaStreamSynchronize(t->stream) != cudaSuccess || cudaGetLastError() != cudaSuccess) {
      rc = fail(B200MPPI_ECUDA, "set_pmf_collapsed: CUDA error");
      break;
    }
    if (bad_out) *bad_out = bad;
    if (speed) t->risk_set = true;
  } while (0);
  cudaFree(raw_d); cudaFree(bv_d); cudaFree(bad_d);
  if (rc) return rc;
  if (pmf_out) std::memcpy(pmf_out, host_out.data(), out_bytes);
  // the collapsed PMF is already resident in t->pmf: finish exactly like set_pmf (cumulative table, bin
  // quantisation, validity, geometry) from the host copy
  return b200mppi_tdm_set_pmf(t, host_out.data(), B, Hp, Wp, bin_values, bounds, res, pxl, pyl);
}

extern "C" int b200mppi_tdm_set_bin_quantisation(b200mppi_tdm* t, const int8_t* qvals, int32_t n) {
  if (!t || !qvals) return fail(B200MPPI_EINVAL, "set_bin_quantisation: null argument");
  if (!t->pmf_set || n != t->B) return fail(B200MPPI_EINVAL, "set_bin_quantisation: call after set_pmf with num_bins values");
  CU(cudaSetDevice(t->cfg.device));
  CU(cudaMemcpyAsync(t->qvals, qvals, (size_t)n, cudaMemcpyHostToDevice, t->stream));
  CU(cudaStreamSynchronize(t->stream));
  {
    const double ratio = 0.01 * (double)(float)(t->bounds[1] - t->bounds[0]);
    double mx = 0.0;
    for (int b = 0; b < n; ++b) mx = std::fmax(mx, std::fabs((double)t->bounds[0] + ratio * (double)qvals[b]));
    t->tr_abs_max = (float)mx;
  }
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_sample_grid_view(b200mppi_tdm* t, void** ptr, int32_t* pitch) {
  if (!t) return fail(B200MPPI_EINVAL, "null tdm");
  if (t->grid_partial) {                      // a raw view must show whole maps
    CU(cudaSetDevice(t->cfg.device));
    const int rc = tdm_complete_grid(t, t->stream);
    if (rc) return rc;
    CU(cudaStreamSynchronize(t->stream));
  }
  if (ptr) *ptr = t->grid;
  if (pitch) *pitch = t->pitch;
  return B200MPPI_OK;
}

static int upload_plane(b200mppi_tdm* t, int8_t** dst, size_t* cap, const int8_t* src, int rows, int cols, int pitch) {
  const size_t bytes = (size_t)rows * pitch;
  if (bytes > *cap) { cudaFree(*dst); *dst = nullptr; CU(cudaMalloc(dst, bytes)); *cap = bytes; }
  CU(cudaMemsetAsync(*dst, 0, bytes, t->stream));
  if (src) CU(cudaMemcpy2DAsync(*dst, pitch, src, cols, cols, rows, cudaMemcpyHostToDevice, t->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_set_masks(b200mppi_tdm* t, const int8_t* obs, const int8_t* unk, int32_t rows,
                                      int32_t cols) {
  if (!t) return fail(B200MPPI_EINVAL, "null tdm");
  if (rows < 1 || cols < 1) return fail(B200MPPI_EINVAL, "set_masks: bad shape");
  CU(cudaSetDevice(t->cfg.device));
  const int pitch = round_up(cols, 16);
  size_t cap2 = t->mask_cap;
  int rc = upload_plane(t, &t->obstacle, &t->mask_cap, obs, rows, cols, pitch);
  if (rc) return rc;
  rc = upload_plane(t, &t->unknown, &cap2, unk, rows, cols, pitch);
  if (rc) return rc;
  CU(cudaStreamSynchronize(t->stream));
  bool b01 = true;
  for (const int8_t* m : {obs, unk})
    if (m)
    {
      const size_t n = (size_t)rows * cols;
      uint64_t bad = 0;                                       // bits other than bit 0 of any byte, eight bytes at a time
      size_t i = 0;
      for (; i + 8 <= n; i += 8) { uint64_t w; std::memcpy(&w, m + i, 8); bad |= w & 0xFEFEFEFEFEFEFEFEull; }
      for (; i < n; ++i) bad |= (uint64_t)(uint8_t)m[i] & 0xFEull;
      b01 = b01 && bad == 0;
    }
  t->masks01 = b01;
  t->mask_rows = rows; t->mask_cols = cols; t->mask_pitch = pitch; t->masks_set = true;
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_set_risk_map(b200mppi_tdm* t, const int8_t* risk, int32_t rows, int32_t cols) {
  if (!t || !risk) return fail(B200MPPI_EINVAL, "set_risk_map: null argument");
  if (rows < 1 || cols < 1) return fail(B200MPPI_EINVAL, "set_risk_map: bad shape");
  CU(cudaSetDevice(t->cfg.device));
  int rc = upload_plane(t, &t->risk, &t->risk_cap, risk, rows, cols, round_up(cols, 16));
  if (rc) return rc;
  CU(cudaStreamSynchronize(t->stream));
  t->risk_set = true;
  return B200MPPI_OK;
}

// Host-side evaluation of the sampler's threshold lookup (the very function the kernel inlines): lets the
// CPU test-suite check the bucket tables against the reference's float arithmetic without a GPU.
extern "C" int b200mppi_debug_sample_threshold(double alpha_dyn, int32_t q_cap, const uint64_t* draws, int64_t n,
                                               uint8_t* q_out) {
  if (!draws || !q_out || n < 0) return fail(B200MPPI_EINVAL, "debug_sample_threshold: bad argument");
  uint64_t T[SAMPLE_TABLE_WORDS];
  if (!build_sample_thresholds(alpha_dyn, q_cap, T))
    return fail(B200MPPI_ESTATE, "debug_sample_threshold: alpha_dyn / q_cap not representable by the bucket table "
                                 "(the sampler falls back to its generic kernel)");
  for (int64_t i = 0; i < n; ++i) q_out[i] = (uint8_t)sample_threshold_q(draws[i], T);
  return B200MPPI_OK;
}

// The approximate float32 operations of the kernels, evaluated on the device by the very inline helpers the kernels
// use (common.cuh; logf / cosf are the libdevice routines of xoro_normal), compiled with the library's flags: their
// results are deterministic functions of the inputs, so the test oracle can take them from here and predict every
// rollout cost bit for bit.
__global__ void debug_device_math_kernel(int op, const float* __restrict__ a, const float* __restrict__ b,
                                         float* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float x = a[i];
    float r;
    switch (op) {
      case B200MPPI_MATH_SIN_APPROX: r = sin_approx(x); break;
      case B200MPPI_MATH_COS_APPROX: r = cos_approx(x); break;
      case B200MPPI_MATH_SQRT_APPROX: r = sqrt_approx(x); break;
      case B200MPPI_MATH_DIV_APPROX: r = div_approx(x, b[i]); break;
      case B200MPPI_MATH_DIV_FULL: r = div_full(x, b[i]); break;
      case B200MPPI_MATH_LOGF: r = logf(x); break;
      default: r = cosf(x); break;                         // B200MPPI_MATH_COSF (op checked on the host)
    }
    out[i] = r;
  }
}

extern "C" int b200mppi_debug_device_math(int32_t op, const float* a, const float* b, float* out, int64_t n) {
  if (op < B200MPPI_MATH_SIN_APPROX || op > B200MPPI_MATH_COSF) return fail(B200MPPI_EINVAL, "debug_device_math: unknown op");
  const bool binary = op == B200MPPI_MATH_DIV_APPROX || op == B200MPPI_MATH_DIV_FULL;
  if (n < 0 || (n > 0 && (!a || !out || (binary && !b)))) return fail(B200MPPI_EINVAL, "debug_device_math: bad argument");
  if (n == 0) return B200MPPI_OK;
  const size_t bytes = (size_t)n * sizeof(float);
  float *da = nullptr, *db = nullptr, *dout = nullptr;
  cudaError_t e = cudaMalloc(&da, bytes);
  if (e == cudaSuccess && binary) e = cudaMalloc(&db, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&dout, bytes);
  if (e == cudaSuccess) e = cudaMemcpy(da, a, bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && binary) e = cudaMemcpy(db, b, bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    const int threads = 256;
    const int64_t blocks = std::min<int64_t>((n + threads - 1) / threads, 65535);
    debug_device_math_kernel<<<(unsigned)blocks, threads>>>(op, da, db, dout, n);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(out, dout, bytes, cudaMemcpyDeviceToHost);
  cudaFree(da);
  cudaFree(db);
  cudaFree(dout);
  if (e != cudaSuccess) return fail(B200MPPI_ECUDA, std::string("debug_device_math: ") + cudaGetErrorString(e));
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_sample_grids(b200mppi_tdm* t, double alpha_dyn) {
  if (!t) return fail(B200MPPI_EINVAL, "null tdm");
  CU(cudaSetDevice(t->cfg.device));
  SamplePlan pl;
  int64_t launches = 0;                       // a TDM keeps no launch count
  int rc = plan_sampling(t, nullptr, alpha_dyn, t->stream, &pl);
  if (rc || (rc = plan_launch(pl, false, t->stream, &launches))) return rc;
  CU(cudaStreamSynchronize(t->stream));
  return B200MPPI_OK;
}

static size_t tdm_grid_bytes(const b200mppi_tdm* t) {
  return (size_t)t->num_maps * t->cfg.max_map_rows * t->cfg.max_map_cols;
}

extern "C" int b200mppi_tdm_get_sample_grids(b200mppi_tdm* t, int8_t* out, size_t bytes) {
  if (!t || !out) return fail(B200MPPI_EINVAL, "null argument");
  if (bytes != tdm_grid_bytes(t)) return fail(B200MPPI_EINVAL, "get_sample_grids: size mismatch");
  CU(cudaSetDevice(t->cfg.device));
  { const int rc = tdm_complete_grid(t, t->stream); if (rc) return rc; }
  CU(cudaMemcpy2DAsync(out, t->cfg.max_map_cols, t->grid, t->pitch, t->cfg.max_map_cols,
                       (size_t)t->num_maps * t->cfg.max_map_rows, cudaMemcpyDeviceToHost, t->stream));
  CU(cudaStreamSynchronize(t->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_set_sample_grids(b200mppi_tdm* t, const int8_t* in, size_t bytes) {
  if (!t || !in) return fail(B200MPPI_EINVAL, "null argument");
  if (bytes != tdm_grid_bytes(t)) return fail(B200MPPI_EINVAL, "set_sample_grids: size mismatch");
  CU(cudaSetDevice(t->cfg.device));
  t->grid_partial = false;                    // every cell is overwritten
  CU(cudaMemcpy2DAsync(t->grid, t->pitch, in, t->cfg.max_map_cols, t->cfg.max_map_cols,
                       (size_t)t->num_maps * t->cfg.max_map_rows, cudaMemcpyHostToDevice, t->stream));
  CU(cudaStreamSynchronize(t->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_tdm_num_generators(b200mppi_tdm* t, int64_t* out) {
  if (!t || !out) return fail(B200MPPI_EINVAL, "null argument");
  *out = t->num_gen;
  return B200MPPI_OK;
}
extern "C" int b200mppi_tdm_get_rng_states(b200mppi_tdm* t, uint64_t* out, size_t bytes) {
  if (!t || !out || bytes != (size_t)t->num_gen * 16) return fail(B200MPPI_EINVAL, "get_rng_states: bad argument");
  CU(cudaSetDevice(t->cfg.device));
  CU(cudaMemcpyAsync(out, t->states, bytes, cudaMemcpyDeviceToHost, t->stream));
  CU(cudaStreamSynchronize(t->stream));
  return B200MPPI_OK;
}
extern "C" int b200mppi_tdm_set_rng_states(b200mppi_tdm* t, const uint64_t* in, size_t bytes) {
  if (!t || !in || bytes != (size_t)t->num_gen * 16) return fail(B200MPPI_EINVAL, "set_rng_states: bad argument");
  CU(cudaSetDevice(t->cfg.device));
  { const int rc = tdm_complete_grid(t, t->stream); if (rc) return rc; }   // completion needs the states it replaces
  CU(cudaMemcpyAsync(t->states, in, bytes, cudaMemcpyHostToDevice, t->stream));
  CU(cudaMemcpyAsync(t->states_alt, in, bytes, cudaMemcpyHostToDevice, t->stream));   // see tdm_init
  CU(cudaStreamSynchronize(t->stream));
  // content-derived signature: two TDMs given identical states compare equal again
  uint64_t h = 0x1234567ULL;
  for (size_t i = 0; i < bytes / 8; ++i) h = mix_sig(h, in[i]);
  t->sig = h;
  return B200MPPI_OK;
}

// --------------------------------------------------------------------------------------------- ground-truth realisations
// A set of `count` (lin, ang) float64 planes on one device; realisation i's lin plane is plane 2 i, its ang plane 2 i + 1.
struct b200mppi_realisations {
  int device = 0, count = 0, rows = 0, cols = 0;
  float res = 1, pxl[2] = {0, 0}, pyl[2] = {0, 0};
  double* d = nullptr;                  // (count, 2, rows, cols)
  size_t plane() const { return (size_t)rows * cols; }
  uintptr_t lo() const { return reinterpret_cast<uintptr_t>(d); }
  uintptr_t hi() const { return lo() + (size_t)2 * count * plane() * sizeof(double); }
};

// The live sets, which trial calls may read in place, and the address ranges of destroyed ones: a pointer into freed
// device memory looks like pageable host memory to cudaPointerGetAttributes, and must not be read as such.  A range is
// forgotten once a new set covers it; the oldest are dropped beyond REALISATION_RETIRED entries.
constexpr size_t REALISATION_RETIRED = 4096;
static std::mutex g_sets_mu;
static std::vector<b200mppi_realisations*> g_sets;
struct RetiredRange { int device; uintptr_t lo, hi; };
static std::vector<RetiredRange> g_retired;

extern "C" int b200mppi_tdm_draw_realisations(b200mppi_tdm* lin, b200mppi_tdm* ang, int32_t count,
                                              b200mppi_realisations** out) {
  if (!lin || !ang || !out) return fail(B200MPPI_EINVAL, "draw_realisations: null argument");
  if (count < 1) return fail(B200MPPI_EINVAL, "draw_realisations: count " + std::to_string(count) + " < 1");
  if (!lin->pmf_set || !ang->pmf_set) return fail(B200MPPI_ESTATE, "draw_realisations: PMF grid not set");
  if (lin->cfg.device != ang->cfg.device)
    return fail(B200MPPI_EINVAL, "draw_realisations: lin is on device " + std::to_string(lin->cfg.device) + ", ang on " +
                                 std::to_string(ang->cfg.device));
  if (lin->cfg.max_map_rows != ang->cfg.max_map_rows || lin->cfg.max_map_cols != ang->cfg.max_map_cols)
    return fail(B200MPPI_EINVAL, "draw_realisations: lin and ang sample planes differ in shape (max_map_dim)");
  CU(cudaSetDevice(lin->cfg.device));
  std::unique_ptr<b200mppi_realisations> s(new b200mppi_realisations());
  s->device = lin->cfg.device; s->count = count; s->rows = lin->cfg.max_map_rows; s->cols = lin->cfg.max_map_cols;
  s->res = lin->res;
  s->pxl[0] = lin->pxl[0]; s->pxl[1] = lin->pxl[1]; s->pyl[0] = lin->pyl[0]; s->pyl[1] = lin->pyl[1];
  struct Mem { double* p = nullptr; ~Mem() { cudaFree(p); } } mem;   // freed unless the set is registered
  CU(cudaMalloc(&mem.p, (size_t)2 * count * s->plane() * sizeof(double)));
  s->d = mem.p;
  // everything on lin's stream, after the work already issued on ang's
  CU(cudaStreamSynchronize(ang->stream));
  const cudaStream_t st = lin->stream;
  int64_t launches = 0;
  int rc;
  auto sample = [&](b200mppi_tdm* t) -> int {         // == b200mppi_tdm_sample_grids(t, 1.0)
    SamplePlan pl;
    int r = plan_sampling(t, nullptr, 1.0, st, &pl);
    return r ? r : plan_launch(pl, false, st, &launches);
  };
  for (int i = 0; i < count; ++i) {
    double* const planes = s->d + (size_t)2 * i * s->plane();
    const RealisationPlane pl{lin->grid, lin->pitch, lin->bounds[0], lin->bounds[1], planes};
    const RealisationPlane pa{ang->grid, ang->pitch, ang->bounds[0], ang->bounds[1], planes + s->plane()};
    if ((rc = sample(lin))) return rc;
    if (lin == ang) {                                 // the second sampling overwrites the first's map 0
      launch_realisation_convert(pl, pl, 1, s->rows, s->cols, st);
      CHECK_LAUNCH();
      if ((rc = sample(ang))) return rc;
      launch_realisation_convert(pa, pa, 1, s->rows, s->cols, st);
    } else {
      if ((rc = sample(ang))) return rc;
      launch_realisation_convert(pl, pa, 2, s->rows, s->cols, st);
    }
    CHECK_LAUNCH();
  }
  CU(cudaStreamSynchronize(st));
  {
    std::lock_guard<std::mutex> g(g_sets_mu);
    g_retired.erase(std::remove_if(g_retired.begin(), g_retired.end(), [&](const RetiredRange& r) {
                      return r.device == s->device && r.lo < s->hi() && s->lo() < r.hi;
                    }), g_retired.end());
    g_sets.push_back(s.get());
  }
  mem.p = nullptr;
  *out = s.release();
  return B200MPPI_OK;
}

extern "C" int b200mppi_realisations_destroy(b200mppi_realisations* s) {
  if (!s) return B200MPPI_OK;
  {
    std::lock_guard<std::mutex> g(g_sets_mu);
    auto it = std::find(g_sets.begin(), g_sets.end(), s);
    if (it == g_sets.end()) return fail(B200MPPI_EINVAL, "realisations_destroy: not a live realisation set");
    g_sets.erase(it);
    if (g_retired.size() >= REALISATION_RETIRED) g_retired.erase(g_retired.begin());
    g_retired.push_back(RetiredRange{s->device, s->lo(), s->hi()});
  }
  cudaSetDevice(s->device);
  cudaFree(s->d);
  delete s;
  return B200MPPI_OK;
}

static bool realisations_live(const b200mppi_realisations* s) {
  std::lock_guard<std::mutex> g(g_sets_mu);
  return s && std::find(g_sets.begin(), g_sets.end(), s) != g_sets.end();
}

extern "C" int b200mppi_realisations_info(const b200mppi_realisations* s, int32_t* count, int32_t* height,
                                          int32_t* width, double* res, double xlimits[2], double ylimits[2],
                                          int32_t* device) {
  if (!realisations_live(s)) return fail(B200MPPI_EINVAL, "realisations_info: not a live realisation set");
  if (count) *count = s->count;
  if (height) *height = s->rows;
  if (width) *width = s->cols;
  if (res) *res = s->res;
  if (xlimits) { xlimits[0] = s->pxl[0]; xlimits[1] = s->pxl[1]; }
  if (ylimits) { ylimits[0] = s->pyl[0]; ylimits[1] = s->pyl[1]; }
  if (device) *device = s->device;
  return B200MPPI_OK;
}

extern "C" int b200mppi_realisations_planes(const b200mppi_realisations* s, int32_t i, const double** lin,
                                            const double** ang) {
  if (!realisations_live(s)) return fail(B200MPPI_EINVAL, "realisations_planes: not a live realisation set");
  if (i < 0 || i >= s->count || !lin || !ang)
    return fail(B200MPPI_EINVAL, "realisations_planes: bad index " + std::to_string(i) + " or null output");
  *lin = s->d + (size_t)2 * i * s->plane();
  *ang = *lin + s->plane();
  return B200MPPI_OK;
}

extern "C" int b200mppi_realisations_copy_out(const b200mppi_realisations* s, int32_t i, double* lin, double* ang) {
  const double* dl;
  const double* da;
  const int rc = b200mppi_realisations_planes(s, i, &dl, &da);
  if (rc) return rc;
  CU(cudaSetDevice(s->device));
  CU(cudaMemcpy(lin, dl, s->plane() * sizeof(double), cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(ang, da, s->plane() * sizeof(double), cudaMemcpyDeviceToHost));
  return B200MPPI_OK;
}

// Where descriptor `d` of a trial call on `device` reads its grids: host arrays (*in_place false), or two planes of a
// live realisation set (*in_place true): both pointers device memory of that device, each at the start of a plane of one
// live set whose planes have the descriptor's height and width.  Anything else is refused, naming `who`.
static int trial_grid_source(const b200mppi_trial_desc& d, int device, const std::string& who, bool* in_place) {
  auto memory_type = [](const void* p, int* dev) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return cudaMemoryTypeUnregistered; }
    *dev = a.device;
    return a.type;
  };
  const void* ptrs[2] = {d.lin, d.ang};
  const b200mppi_realisations* sets[2] = {};
  bool dev_mem[2] = {};
  std::lock_guard<std::mutex> g(g_sets_mu);
  for (int k = 0; k < 2; ++k) {
    const char* name = k ? "ang" : "lin";
    const uintptr_t a = reinterpret_cast<uintptr_t>(ptrs[k]);
    int dev = -1;
    const cudaMemoryType type = memory_type(ptrs[k], &dev);
    dev_mem[k] = type == cudaMemoryTypeDevice || type == cudaMemoryTypeManaged;
    for (const b200mppi_realisations* s : g_sets)
      if (a >= s->lo() && a < s->hi()) sets[k] = s;
    if (!sets[k]) {
      for (const RetiredRange& r : g_retired)         // page-locked host memory is what it says it is
        if (type != cudaMemoryTypeHost && a >= r.lo && a < r.hi)
          return fail(B200MPPI_EINVAL, who + ": the " + name + " grid lies in a destroyed realisation set");
      if (dev_mem[k])
        return fail(B200MPPI_EINVAL, who + ": the " + name + " grid is device memory but not a plane of a live "
                                     "realisation set");
      continue;
    }
    if (!dev_mem[k] || dev != device || sets[k]->device != device)
      return fail(B200MPPI_EINVAL, who + ": the " + name + " grid is a realisation on device " +
                                   std::to_string(sets[k]->device) + ", the batch runs on device " + std::to_string(device));
    if ((a - sets[k]->lo()) % (sets[k]->plane() * sizeof(double)) != 0)
      return fail(B200MPPI_EINVAL, who + ": the " + name + " grid points into the middle of a realisation plane");
  }
  *in_place = sets[0] != nullptr;
  if ((sets[0] != nullptr) != (sets[1] != nullptr))
    return fail(B200MPPI_EINVAL, who + ": one grid is a device realisation, the other host memory");
  if (*in_place && sets[0] != sets[1])
    return fail(B200MPPI_EINVAL, who + ": lin and ang grids are planes of two different realisation sets");
  if (*in_place && (d.height != sets[0]->rows || d.width != sets[0]->cols))
    return fail(B200MPPI_EINVAL, who + ": grid of " + std::to_string(d.height) + " x " + std::to_string(d.width) +
                                 " cells, its realisation planes hold " + std::to_string(sets[0]->rows) + " x " +
                                 std::to_string(sets[0]->cols));
  return B200MPPI_OK;
}

// --------------------------------------------------------------------------------------------- planner
struct b200mppi_planner {
  b200mppi_config cfg{};
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int n_begin = 0, n_local = 0, T = 0, M = 1;
  // MODE_TDM with world_size > 1 shards the MAPS: every rank rolls out all N control sequences on its
  // M/ws maps (n_roll = N), exchanges per-(n,m) costs (all-to-all), and reduces its N/ws slice (n_red)
  bool shard_maps = false;
  int M_total = 1, n_roll = 0, n_red = 0, n_red_begin = 0;
  float* obstacles = nullptr; int num_obstacles = 0, obstacles_cap = 0;   // MODE_BAREBONE: (K,3) x, y, r
  float* costs_x = nullptr;    // (ws, N/ws, M_local): per-(n,m) costs of this rank's n-slice after the exchange
  float* noise = nullptr; float* u_cur = nullptr; float* u_prev = nullptr;
  float* costs = nullptr; float* weights = nullptr; float* costs_nm = nullptr; float* w_raw = nullptr;
  float* cta_partials = nullptr; float* rank_partial = nullptr; float* state_rollout = nullptr;
  uint64_t* states = nullptr;
  float* noiseT = nullptr; float* ctrl = nullptr; int npad = 0;   // windowed rollout kernel inputs
  alignas(64) unsigned char tmaps[4][128];
  const void* tmap_key[8] = {};  // what the cached tensor maps were encoded for (grids, masks, geometry)
  bool use_win = true;
  // reach-box sampling: 0 = whole maps every solve, 1 = box from the speed limit, 2 = box from this solve's
  // own clipped controls (max_n sum_t |v|, reduced by the prepare kernel into reach_d and read back mid-solve)
  int box_mode = 3;              // 3: window-first (planner_window_first), else as 2
  bool disc = true;              // sample the reach disc inside the box (B200MPPI_SAMPLE_DISC=0: the whole box)
  float* reach_d = nullptr;            // two slots, used alternately (noise_prepare_kernel)
  int reach_slot = 0;
  bool reach_valid = false;            // reach_d[reach_slot] holds this iteration's statistic
  unsigned* upd_counter_d = nullptr;   // ticket counter of update_partial_kernel's last-CTA tail
  bool bcast_done = false;             // this iteration's rank partial already went to the peers (update tail)
  bool prepared = false;         // noiseT / ctrl hold this iteration's controls
  bool pushed_direct = false;    // the last rollout kernel stored its costs straight into the peers (and signalled)
  int32_t last_box[5] = {};      // b200mppi_planner_sample_box
  // window-first sampling (stage_sample_tdms): this solve sampled only the window + ring up front (win_used), the
  // rectangle win_rect = [row_lo, row_hi, col_lo, col_hi) of its cells; escape flags of the two solve parities (M each)
  bool win_used = false;
  bool win_pending = false;            // the maps are sampled window-first for the next stage_rollout
  int32_t win_rect[4] = {};
  int32_t win_flagged = 0;             // maps flagged by the last window-first solve
  unsigned char* esc_d = nullptr;
  int esc_par = 0;
  SampleGridsV2Args win_whole{};       // the pair's whole-map plan (completion of the flagged maps)
  ReachBoxConst win_c{};               // the reach-box decision the completion records
  float* h_u = nullptr;        // pinned staging for the T x 2 result (+ one int: exchange status, + the reach statistic at
                               // 2T + 2; a window-first solve's record overwrites [2T, 2T + 8): sample_reach_host)
  // peer-memory exchange (p2p.cu): ONE allocation per planner so that one IPC handle describes it:
  // [ receive buffer (ws, N/ws, M/ws) | gather buffers 2 x (ws, 2T+2) | cost flags | partial flags | counter | status ]
  unsigned char* xbuf = nullptr;
  size_t x_gather = 0, x_flags_cost = 0, x_flags_part = 0, x_counter = 0, x_status = 0, x_bytes = 0;
  unsigned char* peer_x[P2P_MAX_PEERS] = {};
  bool peer_ipc[P2P_MAX_PEERS] = {};
  bool p2p_ready = false;
  uint32_t epoch_cost = 0, epoch_part = 0;
  unsigned long long p2p_timeout_ns = 20000000000ull;   // 20 s: start-up skew between ranks is seconds
  int num_ctas = 1, rows_per_cta = 1;
  b200mppi_tdm* lin = nullptr; b200mppi_tdm* ang = nullptr;
  b200mppi_params prm{};
  bool params_set = false;
  bool profiling = false;
  cudaEvent_t ev[8] = {};
  cudaEvent_t ev_reach = nullptr;   // after the reach read-back copy (stage_sample_tdms)
  float last_ms[B200MPPI_T_COUNT] = {};
  int64_t launches = 0;
  const b200mppi_loop* loop = nullptr;   // the open device loop of a batch holding this planner (b200mppi_batch_loop_open)
};

// The refusal of a call on a planner or batch whose device loop is open: the loop's kernels own its state until it closes
static int loop_busy(const char* fn) {
  return fail(B200MPPI_EINVAL, std::string(fn) + ": a device loop is open on its batch (b200mppi_loop_close it first)");
}

static int planner_check_ready(b200mppi_planner* p) {
  if (p->cfg.mode == B200MPPI_MODE_BAREBONE)
    return p->params_set ? B200MPPI_OK : fail(B200MPPI_ESTATE, "planner: params not set");
  if (!p->lin || !p->ang) return fail(B200MPPI_ESTATE, "planner: TDMs not set");
  if (!p->params_set) return fail(B200MPPI_ESTATE, "planner: params not set");
  if (!p->lin->pmf_set || !p->ang->pmf_set) return fail(B200MPPI_ESTATE, "planner: TDM PMF not initialised");
  if (!p->lin->masks_set) return fail(B200MPPI_ESTATE, "planner: obstacle/unknown maps not set on lin TDM");
  if (p->cfg.mode == B200MPPI_MODE_SPEED_MAP && !p->lin->risk_set)
    return fail(B200MPPI_ESTATE, "planner: risk traction map not set on lin TDM");
  if (p->lin->rows != p->ang->rows || p->lin->cols != p->ang->cols)
    return fail(B200MPPI_EINVAL, "planner: lin/ang TDM shapes differ");
  if (p->lin->mask_rows != p->lin->rows || p->lin->mask_cols != p->lin->cols)
    return fail(B200MPPI_EINVAL, "planner: mask shape differs from padded PMF shape");
  if (p->cfg.mode == B200MPPI_MODE_TDM && p->M_total > cvar_max_maps())
    return fail(B200MPPI_EINVAL, "planner: num_grid_samples exceeds the CVaR kernel's limit (16384)");
  return B200MPPI_OK;
}

static void fill_rollout_params(b200mppi_planner* p, RolloutParams& r) {
  const b200mppi_tdm* l = p->lin; const b200mppi_tdm* a = p->ang;
  if (l && a) {
    r.g.res = l->res; r.g.inv_res = 1.0f / l->res;
    r.g.xlo = l->pxl[0]; r.g.ylo = l->pyl[0];
    r.g.rows = l->rows; r.g.cols = l->cols;
    r.g.grid_rows = l->cfg.max_map_rows; r.g.grid_cols = l->cfg.max_map_cols; r.g.grid_pitch = l->pitch;
    r.g.mask_pitch = l->mask_pitch;
    r.lin_lo = l->bounds[0]; r.ang_lo = a->bounds[0];
    r.lin_ratio = 0.01 * (double)(float)(l->bounds[1] - l->bounds[0]);
    r.ang_ratio = 0.01 * (double)(float)(a->bounds[1] - a->bounds[0]);
  }
  const b200mppi_params& q = p->prm;
  r.dt = q.dt;
  for (int i = 0; i < 3; ++i) r.x0[i] = q.x0[i];
  r.xgoal[0] = q.xgoal[0]; r.xgoal[1] = q.xgoal[1];
  r.tol2 = q.goal_tolerance * q.goal_tolerance;
  r.v_post = q.v_post_rollout; r.lambda = q.lambda_weight;
  r.u_std[0] = q.u_std[0]; r.u_std[1] = q.u_std[1];
  r.vrange[0] = q.vrange[0]; r.vrange[1] = q.vrange[1];
  r.wrange[0] = q.wrange[0]; r.wrange[1] = q.wrange[1];
  r.obs_cost = q.obs_penalty; r.unk_cost = q.unknown_penalty; r.dist_weight = q.dist_weight;
  r.T = p->T; r.N = p->n_local; r.M = p->M;
}

static void fill_update_args(b200mppi_planner* p, UpdateArgs& u, const float* costs) {
  u.costs = costs ? costs : p->costs;
  u.noise = p->noise + (size_t)p->n_red_begin * p->T * 2;      // this rank's slice of the control sequences
  u.w_raw = p->w_raw;
  u.cta_partials = p->cta_partials; u.rank_partial = p->rank_partial; u.u_cur = p->u_cur;
  u.weights = p->weights; u.N = p->n_red; u.T = p->T; u.num_ctas = p->num_ctas;
  u.rows_per_cta = p->rows_per_cta; u.lambda = p->prm.lambda_weight;
  u.vrange[0] = p->prm.vrange[0]; u.vrange[1] = p->prm.vrange[1];
  u.wrange[0] = p->prm.wrange[0]; u.wrange[1] = p->prm.wrange[1];
}

static int planner_init(b200mppi_planner* p, const b200mppi_config* cfg) {
  p->cfg = *cfg;
  const int64_t N = cfg->num_control_rollouts;
  p->n_begin = (int)(N * cfg->rank / cfg->world_size);
  p->n_local = (int)(N * (cfg->rank + 1) / cfg->world_size) - p->n_begin;
  if (p->n_local < 1) return fail(B200MPPI_EINVAL, "planner_create: empty shard");
  p->T = cfg->num_steps;
  p->M_total = cfg->mode == B200MPPI_MODE_TDM ? cfg->num_grid_samples : 1;
  p->shard_maps = cfg->mode == B200MPPI_MODE_TDM && cfg->world_size > 1;
  if (p->shard_maps && (p->M_total % cfg->world_size != 0 || N % cfg->world_size != 0))
    return fail(B200MPPI_EINVAL, "planner_create: MODE_TDM sharding needs num_grid_samples and num_control_rollouts divisible by world_size");
  p->M = p->shard_maps ? p->M_total / cfg->world_size : p->M_total;
  p->n_roll = p->shard_maps ? (int)N : p->n_local;          // rollouts simulated by this rank
  p->n_red = p->n_local;                                    // rollouts reduced (CVaR, softmax) by this rank
  p->n_red_begin = p->shard_maps ? p->n_begin : 0;          // offset of that slice inside the noise buffer
  p->n_local = p->n_roll;                                   // buffers below are sized by the simulated count
  CU(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
  p->own_stream = true;
  const size_t nT = (size_t)p->n_local * p->T;
  CU(cudaMalloc(&p->noise, nT * 2 * sizeof(float)));
  // + 8 ints: the window-first record (sample_window_complete_kernel), copied back with u at the end of solve()
  CU(cudaMalloc(&p->u_cur, ((size_t)p->T * 2 + 8) * sizeof(float)));
  CU(cudaMalloc(&p->u_prev, (size_t)p->T * 2 * sizeof(float)));
  CU(cudaMalloc(&p->costs, (size_t)p->n_red * sizeof(float)));
  CU(cudaMalloc(&p->weights, (size_t)p->n_red * sizeof(float)));
  CU(cudaMalloc(&p->w_raw, (size_t)p->n_red * sizeof(float)));
  CU(cudaMalloc(&p->costs_nm, (size_t)p->n_local * p->M * sizeof(float)));
  if (p->shard_maps) CU(cudaMalloc(&p->costs_x, (size_t)p->n_local * p->M * sizeof(float)));
  p->npad = round_up(p->n_local, 32);
  CU(cudaMalloc(&p->noiseT, (size_t)(p->T + 1) * p->npad * 2 * sizeof(double)));      // + 1 row: unguarded prefetch
  CU(cudaMemsetAsync(p->noiseT, 0, (size_t)(p->T + 1) * p->npad * 2 * sizeof(double), p->stream));
  CU(cudaMalloc(&p->ctrl, (size_t)p->npad * sizeof(float)));
  p->use_win = getenv("B200MPPI_NO_WINDOW") == nullptr;
  CU(cudaMalloc(&p->reach_d, 256));
  CU(cudaMemsetAsync(p->reach_d, 0, 256, p->stream));
  CU(cudaMalloc(&p->upd_counter_d, 256));
  CU(cudaMemsetAsync(p->upd_counter_d, 0, 256, p->stream));
  if (const char* e = getenv("B200MPPI_SAMPLE_BOX")) {
    if (!strcmp(e, "off") || !strcmp(e, "0")) p->box_mode = 0;
    else if (!strcmp(e, "static")) p->box_mode = 1;
    else if (!strcmp(e, "window")) p->box_mode = 3;
    else p->box_mode = 2;                                  // "dynamic" (and, as before window-first, any other value)
  }
  if (const char* e = getenv("B200MPPI_SAMPLE_DISC")) p->disc = atoi(e) != 0;
  p->num_ctas = update_num_ctas(p->n_red);
  p->rows_per_cta = (p->n_red + p->num_ctas - 1) / p->num_ctas;
  p->num_ctas = (p->n_red + p->rows_per_cta - 1) / p->rows_per_cta;
  CU(cudaMalloc(&p->cta_partials, (size_t)p->num_ctas * (2 * p->T + 2) * sizeof(float)));
  CU(cudaMalloc(&p->rank_partial, (size_t)(2 * p->T + 2) * sizeof(float)));
  const int V = cfg->num_vis_state_rollouts < 1 ? 1 : cfg->num_vis_state_rollouts;
  CU(cudaMalloc(&p->state_rollout, (size_t)V * (p->T + 1) * 3 * sizeof(float)));
  CU(cudaMemsetAsync(p->noise, 0, nT * 2 * sizeof(float), p->stream));
  CU(cudaMemsetAsync(p->u_cur, 0, (size_t)p->T * 2 * sizeof(float), p->stream));
  CU(cudaMemsetAsync(p->u_prev, 0, (size_t)p->T * 2 * sizeof(float), p->stream));
  CU(cudaMemsetAsync(p->costs, 0, (size_t)p->n_red * sizeof(float), p->stream));
  CU(cudaMemsetAsync(p->weights, 0, (size_t)p->n_red * sizeof(float), p->stream));
  CU(cudaMemsetAsync(p->state_rollout, 0, (size_t)V * (p->T + 1) * 3 * sizeof(float), p->stream));
  CU(cudaMallocHost(&p->h_u, ((size_t)p->T * 2 + 4 + 8) * sizeof(float)));
  // generators n_global*T + t of this shard (mppi.py:118,1367)
  std::vector<uint64_t> h(nT * 2);
  create_xoroshiro_states(h.data(), p->shard_maps ? 0 : (int64_t)p->n_begin * p->T, (int64_t)nT, cfg->seed);
  CU(cudaMalloc(&p->states, h.size() * sizeof(uint64_t)));
  CU(cudaMemcpyAsync(p->states, h.data(), h.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, p->stream));
  for (auto& e : p->ev) CU(cudaEventCreate(&e));
  CU(cudaEventCreateWithFlags(&p->ev_reach, cudaEventDisableTiming));
  CU(cudaStreamSynchronize(p->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_destroy(b200mppi_planner* p);

extern "C" int b200mppi_planner_create(const b200mppi_config* cfg, b200mppi_planner** out) {
  if (!cfg || !out) return fail(B200MPPI_EINVAL, "planner_create: null argument");
  if (cfg->num_steps < 1 || cfg->num_steps > 1024 || cfg->num_control_rollouts < 1 || cfg->world_size < 1 ||
      cfg->rank < 0 || cfg->rank >= cfg->world_size || cfg->num_grid_samples < 1)
    return fail(B200MPPI_EINVAL, "planner_create: bad sizes (1 <= num_steps <= 1024)");
  if (b200mppi_device_count() < 1) return fail(B200MPPI_ECUDA, "planner_create: no CUDA device (no CPU fallback)");
  CU(cudaSetDevice(cfg->device));
  b200mppi_planner* p = new b200mppi_planner();
  const int rc = planner_init(p, cfg);
  if (rc) {                                   // release whatever was allocated before the failure
    const std::string keep = g_err;
    b200mppi_planner_destroy(p);
    g_err = keep;
    return rc;
  }
  *out = p;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_destroy(b200mppi_planner* p) {
  if (!p) return B200MPPI_OK;
  if (p->loop) return loop_busy("planner_destroy");
  cudaSetDevice(p->cfg.device);
  if (p->stream) cudaStreamSynchronize(p->stream);
  cudaFree(p->noise); cudaFree(p->u_cur); cudaFree(p->u_prev); cudaFree(p->costs); cudaFree(p->weights);
  cudaFree(p->w_raw); cudaFree(p->costs_nm); cudaFree(p->cta_partials); cudaFree(p->rank_partial);
  cudaFree(p->state_rollout); cudaFree(p->states); cudaFree(p->noiseT); cudaFree(p->ctrl); cudaFree(p->costs_x);
  cudaFree(p->obstacles); cudaFree(p->reach_d); cudaFree(p->upd_counter_d); cudaFree(p->esc_d);
  for (int s = 0; s < P2P_MAX_PEERS; ++s)
    if (p->peer_ipc[s] && p->peer_x[s]) cudaIpcCloseMemHandle(p->peer_x[s]);
  cudaFree(p->xbuf);
  if (p->h_u) cudaFreeHost(p->h_u);
  for (auto& e : p->ev) if (e) cudaEventDestroy(e);
  if (p->ev_reach) cudaEventDestroy(p->ev_reach);
  if (p->own_stream && p->stream) cudaStreamDestroy(p->stream);
  delete p;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_set_stream(b200mppi_planner* p, void* s) {
  if (p && p->loop) return loop_busy("planner_set_stream");
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  if (p->own_stream && p->stream) { cudaStreamSynchronize(p->stream); cudaStreamDestroy(p->stream); }
  p->stream = (cudaStream_t)s;
  p->own_stream = false;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_set_tdms(b200mppi_planner* p, b200mppi_tdm* lin, b200mppi_tdm* ang) {
  if (p && p->loop) return loop_busy("planner_set_tdms");
  if (!p || !lin || !ang) return fail(B200MPPI_EINVAL, "set_tdms: null argument");
  if (lin->cfg.device != p->cfg.device || ang->cfg.device != p->cfg.device)
    return fail(B200MPPI_EINVAL, "set_tdms: TDMs live on another device");
  if (lin->num_maps != ang->num_maps || lin->cfg.max_map_rows != ang->cfg.max_map_rows ||
      lin->cfg.max_map_cols != ang->cfg.max_map_cols)
    return fail(B200MPPI_EINVAL, "set_tdms: lin/ang allocation shapes differ");
  if (p->cfg.mode == B200MPPI_MODE_TDM && lin->num_maps < p->M)
    return fail(B200MPPI_EINVAL, "set_tdms: TDM holds fewer sampled maps than the planner's num_grid_samples");
  if (p->shard_maps && (lin->cfg.rank != p->cfg.rank || lin->cfg.world_size != p->cfg.world_size ||
                        ang->cfg.rank != p->cfg.rank || ang->cfg.world_size != p->cfg.world_size))
    return fail(B200MPPI_EINVAL, "set_tdms: the TDMs' rank / world_size differ from the planner's (each rank samples its own maps)");
  p->lin = lin; p->ang = ang;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_set_params(b200mppi_planner* p, const b200mppi_params* q) {
  if (p && p->loop) return loop_busy("planner_set_params");
  if (!p || !q) return fail(B200MPPI_EINVAL, "set_params: null argument");
  if (!(q->dt > 0) || q->num_opt < 0) return fail(B200MPPI_EINVAL, "set_params: bad dt/num_opt");
  p->prm = *q;
  p->params_set = true;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_set_u(b200mppi_planner* p, const float* u) {
  if (p && p->loop) return loop_busy("planner_set_u");
  if (!p || !u) return fail(B200MPPI_EINVAL, "set_u: null argument");
  CU(cudaSetDevice(p->cfg.device));
  std::memcpy(p->h_u, u, (size_t)p->T * 2 * sizeof(float));
  CU(cudaMemcpyAsync(p->u_cur, p->h_u, (size_t)p->T * 2 * sizeof(float), cudaMemcpyHostToDevice, p->stream));
  CU(cudaStreamSynchronize(p->stream));
  p->prepared = false;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_get_u(b200mppi_planner* p, float* u) {
  if (p && p->loop) return loop_busy("planner_get_u");
  if (!p || !u) return fail(B200MPPI_EINVAL, "get_u: null argument");
  CU(cudaSetDevice(p->cfg.device));
  CU(cudaMemcpyAsync(p->h_u, p->u_cur, (size_t)p->T * 2 * sizeof(float), cudaMemcpyDeviceToHost, p->stream));
  CU(cudaStreamSynchronize(p->stream));
  std::memcpy(u, p->h_u, (size_t)p->T * 2 * sizeof(float));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_shift_u(b200mppi_planner* p, int32_t shifts) {
  if (p && p->loop) return loop_busy("planner_shift_u");
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  CU(cudaSetDevice(p->cfg.device));
  launch_shift_u(p->u_cur, p->T, shifts, p->stream);
  p->prepared = false;
  p->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

// ---- stages
static bool planner_uses_window(const b200mppi_planner* p) {
  if (p->cfg.mode != B200MPPI_MODE_TDM || !p->use_win) return false;
  int WW, WH; size_t smem;
  rollout_win_geometry(p->T, &WW, &WH, &smem);
  return smem <= 232448;
}

// control noise, and (windowed stochastic rollouts) the transposed clipped controls + per-n control cost + the
// reach statistic max_n sum_t |v| of this iteration
static int stage_noise(b200mppi_planner* p) {
  p->prepared = false;
  if (planner_uses_window(p)) {             // ONE launch: noise in both layouts, control costs, reach statistic
    p->reach_slot ^= 1;
    launch_noise_prepare(p->states, p->noise, p->u_cur, p->noiseT, p->ctrl, p->reach_d, p->reach_slot, p->n_local, p->T,
                         p->npad, p->prm.lambda_weight, p->prm.u_std[0], p->prm.u_std[1], p->prm.vrange, p->prm.wrange,
                         p->stream);
    p->launches++;
    CHECK_LAUNCH();
    p->prepared = true;
    p->reach_valid = true;
    return B200MPPI_OK;
  }
  launch_sample_noise(p->states, p->noise, p->n_local, p->T, p->prm.u_std[0], p->prm.u_std[1], nullptr, p->stream);
  p->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

// tensor maps of the windowed rollout: encoded once per (buffers, geometry) -- the window origin is a launch coordinate.
// The allocation shapes are part of the key: a TDM pair of another shape may be handed the freed addresses of the last.
static bool planner_tensor_maps(b200mppi_planner* p, int WW, int WH) {
  const b200mppi_tdm* l = p->lin; const b200mppi_tdm* g = p->ang;
  const void* key[8] = {l->grid, g->grid, l->obstacle, l->unknown,
                        (const void*)(((size_t)l->mask_rows << 40) ^ ((size_t)l->mask_cols << 20) ^ (size_t)l->mask_pitch),
                        (const void*)(((size_t)WW << 40) ^ ((size_t)WH << 20) ^ (size_t)l->num_maps),
                        (const void*)(((size_t)l->cfg.max_map_rows << 40) ^ ((size_t)l->cfg.max_map_cols << 20) ^ (size_t)l->pitch),
                        (const void*)(((size_t)g->cfg.max_map_rows << 40) ^ ((size_t)g->cfg.max_map_cols << 20) ^ (size_t)g->pitch)};
  if (!std::memcmp(key, p->tmap_key, sizeof(key))) return true;
  const bool ok =
      make_u8_tensor_map(p->tmaps[0], l->grid, 3, l->cfg.max_map_cols, l->cfg.max_map_rows, l->num_maps, l->pitch, WW, WH) &&
      make_u8_tensor_map(p->tmaps[1], g->grid, 3, g->cfg.max_map_cols, g->cfg.max_map_rows, g->num_maps, g->pitch, WW, WH) &&
      make_u8_tensor_map(p->tmaps[2], l->obstacle, 2, l->mask_cols, l->mask_rows, 1, l->mask_pitch, WW, WH) &&
      make_u8_tensor_map(p->tmaps[3], l->unknown, 2, l->mask_cols, l->mask_rows, 1, l->mask_pitch, WW, WH);
  if (ok) std::memcpy(p->tmap_key, key, sizeof(key)); else std::memset(p->tmap_key, 0, sizeof(key));
  return ok;
}

// Per-(m, n) costs of this rank's rollouts, map-major (kernels.h, CostDst).
//   one rank                     : costs_nm = (M, N)
//   maps sharded, staged exchange: costs_nm = (ws, M/ws, N/ws) -- block d = what rank d will reduce (all-to-all send buffer)
//   maps sharded, peer memory    : block d = rows [rank*M/ws, ...) of rank d's receive buffer (ws*M/ws, N/ws)   [direct]
static void fill_cost_dst(b200mppi_planner* p, CostDst& d, bool direct) {
  d = CostDst{};
  if (!p->shard_maps) {
    d.base[0] = p->costs_nm; d.n_per = p->n_local > 0 ? p->n_local : 1; d.ld = p->n_local; d.row0 = 0;
    return;
  }
  const int ws = p->cfg.world_size;
  d.n_per = p->n_red; d.ld = p->n_red;
  d.row0 = direct ? p->cfg.rank * p->M : 0;
  for (int r = 0; r < ws; ++r)
    d.base[r] = direct ? (float*)p->peer_x[r] : p->costs_nm + (size_t)r * p->M * p->n_red;
}

static void fill_rollout_args(b200mppi_planner* p, RolloutArgs& a) {
  a = RolloutArgs{};
  fill_rollout_params(p, a.p);
  a.mode = p->cfg.mode;
  if (p->cfg.mode != B200MPPI_MODE_BAREBONE) {
    a.lin_grid = p->lin->grid; a.ang_grid = p->ang->grid;
    a.obstacle = p->lin->obstacle; a.unknown = p->lin->unknown; a.risk = p->lin->risk;
  }
  a.obstacles = p->obstacles; a.num_obstacles = p->num_obstacles;
  a.noise = p->noise; a.u_cur = p->u_cur; a.costs = p->costs;
  fill_cost_dst(p, a.dst, false);
}

// The planner's part of the windowed rollout's arguments: window (centred on the robot's cell) and buffers.
// win_origin (kernels.h), shared with the plant step of stochastic trials, takes the six window fields from WW on
static_assert(offsetof(RolloutWinArgs, WH) == offsetof(RolloutWinArgs, WW) + 4 &&
              offsetof(RolloutWinArgs, wx0) == offsetof(RolloutWinArgs, WW) + 8 &&
              offsetof(RolloutWinArgs, wy0) == offsetof(RolloutWinArgs, WW) + 12 &&
              offsetof(RolloutWinArgs, ww) == offsetof(RolloutWinArgs, WW) + 16 &&
              offsetof(RolloutWinArgs, wh) == offsetof(RolloutWinArgs, WW) + 20, "RolloutWinArgs window fields");

static void fill_win_args(const b200mppi_planner* p, int WW, int WH, RolloutWinArgs& w) {
  const b200mppi_tdm* l = p->lin; const b200mppi_tdm* g = p->ang;
  w.WW = WW; w.WH = WH;
  // TMA: the inner (x) start coordinate is kept 16-byte aligned for 1-byte elements (an unaligned c0 faulted
  // with 'illegal instruction' when probed)
  win_origin(p->prm.x0[0], p->prm.x0[1], l->pxl[0], l->pyl[0], l->res, l->cols, l->rows, &w.WW);
  w.npad = p->npad;
  w.masks01 = l->masks01 ? 1 : 0;
  w.lin_grid = l->grid; w.ang_grid = g->grid; w.obstacle = l->obstacle; w.unknown = l->unknown;
  w.noiseT = p->noiseT; w.ctrl = p->ctrl; w.u_cur = p->u_cur;
}

static void last_box_whole_map(b200mppi_planner* p);

static int stage_rollout(b200mppi_planner* p) {
  RolloutArgs a;
  fill_rollout_args(p, a);
  p->pushed_direct = false;
  bool done = false;
  if (planner_uses_window(p)) {
    // stochastic mode: TMA-staged map windows (rollout_win.cu); window centred on the robot's cell
    int WW, WH; size_t smem;
    rollout_win_geometry(p->T, &WW, &WH, &smem);
    if (planner_tensor_maps(p, WW, WH)) {
      if (!p->prepared) {                       // noise came from outside (set_noise): derive the controls now
        launch_prepare_rollout(p->noise, p->u_cur, p->noiseT, p->ctrl, nullptr, p->n_local, p->T, p->npad,
                               p->prm.lambda_weight, p->prm.u_std[0], p->prm.u_std[1], p->prm.vrange, p->prm.wrange, p->stream);
        p->launches++;
        CHECK_LAUNCH();
      }
      p->prepared = false;                      // u_cur changes with the update that follows
      RolloutWinArgs w{};
      w.p = a.p;
      fill_win_args(p, WW, WH, w);
      // sharded + peers connected: the all-to-all is this kernel's epilogue (stores into the peers, then the flags)
      const bool direct = p->shard_maps && p->p2p_ready;
      fill_cost_dst(p, w.dst, direct);
      if (direct) {
        const int ws = p->cfg.world_size;
        w.sig.ws = ws; w.sig.rank = p->cfg.rank;
        w.sig.counter = (unsigned*)(p->xbuf + p->x_counter);
        w.sig.epoch = ++p->epoch_cost;
        for (int r = 0; r < ws; ++r) w.sig.peer_flags[r] = (uint32_t*)(p->peer_x[r] + p->x_flags_cost);
      }
      if (p->win_pending) w.esc = p->esc_d + (size_t)p->esc_par * p->M;
      CU(launch_rollout_win(w, p->tmaps[0], p->tmaps[1], p->tmaps[2], p->tmaps[3], p->stream));
      p->launches++;
      p->pushed_direct = direct;
      done = true;
      if (p->win_pending) {
        p->win_pending = false;
        // the flagged maps: completed from the pre-call states (the commit swapped them into states_alt), then rerun
        SampleGridsV2Args c = p->win_whole;
        c.t[0].states = p->lin->states_alt;
        launch_sample_window_complete(c, p->win_c, p->prm.x0[0], p->prm.x0[1], p->reach_d + p->reach_slot,
                                      (int*)(p->u_cur + (size_t)p->T * 2), w.esc,
                                      p->esc_d + (size_t)(p->esc_par ^ 1) * p->M, p->stream);
        CHECK_LAUNCH();
        w.redo = 1;
        CU(launch_rollout_win(w, p->tmaps[0], p->tmaps[1], p->tmaps[2], p->tmaps[3], p->stream));
        p->launches += 2;
        p->esc_par ^= 1;
      }
    }
  }
  if (!done && p->win_pending) {                 // no windowed launch after all: the generic kernel needs whole maps
    p->win_pending = p->win_used = false;          // no window-first record: sample_box() reports the whole maps
    last_box_whole_map(p);
    int rc;
    if ((rc = tdm_complete_grid(p->lin, p->stream)) || (rc = tdm_complete_grid(p->ang, p->stream))) return rc;
  }
  if (!done) {
    launch_rollout(a, p->stream);
    p->launches++;
    CHECK_LAUNCH();
  }
  if (p->profiling) cudaEventRecord(p->ev[3], p->stream);
  if (p->cfg.mode == B200MPPI_MODE_TDM && !p->shard_maps) {
    launch_cvar(p->costs_nm, p->costs, p->n_local, p->n_local, p->M, p->prm.cvar_alpha, FlagWait{}, p->stream);
    p->launches++;
    CHECK_LAUNCH();
  }
  return B200MPPI_OK;
}

static int after_u_update(b200mppi_planner* p) {
  p->prepared = false;                        // u_cur moved
  if (p->cfg.mode != B200MPPI_MODE_TDM)   // self.u_prev_d = self.u_cur_d (alias, mppi.py:292,362)
    CU(cudaMemcpyAsync(p->u_prev, p->u_cur, (size_t)p->T * 2 * sizeof(float), cudaMemcpyDeviceToDevice, p->stream));
  return B200MPPI_OK;
}

// CTA partials of this rank's rollouts; the kernel's last CTA merges them into the rank partial and then
//   UPD_TAIL_APPLY (one rank)      applies the update: the whole update is this one launch,
//   UPD_TAIL_BCAST (peers connected) pushes the partial to every peer and raises the flags,
//   UPD_TAIL_RANK                  leaves it in rank_partial for a staged (collective-library) all-gather.
static int stage_update_partial(b200mppi_planner* p, int tail) {
  UpdateArgs u{};
  fill_update_args(p, u, nullptr);
  UpdateTail tl{};
  tl.counter = p->upd_counter_d;
  tl.mode = tail;
  p->bcast_done = false;
  if (tail == UPD_TAIL_BCAST) {
    const int ws = p->cfg.world_size;
    tl.ws = ws; tl.rank = p->cfg.rank;
    tl.epoch = ++p->epoch_part;
    const size_t parity_off = (size_t)(tl.epoch & 1u) * ws * (2 * p->T + 2) * sizeof(float);
    for (int s = 0; s < ws; ++s) {
      tl.peer_gather[s] = (float*)(p->peer_x[s] + p->x_gather + parity_off);
      tl.peer_flags[s] = (uint32_t*)(p->peer_x[s] + p->x_flags_part);
    }
    p->bcast_done = true;
  }
  launch_update_partial(u, tl, p->stream);
  p->launches++;
  CHECK_LAUNCH();
  if (tail == UPD_TAIL_APPLY) return after_u_update(p);
  return B200MPPI_OK;
}

static int stage_update_finish(b200mppi_planner* p, const float* gathered, int count, const FlagWait& fw) {
  UpdateArgs u{};
  fill_update_args(p, u, nullptr);
  launch_update_finish(u, gathered, count, fw, p->stream);
  p->launches++;
  CHECK_LAUNCH();
  return after_u_update(p);
}

extern "C" int b200mppi_planner_set_obstacles(b200mppi_planner* p, const float* xy, const float* rad, int32_t count) {
  if (p && p->loop) return loop_busy("planner_set_obstacles");
  if (!p || count < 0 || (count > 0 && (!xy || !rad))) return fail(B200MPPI_EINVAL, "set_obstacles: bad argument");
  CU(cudaSetDevice(p->cfg.device));
  if (count > p->obstacles_cap) {
    cudaFree(p->obstacles); p->obstacles = nullptr;
    CU(cudaMalloc(&p->obstacles, (size_t)count * 3 * sizeof(float)));
    p->obstacles_cap = count;
  }
  if (count > 0) {
    std::vector<float> h((size_t)count * 3);
    for (int k = 0; k < count; ++k) { h[3 * k] = xy[2 * k]; h[3 * k + 1] = xy[2 * k + 1]; h[3 * k + 2] = rad[k]; }
    CU(cudaMemcpyAsync(p->obstacles, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice, p->stream));
    CU(cudaStreamSynchronize(p->stream));
  }
  p->num_obstacles = count;
  return B200MPPI_OK;
}

// The constants of a planner's reach-box decision (reach_box_decide, kernels.h) for the plan of its pair: the box is
// sized from the speed limit or, when the maps are sampled once for ONE set of controls (num_opt = 1, box_mode 2), from
// the reach statistic of the controls actually drawn (reach_d, reduced by the prepare kernel).
static void fill_reach_const(const b200mppi_planner* p, const SamplePlan& pl, ReachBoxConst* c) {
  const b200mppi_tdm* l = p->lin;
  const b200mppi_params& q = p->prm;
  *c = ReachBoxConst{};
  c->mode = (p->box_mode == 0 || !planner_uses_window(p)) ? 0 : (p->box_mode >= 2 && q.num_opt == 1) ? 2 : 1;
  c->disc = p->disc ? 1 : 0;
  c->T = p->T;
  c->vr0 = q.vrange[0]; c->vr1 = q.vrange[1]; c->dt = q.dt; c->tr_abs_max = l->tr_abs_max;
  c->res = l->res; c->pxl = l->pxl[0]; c->pyl = l->pyl[0]; c->rows = l->rows; c->cols = l->cols;
  const SampleGridsV2Args& a = pl.a[0];
  c->nt = !pl.v2[0] ? 0 : pl.fused ? 2 : 1;
  c->tx = a.tx; c->ty = a.ty; c->num_maps = a.num_maps; c->bpad0 = a.t[0].bpad; c->bpad1 = a.t[1].bpad;
}

// A solve's map sampling in three steps, shared by solve() (stage_sample_tdms) and the stochastic batch:
//   plan_sampling with sample_alpha; then, if sample_reads_reach, the 4-byte reach statistic is copied to the host
//   (sample_reach_host) behind an event, a fused pair's state advance is queued (it does not depend on the box: it runs
//   while the host wakes up, and should the sampling take whole maps after all, that launch stores the very same states
//   again), and the host waits for the event; finally sample_finish sizes the box and launches the sampler.
// det / speed-map solves call sample_grids() with the default alpha_dyn = 1.0 (mppi.py:248-249,322-323)
static double sample_alpha(const b200mppi_planner* p) {
  return p->cfg.mode == B200MPPI_MODE_TDM ? p->prm.alpha_dyn : 1.0;
}

// a box from this solve's own controls: the host waits for their reach statistic only (an event, not the stream)
static bool sample_reads_reach(const b200mppi_planner* p) {
  return p->box_mode >= 2 && p->prm.num_opt == 1 && p->prepared && p->reach_valid && planner_uses_window(p);
}

// h_u[2T + 2]: the reach statistic read back by a reach-box solve.  A window-first solve never reads it back; its record
// (8 ints behind u in u_cur, copied with u) occupies h_u[2T .. 2T + 8), this slot and the exchange status included.
static float* sample_reach_host(b200mppi_planner* p) { return p->h_u + (size_t)p->T * 2 + 2; }

// The sampling of the pair of the n planners ps (a TDM group of a batch; n = 1: one planner's solve), each deciding its
// box from reach[j] (the read-back statistic or null: static box), the pair sampling their hull (reach_box_hull); every
// member's sample_box() reports the box actually sampled.  advanced: a fused pair's state advance is already queued.
static int sample_finish_group(b200mppi_planner* const* ps, const float* const* reach, int n, SamplePlan& plan,
                               bool advanced, cudaStream_t st, int64_t* launches) {
  ReachBoxConst c;
  ReachBox box;
  for (int j = 0; j < n; ++j) {
    const b200mppi_planner* p = ps[j];
    fill_reach_const(p, plan, &c);
    ReachBox m;
    reach_box_decide(c, p->prm.x0[0], p->prm.x0[1], reach[j], &m);
    reach_box_hull_add(&box, j, m);
  }
  const int how = reach_box_hull_close(c, n, &box);
  if (box.geo) plan_box(&plan, box);                      // an unfused pair's TDM 1 may take the box on its own
  const int rc = plan_launch(plan, advanced, st, launches);
  const bool used = plan.boxed[0];                        // the box may not fit the sampler's launch: whole maps
  for (int j = 0; j < n; ++j) {
    b200mppi_planner* p = ps[j];
    p->last_box[0] = used ? how : 0;
    p->last_box[1] = used ? box.row_lo : 0; p->last_box[2] = used ? box.row_hi : p->lin->rows;
    p->last_box[3] = used ? box.col_lo : 0; p->last_box[4] = used ? box.col_hi : p->lin->cols;
  }
  return rc;
}

static int sample_finish(b200mppi_planner* p, SamplePlan& plan, const float* reach, bool advanced, cudaStream_t st,
                         int64_t* launches) {
  return sample_finish_group(&p, &reach, 1, plan, advanced, st, launches);
}

// Window-first sampling: a single-rank solve() of one iteration with the windowed rollout samples only the cells
// around the window the rollout kernel stages (win_origin) -- known from x0 alone, so no host wait -- plus a ring of
// WIN_SAMPLE_RING cells.  The rollout flags the maps whose lanes read outside that rectangle (an escape); a completion
// launch then re-walks those maps whole and records the reach box the solve would have sampled, and a redo launch
// reruns their rollouts (stage_rollout).  Costs, u and every state are those of whole-map sampling.  Applies to a
// fused pair whose maps are larger than the window and whose whole-map and windowed launches fit the staged sampler;
// otherwise the solve samples its reach box.
static bool planner_window_first(const b200mppi_planner* p, const SamplePlan& plan) {
  if (p->box_mode != 3 || p->cfg.world_size != 1 || p->shard_maps || p->prm.num_opt != 1 || !p->prepared ||
      !planner_uses_window(p) || !plan.fused || !plan.v2[0])
    return false;
  int WW, WH; size_t smem;
  rollout_win_geometry(p->T, &WW, &WH, &smem);
  return p->lin->cols > WW || p->lin->rows > WH;
}

static int stage_sample_window(b200mppi_planner* p, SamplePlan& plan, bool* used) {
  *used = false;
  const b200mppi_tdm* l = p->lin;
  RolloutWinArgs w{};
  int WW, WH; size_t smem;
  rollout_win_geometry(p->T, &WW, &WH, &smem);
  w.WW = WW; w.WH = WH;
  win_origin(p->prm.x0[0], p->prm.x0[1], l->pxl[0], l->pyl[0], l->res, l->cols, l->rows, &w.WW);
  const int R = WIN_SAMPLE_RING;
  ReachBox b{};
  b.geo = 1; b.how = 2;
  b.row_lo = std::max(w.wy0 - R, 0); b.row_hi = std::min(w.wy0 + w.wh + R, l->rows);
  b.col_lo = std::max(w.wx0 - R, 0); b.col_hi = std::min(w.wx0 + w.ww + R, l->cols);
  const SampleGridsV2Args whole = plan.a[0];
  plan_box(&plan, b);
  if (!plan.boxed[0]) return B200MPPI_OK;                 // the windowed launch does not fit: sample the reach box
  if (!p->esc_d) {
    CU(cudaMalloc(&p->esc_d, (size_t)2 * p->M));
    CU(cudaMemsetAsync(p->esc_d, 0, (size_t)2 * p->M, p->stream));
  }
  p->win_whole = whole;
  p->win_whole.write_states = 0;
  fill_reach_const(p, plan, &p->win_c);
  p->win_rect[0] = b.row_lo; p->win_rect[1] = b.row_hi; p->win_rect[2] = b.col_lo; p->win_rect[3] = b.col_hi;
  p->win_used = p->win_pending = *used = true;
  return plan_launch(plan, false, p->stream, &p->launches);
}

static int stage_sample_tdms(b200mppi_planner* p) {
  if (p->cfg.mode == B200MPPI_MODE_BAREBONE) return B200MPPI_OK;      // no maps
  SamplePlan plan;
  int rc = plan_sampling(p->lin, p->ang, sample_alpha(p), p->stream, &plan);
  if (rc) return rc;
  p->win_used = p->win_pending = false;
  if (planner_window_first(p, plan)) {
    bool used;
    if ((rc = stage_sample_window(p, plan, &used)) || used) return rc;
    if ((rc = plan_sampling(p->lin, p->ang, sample_alpha(p), p->stream, &plan))) return rc;
  }
  const float* reach = nullptr;
  bool advanced = false;
  if (sample_reads_reach(p)) {
    float* h = sample_reach_host(p);
    CU(cudaMemcpyAsync(h, p->reach_d + p->reach_slot, sizeof(float), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaEventRecord(p->ev_reach, p->stream));
    if (plan.fused) {
      launch_plan_advance(plan, 0, p->stream);
      CHECK_LAUNCH();
      p->launches++;
      advanced = true;
    }
    CU(cudaEventSynchronize(p->ev_reach));
    reach = h;
  }
  return sample_finish(p, plan, reach, advanced, p->stream, &p->launches);
}

static void collect_timings(b200mppi_planner* p) {
  // ev: 0 solve start, 6 iteration start, 1 after noise (+ controls), 7 before / 2 after map sampling (first iteration),
  //     3 after rollout, 4 after cvar, 5 after update (last iteration)
  if (!p->profiling) return;
  float ms = 0;
  auto dt = [&](int a, int b) { ms = 0; cudaEventElapsedTime(&ms, p->ev[a], p->ev[b]); return ms; };
  const bool one = p->prm.num_opt <= 1;                   // the sampling of a multi-iteration solve precedes ev[6]
  p->last_ms[B200MPPI_T_SAMPLE_GRIDS] = dt(7, 2);
  p->last_ms[B200MPPI_T_NOISE] = dt(6, 1);
  p->last_ms[B200MPPI_T_ROLLOUT] = dt(one ? 2 : 1, 3);
  p->last_ms[B200MPPI_T_CVAR] = dt(3, 4);
  p->last_ms[B200MPPI_T_UPDATE] = dt(4, 5);
  p->last_ms[B200MPPI_T_TOTAL] = dt(0, 5);
}

// one optimisation iteration up to the per-(n,m) costs: noise (+ controls) -> [first iteration: maps] -> rollouts.
// The noise comes first because the map sampler is sized by the reach of the controls it yields (planner_reach_box).
static int iteration_rollouts(b200mppi_planner* p, bool first) {
  int rc;
  if (p->profiling) cudaEventRecord(p->ev[6], p->stream);
  if ((rc = stage_noise(p))) return rc;
  if (p->profiling) cudaEventRecord(p->ev[1], p->stream);
  if (first) {
    if (p->profiling) cudaEventRecord(p->ev[7], p->stream);
    if ((rc = stage_sample_tdms(p))) return rc;
    if (p->profiling) cudaEventRecord(p->ev[2], p->stream);
  }
  if ((rc = stage_rollout(p))) return rc;
  if (p->profiling) cudaEventRecord(p->ev[4], p->stream);
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_solve(b200mppi_planner* p, float* u_out) {
  if (p && p->loop) return loop_busy("planner_solve");
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  if (p->cfg.world_size != 1) return fail(B200MPPI_ESTATE, "solve: world_size > 1, use solve_local/solve_finish");
  int rc = planner_check_ready(p);
  if (rc) return rc;
  CU(cudaSetDevice(p->cfg.device));
  if (p->profiling) cudaEventRecord(p->ev[0], p->stream);
  if (p->prm.num_opt <= 0 && (rc = stage_sample_tdms(p))) return rc;     // the reference samples before its loop
  for (int k = 0; k < p->prm.num_opt; ++k) {
    if ((rc = iteration_rollouts(p, k == 0))) return rc;
    if ((rc = stage_update_partial(p, UPD_TAIL_APPLY))) return rc;
    if (p->profiling) cudaEventRecord(p->ev[5], p->stream);
  }
  // a window-first solve: its record (sample_window_complete_kernel) sits behind u and comes back in the same copy
  const bool win = p->win_used && p->prm.num_opt > 0;
  CU(cudaMemcpyAsync(p->h_u, p->u_cur, ((size_t)p->T * 2 + (win ? 8 : 0)) * sizeof(float), cudaMemcpyDeviceToHost,
                     p->stream));
  CU(cudaStreamSynchronize(p->stream));
  if (u_out) std::memcpy(u_out, p->h_u, (size_t)p->T * 2 * sizeof(float));
  if (win) {
    const int32_t* rec = reinterpret_cast<const int32_t*>(p->h_u + (size_t)p->T * 2);
    for (int i = 0; i < 5; ++i) p->last_box[i] = rec[i];
    p->win_flagged = rec[5];
  }
  if (p->prm.num_opt > 0) collect_timings(p);
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_solve_local(b200mppi_planner* p, int32_t first_iteration) {
  if (p && p->loop) return loop_busy("planner_solve_local");
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  int rc = planner_check_ready(p);
  if (rc) return rc;
  CU(cudaSetDevice(p->cfg.device));
  if (p->profiling && first_iteration) cudaEventRecord(p->ev[0], p->stream);
  if ((rc = iteration_rollouts(p, first_iteration != 0))) return rc;
  if (p->shard_maps) return B200MPPI_OK;                     // the costs go through the all-to-all first
  if ((rc = stage_update_partial(p, p->p2p_ready ? UPD_TAIL_BCAST : UPD_TAIL_RANK))) return rc;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_solve_reduce(b200mppi_planner* p, const float* exchanged_dev) {
  if (p && p->loop) return loop_busy("planner_solve_reduce");
  if (!p || !exchanged_dev) return fail(B200MPPI_EINVAL, "solve_reduce: null argument");
  if (!p->shard_maps) return fail(B200MPPI_ESTATE, "solve_reduce: only for MODE_TDM with world_size > 1");
  CU(cudaSetDevice(p->cfg.device));
  // exchanged_dev: (world_size, M_local, N/ws) -- block g holds rank g's maps for THIS rank's control sequences,
  // i.e. the map-major (M_total, N/ws) array of a one-rank solve restricted to them
  launch_cvar(exchanged_dev, p->costs, p->n_red, p->n_red, p->M_total, p->prm.cvar_alpha, FlagWait{}, p->stream);
  p->launches++;
  CHECK_LAUNCH();
  if (p->profiling) cudaEventRecord(p->ev[4], p->stream);
  return stage_update_partial(p, UPD_TAIL_RANK);
}

extern "C" int b200mppi_planner_solve_finish(b200mppi_planner* p, const float* gathered_dev, float* u_out) {
  if (p && p->loop) return loop_busy("planner_solve_finish");
  if (!p || !gathered_dev) return fail(B200MPPI_EINVAL, "solve_finish: null argument");
  if (p->cfg.world_size > 512) return fail(B200MPPI_EINVAL, "solve_finish: world_size > 512");
  CU(cudaSetDevice(p->cfg.device));
  int rc = stage_update_finish(p, gathered_dev, p->cfg.world_size, FlagWait{});
  if (rc) return rc;
  if (p->profiling) cudaEventRecord(p->ev[5], p->stream);
  if (u_out) {
    CU(cudaMemcpyAsync(p->h_u, p->u_cur, (size_t)p->T * 2 * sizeof(float), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    std::memcpy(u_out, p->h_u, (size_t)p->T * 2 * sizeof(float));
    collect_timings(p);
  }
  return B200MPPI_OK;
}

// ---------------------------------------------------------------------------------------------
// Peer-memory exchange (p2p.cu): the sharded solve without NCCL on the data path.
static int p2p_alloc(b200mppi_planner* p) {
  if (p->xbuf) return B200MPPI_OK;
  const int ws = p->cfg.world_size;
  if (ws < 2) return fail(B200MPPI_ESTATE, "p2p: world_size is 1");
  if (ws > P2P_MAX_PEERS) return fail(B200MPPI_EINVAL, "p2p: world_size > 16 (use the NCCL exchange)");
  CU(cudaSetDevice(p->cfg.device));
  auto up = [](size_t v) { return (v + 255) / 256 * 256; };
  const size_t len = (size_t)(2 * p->T + 2);
  size_t off = 0;
  off += up(p->shard_maps ? (size_t)p->n_local * p->M * sizeof(float) : 0);
  p->x_gather = off;      off += up(2 * (size_t)ws * len * sizeof(float));
  p->x_flags_cost = off;  off += up((size_t)ws * sizeof(uint32_t));
  p->x_flags_part = off;  off += up((size_t)ws * sizeof(uint32_t));
  p->x_counter = off;     off += 256;
  p->x_status = off;      off += 256;
  p->x_bytes = off;
  CU(cudaMalloc(&p->xbuf, off));
  CU(cudaMemset(p->xbuf, 0, off));
  if (const char* e = getenv("B200MPPI_P2P_TIMEOUT_MS")) {
    const long ms = atol(e);
    if (ms > 0) p->p2p_timeout_ns = (unsigned long long)ms * 1000000ull;
  }
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_p2p_export(b200mppi_planner* p, void* handle_out, size_t bytes) {
  if (!p || !handle_out) return fail(B200MPPI_EINVAL, "p2p_export: null argument");
  if (bytes < sizeof(cudaIpcMemHandle_t)) return fail(B200MPPI_EINVAL, "p2p_export: handle buffer < 64 bytes");
  int rc = p2p_alloc(p);
  if (rc) return rc;
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, p->xbuf));
  std::memcpy(handle_out, &h, sizeof(h));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_p2p_import(b200mppi_planner* p, const void* handles, size_t bytes) {
  if (!p || !handles) return fail(B200MPPI_EINVAL, "p2p_import: null argument");
  const int ws = p->cfg.world_size;
  if (bytes < (size_t)ws * sizeof(cudaIpcMemHandle_t)) return fail(B200MPPI_EINVAL, "p2p_import: need world_size handles");
  int rc = p2p_alloc(p);
  if (rc) return rc;
  CU(cudaSetDevice(p->cfg.device));
  for (int s = 0; s < ws; ++s) {
    if (s == p->cfg.rank) { p->peer_x[s] = p->xbuf; continue; }
    if (p->peer_x[s]) continue;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, (const unsigned char*)handles + (size_t)s * sizeof(h), sizeof(h));
    void* ptr = nullptr;
    CU(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    p->peer_x[s] = (unsigned char*)ptr;
    p->peer_ipc[s] = true;
  }
  p->p2p_ready = true;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_p2p_connect_local(b200mppi_planner* p, b200mppi_planner* const* peers, int32_t count) {
  if (!p || !peers) return fail(B200MPPI_EINVAL, "p2p_connect_local: null argument");
  if (count != p->cfg.world_size) return fail(B200MPPI_EINVAL, "p2p_connect_local: need world_size planners");
  for (int s = 0; s < count; ++s) {
    b200mppi_planner* q = peers[s];
    if (!q || q->cfg.rank != s || q->cfg.world_size != count || q->T != p->T || q->n_local != p->n_local || q->M != p->M)
      return fail(B200MPPI_EINVAL, "p2p_connect_local: peers[s] must be rank s of the same configuration");
    int rc = p2p_alloc(q);
    if (rc) return rc;
    if (q->cfg.device != p->cfg.device) {
      CU(cudaSetDevice(p->cfg.device));
      int can = 0;
      CU(cudaDeviceCanAccessPeer(&can, p->cfg.device, q->cfg.device));
      if (!can) return fail(B200MPPI_ECUDA, "p2p_connect_local: no peer access between the devices");
      const cudaError_t e = cudaDeviceEnablePeerAccess(q->cfg.device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CU(e);
      (void)cudaGetLastError();
    }
    p->peer_x[s] = q->xbuf;
  }
  p->p2p_ready = true;
  return B200MPPI_OK;
}

static int p2p_check(b200mppi_planner* p, const char* who) {
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  if (!p->p2p_ready) return fail(B200MPPI_ESTATE, std::string(who) + ": peers not connected (p2p_import / p2p_connect_local)");
  CU(cudaSetDevice(p->cfg.device));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_p2p_push(b200mppi_planner* p) {
  int rc = p2p_check(p, "p2p_push");
  if (rc) return rc;
  if (!p->shard_maps) return fail(B200MPPI_ESTATE, "p2p_push: only MODE_TDM shards the maps");
  if (p->pushed_direct) return B200MPPI_OK;      // the rollout kernel stored into the peers and raised the flags itself
  P2PPushArgs a{};
  a.costs_nm = p->costs_nm;
  a.ws = p->cfg.world_size; a.rank = p->cfg.rank; a.n_red = p->n_red; a.Mc = p->M;
  a.counter = (unsigned*)(p->xbuf + p->x_counter);
  a.epoch = ++p->epoch_cost;
  for (int s = 0; s < a.ws; ++s) {
    a.peer_recv[s] = (float*)p->peer_x[s];
    a.peer_flags[s] = (uint32_t*)(p->peer_x[s] + p->x_flags_cost);
  }
  launch_p2p_push(a, p->stream);
  p->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_p2p_reduce(b200mppi_planner* p) {
  int rc = p2p_check(p, "p2p_reduce");
  if (rc) return rc;
  const int ws = p->cfg.world_size;
  int* status = (int*)(p->xbuf + p->x_status);
  if (p->shard_maps) {
    // the CVaR kernel itself waits for every rank's cost flag, then reads the receive buffer: (M_total, N/ws), map-major
    const FlagWait fw{(const uint32_t*)(p->xbuf + p->x_flags_cost), ws, p->epoch_cost, p->p2p_timeout_ns, status};
    launch_cvar((const float*)p->xbuf, p->costs, p->n_red, p->n_red, p->M_total, p->prm.cvar_alpha, fw, p->stream);
    p->launches++;
    CHECK_LAUNCH();
    if (p->profiling) cudaEventRecord(p->ev[4], p->stream);
    if ((rc = stage_update_partial(p, UPD_TAIL_BCAST))) return rc;     // partial -> every peer, by the kernel's last CTA
  } else if (!p->bcast_done) {
    // N-sharded modes: solve_local ran before the peers were connected -- redo the (cheap) partial with the broadcast tail
    if ((rc = stage_update_partial(p, UPD_TAIL_BCAST))) return rc;
  }
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_p2p_finish(b200mppi_planner* p, float* u_out) {
  int rc = p2p_check(p, "p2p_finish");
  if (rc) return rc;
  const int ws = p->cfg.world_size;
  int* status = (int*)(p->xbuf + p->x_status);
  // the apply kernel waits for every rank's partial flag itself
  const FlagWait fw{(const uint32_t*)(p->xbuf + p->x_flags_part), ws, p->epoch_part, p->p2p_timeout_ns, status};
  const size_t parity_off = (size_t)(p->epoch_part & 1u) * ws * (2 * p->T + 2) * sizeof(float);
  if ((rc = stage_update_finish(p, (const float*)(p->xbuf + p->x_gather + parity_off), ws, fw))) return rc;
  p->bcast_done = false;
  if (p->profiling) cudaEventRecord(p->ev[5], p->stream);
  if (u_out) {
    int* h_status = (int*)(p->h_u + (size_t)p->T * 2);
    CU(cudaMemcpyAsync(p->h_u, p->u_cur, (size_t)p->T * 2 * sizeof(float), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaMemcpyAsync(h_status, status, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    if (*h_status != 0) {
      const int who = *h_status - 1;
      cudaMemsetAsync(status, 0, sizeof(int), p->stream);
      return fail(B200MPPI_ECUDA, "p2p exchange: timed out waiting for rank " + std::to_string(who));
    }
    std::memcpy(u_out, p->h_u, (size_t)p->T * 2 * sizeof(float));
    collect_timings(p);
  }
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_solve_p2p(b200mppi_planner* p, float* u_out) {
  if (p && p->loop) return loop_busy("planner_solve_p2p");
  int rc = p2p_check(p, "solve_p2p");
  if (rc) return rc;
  if (!u_out) return fail(B200MPPI_EINVAL, "solve_p2p: null output");
  const int num_opt = p->prm.num_opt;
  for (int k = 0; k < num_opt; ++k) {
    if ((rc = b200mppi_planner_solve_local(p, k == 0 ? 1 : 0))) return rc;
    if (p->shard_maps && (rc = b200mppi_planner_p2p_push(p))) return rc;
    if ((rc = b200mppi_planner_p2p_reduce(p))) return rc;
    if ((rc = b200mppi_planner_p2p_finish(p, k == num_opt - 1 ? u_out : nullptr))) return rc;
  }
  if (num_opt <= 0) return b200mppi_planner_get_u(p, u_out);
  return B200MPPI_OK;
}

// Host combine of gathered (beta, S, V[2T]) partials: same math as update_apply_kernel.
extern "C" int b200mppi_combine_partials_host(const float* g, int32_t ws, int32_t T, float lambda,
                                              const float* u_in, const float vr[2], const float wr[2],
                                              float* u_out) {
  if (!g || !u_in || !u_out || !vr || !wr || ws < 1 || T < 1) return fail(B200MPPI_EINVAL, "combine: bad argument");
  const int stride = 2 * T + 2;
  float beta = INFINITY;
  for (int r = 0; r < ws; ++r) beta = std::fmin(beta, g[(size_t)r * stride]);
  std::vector<float> sc(ws);
  float W = 0.0f;
  for (int r = 0; r < ws; ++r) {
    const float b = g[(size_t)r * stride];
    sc[r] = std::isinf(b) ? 0.0f : (float)std::exp((-1.0 / (double)lambda) * (double)(b - beta));
    W = std::fmaf(g[(size_t)r * stride + 1], sc[r], W);
  }
  for (int j = 0; j < 2 * T; ++j) {
    float v = 0.0f;
    for (int r = 0; r < ws; ++r) v = std::fmaf(g[(size_t)r * stride + 2 + j], sc[r], v);
    const float u = (W == 0.0f) ? u_in[j] : u_in[j] + v / W;      // every cost +inf: a zero step
    const float lo = (j & 1) ? wr[0] : vr[0], hi = (j & 1) ? wr[1] : vr[1];
    u_out[j] = std::fmax(lo, std::fmin(hi, u));
  }
  return B200MPPI_OK;
}

// ---- stage-level entry points
extern "C" int b200mppi_planner_sample_noise(b200mppi_planner* p) {
  if (p && p->loop) return loop_busy("planner_sample_noise");
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  if (!p->params_set) return fail(B200MPPI_ESTATE, "sample_noise: params not set");
  CU(cudaSetDevice(p->cfg.device));
  int rc = stage_noise(p);
  if (rc) return rc;
  CU(cudaStreamSynchronize(p->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_rollout(b200mppi_planner* p) {
  if (p && p->loop) return loop_busy("planner_rollout");
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  int rc = planner_check_ready(p);
  if (rc) return rc;
  CU(cudaSetDevice(p->cfg.device));
  if (p->cfg.mode != B200MPPI_MODE_BAREBONE) {            // the maps of the last solve may be boxed
    if ((rc = tdm_complete_grid(p->lin, p->stream))) return rc;
    if ((rc = tdm_complete_grid(p->ang, p->stream))) return rc;
  }
  if ((rc = stage_rollout(p))) return rc;
  CU(cudaStreamSynchronize(p->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_cvar(b200mppi_planner* p) {
  if (p && p->loop) return loop_busy("planner_cvar");
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  if (!p->params_set) return fail(B200MPPI_ESTATE, "cvar: params not set");
  if (p->cfg.mode != B200MPPI_MODE_TDM) return fail(B200MPPI_ESTATE, "cvar: only MODE_TDM has per-(n,m) costs");
  if (p->M > cvar_max_maps()) return fail(B200MPPI_EINVAL, "cvar: num_grid_samples exceeds the CVaR kernel's limit (16384)");
  CU(cudaSetDevice(p->cfg.device));
  if (p->shard_maps) return fail(B200MPPI_ESTATE, "cvar: maps are sharded, use solve_reduce");
  launch_cvar(p->costs_nm, p->costs, p->n_local, p->n_local, p->M, p->prm.cvar_alpha, FlagWait{}, p->stream);
  p->launches++;
  CHECK_LAUNCH();
  CU(cudaStreamSynchronize(p->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_update(b200mppi_planner* p, const float* costs_host) {
  if (p && p->loop) return loop_busy("planner_update");
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  if (!p->params_set) return fail(B200MPPI_ESTATE, "update: params not set");
  CU(cudaSetDevice(p->cfg.device));
  if (costs_host)
    CU(cudaMemcpyAsync(p->costs, costs_host, (size_t)p->n_red * sizeof(float), cudaMemcpyHostToDevice, p->stream));
  int rc = stage_update_partial(p, p->cfg.world_size == 1 ? UPD_TAIL_APPLY : UPD_TAIL_RANK);
  if (rc) return rc;
  CU(cudaStreamSynchronize(p->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_get_state_rollout(b200mppi_planner* p, float* out, size_t bytes) {
  if (p && p->loop) return loop_busy("planner_get_state_rollout");
  if (!p || !out) return fail(B200MPPI_EINVAL, "null argument");
  int rc = planner_check_ready(p);
  if (rc) return rc;
  const int V = p->cfg.num_vis_state_rollouts < 1 ? 1 : p->cfg.num_vis_state_rollouts;
  const size_t need = (size_t)V * (p->T + 1) * 3 * sizeof(float);
  if (bytes != need) return fail(B200MPPI_EINVAL, "get_state_rollout: size mismatch");
  if (p->cfg.mode == B200MPPI_MODE_TDM ? V > p->lin->num_maps : V > p->n_local)
    return fail(B200MPPI_EINVAL, "get_state_rollout: more vis rollouts than maps / local rollouts");
  CU(cudaSetDevice(p->cfg.device));
  VisArgs a{};
  fill_rollout_params(p, a.p);
  a.mode = p->cfg.mode; a.V = V;
  if (p->cfg.mode != B200MPPI_MODE_BAREBONE) {
    if ((rc = tdm_complete_grid(p->lin, p->stream))) return rc;   // the optimal sequence may leave the last solve's box
    if ((rc = tdm_complete_grid(p->ang, p->stream))) return rc;
    a.lin_grid = p->lin->grid; a.ang_grid = p->ang->grid;
  }
  a.noise = p->noise; a.u_cur = p->u_cur; a.u_prev = p->u_prev; a.out = p->state_rollout;
  launch_state_rollout(a, p->stream);
  p->launches++;
  CHECK_LAUNCH();
  CU(cudaMemcpyAsync(out, p->state_rollout, need, cudaMemcpyDeviceToHost, p->stream));
  CU(cudaStreamSynchronize(p->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_buffer(b200mppi_planner* p, int32_t id, void** ptr, size_t* bytes) {
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  void* d = nullptr; size_t b = 0;
  const size_t nl = p->n_local, T = p->T;
  const int V = p->cfg.num_vis_state_rollouts < 1 ? 1 : p->cfg.num_vis_state_rollouts;
  switch (id) {
    case B200MPPI_BUF_NOISE: d = p->noise; b = nl * T * 2 * sizeof(float); break;
    case B200MPPI_BUF_U_CUR: d = p->u_cur; b = T * 2 * sizeof(float); break;
    case B200MPPI_BUF_U_PREV: d = p->u_prev; b = T * 2 * sizeof(float); break;
    case B200MPPI_BUF_COSTS: d = p->costs; b = (size_t)p->n_red * sizeof(float); break;
    case B200MPPI_BUF_WEIGHTS: d = p->weights; b = (size_t)p->n_red * sizeof(float); break;
    case B200MPPI_BUF_COSTS_NM: d = p->costs_nm; b = nl * p->M * sizeof(float); break;
    case B200MPPI_BUF_RNG: d = p->states; b = nl * T * 16; break;
    case B200MPPI_BUF_PARTIAL: d = p->rank_partial; b = (2 * T + 2) * sizeof(float); break;
    case B200MPPI_BUF_STATE_ROLLOUT: d = p->state_rollout; b = (size_t)V * (T + 1) * 3 * sizeof(float); break;
    default: return fail(B200MPPI_EINVAL, "buffer: unknown id");
  }
  if (ptr) *ptr = d;
  if (bytes) *bytes = b;
  return B200MPPI_OK;
}

// B200MPPI_BUF_COSTS_NM through copy_out / copy_in is the LOGICAL array (n_local, M_local), element [n][m] -- the
// device buffer is map-major and, for a map-sharded planner, split into per-destination blocks (fill_cost_dst):
// logical [n][m]  <->  block n / n_per, row m, column n % n_per.
static void costs_logical(const b200mppi_planner* p, const float* dev_layout, float* logical, bool to_logical) {
  const int N = p->n_local, M = p->M;
  const int n_per = p->shard_maps ? p->n_red : N;
  for (int n = 0; n < N; ++n) {
    const int blk = n / n_per, c = n - blk * n_per;
    for (int m = 0; m < M; ++m) {
      const size_t di = ((size_t)blk * M + m) * n_per + c, li = (size_t)n * M + m;
      if (to_logical) logical[li] = dev_layout[di]; else const_cast<float*>(dev_layout)[di] = logical[li];
    }
  }
}

extern "C" int b200mppi_planner_copy_out(b200mppi_planner* p, int32_t id, void* dst, size_t bytes) {
  if (p && p->loop) return loop_busy("planner_copy_out");
  void* d; size_t b;
  int rc = b200mppi_planner_buffer(p, id, &d, &b);
  if (rc) return rc;
  if (!dst || bytes != b) return fail(B200MPPI_EINVAL, "copy_out: size mismatch");
  CU(cudaSetDevice(p->cfg.device));
  if (id == B200MPPI_BUF_COSTS_NM) {
    std::vector<float> tmp(b / sizeof(float));
    CU(cudaMemcpyAsync(tmp.data(), d, b, cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    costs_logical(p, tmp.data(), (float*)dst, true);
    return B200MPPI_OK;
  }
  CU(cudaMemcpyAsync(dst, d, b, cudaMemcpyDeviceToHost, p->stream));
  CU(cudaStreamSynchronize(p->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_copy_in(b200mppi_planner* p, int32_t id, const void* src, size_t bytes) {
  if (p && p->loop) return loop_busy("planner_copy_in");
  void* d; size_t b;
  int rc = b200mppi_planner_buffer(p, id, &d, &b);
  if (rc) return rc;
  if (!src || bytes != b) return fail(B200MPPI_EINVAL, "copy_in: size mismatch");
  CU(cudaSetDevice(p->cfg.device));
  p->prepared = false;
  if (id == B200MPPI_BUF_COSTS_NM) {
    std::vector<float> tmp(b / sizeof(float));
    costs_logical(p, tmp.data(), const_cast<float*>((const float*)src), false);
    CU(cudaMemcpyAsync(d, tmp.data(), b, cudaMemcpyHostToDevice, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    return B200MPPI_OK;
  }
  CU(cudaMemcpyAsync(d, src, b, cudaMemcpyHostToDevice, p->stream));
  CU(cudaStreamSynchronize(p->stream));
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_set_noise(b200mppi_planner* p, const float* noise, size_t bytes) {
  if (p && p->loop) return loop_busy("planner_set_noise");
  return b200mppi_planner_copy_in(p, B200MPPI_BUF_NOISE, noise, bytes);
}

extern "C" int b200mppi_planner_synchronize(b200mppi_planner* p) {
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  CU(cudaSetDevice(p->cfg.device));
  CU(cudaStreamSynchronize(p->stream));
  collect_timings(p);                          // stage-level callers (solve_local + synchronize) get their stage times too
  (void)cudaGetLastError();                    // events of stages that did not run are unrecorded
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_set_profiling(b200mppi_planner* p, int32_t enable) {
  if (!p) return fail(B200MPPI_EINVAL, "null planner");
  p->profiling = enable != 0;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_last_timings(b200mppi_planner* p, float* ms) {
  if (!p || !ms) return fail(B200MPPI_EINVAL, "null argument");
  for (int i = 0; i < B200MPPI_T_COUNT; ++i) ms[i] = p->last_ms[i];
  return B200MPPI_OK;
}

// Debug hook (tools/rollout_cta_times.py): per-CTA start / end times (ns, %globaltimer) and chunk shares of the NEXT
// windowed rollout launches of this process; enable = 0 switches it off.  out: 6 x int64 per CTA (start ns, end ns, share
// lo / hi in chunks, lane-steps on the slow path, of which outside the staged window), `ctas` records.
extern "C" int b200mppi_debug_rollout_cta_times(int32_t enable, int64_t* out, int32_t ctas) {
  static long long* dev = nullptr;
  if (enable) {
    if (!dev) CU(cudaMalloc(&dev, 1024 * 6 * sizeof(long long)));
    CU(cudaMemset(dev, 0, 1024 * 6 * sizeof(long long)));
    rollout_win_set_debug(dev);
  }
  if (out && dev && ctas > 0 && ctas <= 1024) {
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(out, dev, (size_t)ctas * 6 * sizeof(long long), cudaMemcpyDeviceToHost));
  }
  if (!enable) rollout_win_set_debug(nullptr);
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_sample_window(b200mppi_planner* p, int32_t out[6]) {
  if (!p || !out) return fail(B200MPPI_EINVAL, "sample_window: null argument");
  out[0] = p->win_used ? 1 : 0;
  for (int i = 0; i < 4; ++i) out[1 + i] = p->win_used ? p->win_rect[i] : 0;
  out[5] = p->win_used ? p->win_flagged : 0;
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_sample_box(b200mppi_planner* p, int32_t out[5]) {
  if (!p || !out) return fail(B200MPPI_EINVAL, "null argument");
  for (int i = 0; i < 5; ++i) out[i] = p->last_box[i];
  return B200MPPI_OK;
}

extern "C" int b200mppi_planner_launch_count(b200mppi_planner* p, int64_t* out) {
  if (!p || !out) return fail(B200MPPI_EINVAL, "null argument");
  *out = p->launches;
  return B200MPPI_OK;
}

// --------------------------------------------------------------------------------------------- batch
// K independent one-map planners of equal N and T solved with one launch per stage (noise, map sampling, rollout,
// update) for the whole batch.  The per-planner kernel arguments travel as descriptor arrays in device memory (a
// grid coordinate selects the planner): rebuilt every solve -- params, maps and TDM buffers may change in between --
// and uploaded with ONE copy from pinned staging.  Every kernel of a planner computes exactly what it computes in that
// planner's own solve(), in the same order, so the results are those of K solve() calls, bit for bit.
struct b200mppi_batch {
  std::vector<b200mppi_planner*> pl;
  int device = 0, mode = 0, T = 0, N = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaEvent_t ev = nullptr;            // orders the batch after the work already issued on a member's stream
  // descriptor arrays, one allocation: [NoiseDesc K | SampleGridsV2Args K | RolloutArgs K | UpdateBatchDesc K]
  size_t off_sample = 0, off_roll = 0, off_upd = 0, desc_bytes = 0;
  unsigned char* h_desc = nullptr;     // pinned staging
  unsigned char* d_desc = nullptr;
  float* u_d = nullptr;                // (K, T, 2): every planner's new u, written by its update's last CTA
  float* h_u = nullptr;                // pinned (K, T, 2)
  int64_t launches = 0;
  // stochastic batch (b200mppi_batch_create_stochastic): MODE_TDM planners, windowed rollouts.  Descriptors:
  // [NoisePrepDesc K | RolloutWinArgs K | CUtensorMap 4K (64-byte aligned) | CvarDesc K | UpdateBatchDesc K]
  bool stochastic = false;
  int M = 0;
  size_t off_win = 0, off_tm = 0, off_cvar = 0;
  // b200mppi_batch_get_state_rollout's section, after the solve's (a solve does not upload it):
  // [RolloutParams K | VisBatchDesc K] from off_vis, vis_bytes long
  size_t off_vis = 0, off_visd = 0, vis_bytes = 0;
  bool share = false;                  // b200mppi_batch_share_tdms: planners on one TDM pair sample it once per call
  // the one-map planners are pl[0 .. nmap), the MODE_TDM planners pl[nmap .. K): nmap is K in a one-map batch, 0 in a
  // stochastic one.  A mixed batch (b200mppi_batch_create_mixed) holds both, and its descriptors both sections:
  // [NoiseDesc nmap | SampleGridsV2Args nmap | RolloutArgs nmap | NoisePrepDesc | RolloutWinArgs | CUtensorMap 4x |
  //  CvarDesc (K - nmap each) | UpdateBatchDesc K]; its mode is the one-map planners' mode, ROLLOUT_MODE_PER_DESC when
  // they mix MODE_DET_DYN and MODE_SPEED_MAP
  bool mixed = false;
  int nmap = 0;
  size_t off_nprep = 0;
  const b200mppi_loop* loop = nullptr;   // its open device loop (b200mppi_batch_loop_open)
};

// Hands out 256-byte-aligned sections of one allocation, in order: take returns a section's offset.  An empty section
// takes no bytes.
struct Sections {
  size_t end = 0;
  size_t take(size_t bytes) {
    const size_t at = end;
    end += (bytes + 255) / 256 * 256;
    return at;
  }
};

extern "C" int b200mppi_batch_destroy(b200mppi_batch* b) {
  if (b && b->loop) return loop_busy("batch_destroy");
  if (!b) return B200MPPI_OK;
  cudaSetDevice(b->device);
  if (b->stream) cudaStreamSynchronize(b->stream);
  cudaFree(b->d_desc); cudaFree(b->u_d);
  if (b->h_desc) cudaFreeHost(b->h_desc);
  if (b->h_u) cudaFreeHost(b->h_u);
  if (b->ev) cudaEventDestroy(b->ev);
  if (b->own_stream && b->stream) cudaStreamDestroy(b->stream);
  delete b;
  return B200MPPI_OK;
}

static int batch_init(b200mppi_batch* b) {
  const size_t K = b->pl.size(), K1 = b->nmap, K2 = K - K1;
  Sections s;
  s.take(K1 * sizeof(NoiseDesc));                      // at 0
  b->off_sample = s.take(K1 * sizeof(SampleGridsV2Args));
  b->off_roll = s.take(K1 * sizeof(RolloutArgs));
  b->off_nprep = s.take(K2 * sizeof(NoisePrepDesc));
  b->off_win = s.take(K2 * sizeof(RolloutWinArgs));
  b->off_tm = s.take(K2 * sizeof(b200mppi_planner::tmaps));
  b->off_cvar = s.take(K2 * sizeof(CvarDesc));
  b->off_upd = s.take(K * sizeof(UpdateBatchDesc));
  b->desc_bytes = s.end;
  b->off_vis = s.take(K * sizeof(RolloutParams));
  b->off_visd = s.take(K * sizeof(VisBatchDesc));
  b->vis_bytes = s.end - b->off_vis;
  CU(cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking));
  b->own_stream = true;
  CU(cudaEventCreateWithFlags(&b->ev, cudaEventDisableTiming));
  CU(cudaMallocHost(&b->h_desc, b->desc_bytes + b->vis_bytes));
  CU(cudaMalloc(&b->d_desc, b->desc_bytes + b->vis_bytes));
  const size_t ubytes = K * (size_t)b->T * 2 * sizeof(float);
  CU(cudaMallocHost(&b->h_u, ubytes));
  CU(cudaMalloc(&b->u_d, ubytes));
  return B200MPPI_OK;
}

// One-map batches hold MODE_DET_DYN, MODE_SPEED_MAP or MODE_BAREBONE planners of one mode; stochastic batches hold
// MODE_TDM planners of equal M; mixed batches hold MODE_DET_DYN and MODE_SPEED_MAP planners in any order, then MODE_TDM
// planners of equal M.  All hold single-rank planners of one device, T and N.
enum class BatchKind { onemap, stochastic, mixed };

static int batch_create(b200mppi_planner* const* planners, int32_t count, BatchKind kind, b200mppi_batch** out) {
  const bool stochastic = kind == BatchKind::stochastic, mixed = kind == BatchKind::mixed;
  const std::string fn = stochastic ? "batch_create_stochastic" : mixed ? "batch_create_mixed" : "batch_create";
  if (!planners || !out) return fail(B200MPPI_EINVAL, fn + ": null argument");
  if (count < 1) return fail(B200MPPI_EINVAL, fn + ": count < 1");
  if (count > 65535) return fail(B200MPPI_EINVAL, fn + ": more than 65535 planners");
  for (int i = 0; i < count; ++i) {
    const b200mppi_planner* p = planners[i];
    const std::string who = fn + ": planner " + std::to_string(i);
    if (!p) return fail(B200MPPI_EINVAL, who + " is null");
    for (int j = 0; j < i; ++j)
      if (planners[j] == p) return fail(B200MPPI_EINVAL, who + " is planner " + std::to_string(j) + " again");
    if (stochastic && p->cfg.mode != B200MPPI_MODE_TDM)
      return fail(B200MPPI_EINVAL, who + " has mode " + std::to_string(p->cfg.mode) +
                                       " (a stochastic batch holds MODE_TDM planners)");
    if (mixed && p->cfg.mode == B200MPPI_MODE_BAREBONE)
      return fail(B200MPPI_EINVAL, who + " is MODE_BAREBONE (a mixed batch holds MODE_DET_DYN, MODE_SPEED_MAP and "
                                         "MODE_TDM planners; barebone planners run in b200mppi_batch_create batches)");
    if (mixed && i > 0 && planners[i - 1]->cfg.mode == B200MPPI_MODE_TDM && p->cfg.mode != B200MPPI_MODE_TDM)
      return fail(B200MPPI_EINVAL, who + " has mode " + std::to_string(p->cfg.mode) + " after a MODE_TDM planner (a "
                                         "mixed batch takes its one-map planners first, then its MODE_TDM planners)");
    if (kind == BatchKind::onemap && p->cfg.mode == B200MPPI_MODE_TDM)
      return fail(B200MPPI_EINVAL, who + " is MODE_TDM: the stochastic mode is not batched (batches hold "
                                         "MODE_DET_DYN, MODE_SPEED_MAP or MODE_BAREBONE planners)");
    if (p->cfg.world_size != 1)
      return fail(B200MPPI_EINVAL, who + " has world_size " + std::to_string(p->cfg.world_size) +
                                       " (a batch holds single-rank planners)");
    const b200mppi_planner* q = planners[0];
    if (p->cfg.device != q->cfg.device)
      return fail(B200MPPI_EINVAL, who + " is on device " + std::to_string(p->cfg.device) + ", planner 0 on device " +
                                       std::to_string(q->cfg.device));
    if (kind == BatchKind::onemap && p->cfg.mode != q->cfg.mode)
      return fail(B200MPPI_EINVAL, who + " has mode " + std::to_string(p->cfg.mode) + ", planner 0 mode " +
                                       std::to_string(q->cfg.mode) + " (modes cannot be mixed)");
    if (p->T != q->T) return fail(B200MPPI_EINVAL, who + " has num_steps " + std::to_string(p->T) + ", planner 0 " +
                                                      std::to_string(q->T) + " (T must be equal)");
    if (p->n_local != q->n_local)
      return fail(B200MPPI_EINVAL, who + " has num_control_rollouts " + std::to_string(p->n_local) + ", planner 0 " +
                                       std::to_string(q->n_local) + " (N must be equal)");
    int t = 0;                                         // the batch's first MODE_TDM planner
    while (planners[t]->cfg.mode != B200MPPI_MODE_TDM && t < i) ++t;
    if (p->cfg.mode == B200MPPI_MODE_TDM && p->M != planners[t]->M)
      return fail(B200MPPI_EINVAL, who + " has num_grid_samples " + std::to_string(p->M) + ", planner " +
                                       std::to_string(t) + " " + std::to_string(planners[t]->M) + " (M must be equal)");
  }
  // any M a planner can have (planner_create: at most cvar_max_maps()).  Index ranges at the largest batch, 65535
  // planners of 16384 maps: the windowed rollout's count * M (planner, map) units stay below 2^30 (an int), its chunk
  // totals are 64-bit; the CVaR and sampler grids put the planner on y or z (<= 65535) and the map groups on y
  // (<= 16384); the state advance's grid x and every descriptor offset are computed in 64 bits.
  CU(cudaSetDevice(planners[0]->cfg.device));
  b200mppi_batch* b = new b200mppi_batch();
  b->pl.assign(planners, planners + count);
  b->device = planners[0]->cfg.device; b->mode = planners[0]->cfg.mode;
  b->T = planners[0]->T; b->N = planners[0]->n_local;
  b->stochastic = stochastic;
  b->mixed = mixed;
  while (b->nmap < count && planners[b->nmap]->cfg.mode != B200MPPI_MODE_TDM) ++b->nmap;
  for (int i = 1; i < b->nmap; ++i)
    if (planners[i]->cfg.mode != b->mode) b->mode = ROLLOUT_MODE_PER_DESC;
  if (b->nmap < count) b->M = planners[b->nmap]->M;
  const int rc = batch_init(b);
  if (rc) {
    const std::string keep = g_err;
    b200mppi_batch_destroy(b);
    g_err = keep;
    return rc;
  }
  *out = b;
  return B200MPPI_OK;
}

extern "C" int b200mppi_batch_create(b200mppi_planner* const* planners, int32_t count, b200mppi_batch** out) {
  return batch_create(planners, count, BatchKind::onemap, out);
}

// K independent MODE_TDM planners of equal N, T and M solved with one launch per stage (noise + controls, windowed
// rollout, CVaR, update); the map sampling stays per planner (each planner's reach box is its own).  The results are
// those of K solve() calls in planner order, bit for bit (include/b200mppi.h).
extern "C" int b200mppi_batch_create_stochastic(b200mppi_planner* const* planners, int32_t count, b200mppi_batch** out) {
  return batch_create(planners, count, BatchKind::stochastic, out);
}

// MODE_DET_DYN and MODE_SPEED_MAP planners, then MODE_TDM planners, of equal N and T: each kind's stages as in its own
// batch, one update launch over all K planners (include/b200mppi.h)
extern "C" int b200mppi_batch_create_mixed(b200mppi_planner* const* planners, int32_t count, b200mppi_batch** out) {
  return batch_create(planners, count, BatchKind::mixed, out);
}

extern "C" int b200mppi_batch_set_stream(b200mppi_batch* b, void* s) {
  if (b && b->loop) return loop_busy("batch_set_stream");
  if (!b) return fail(B200MPPI_EINVAL, "null batch");
  if (b->own_stream && b->stream) { cudaStreamSynchronize(b->stream); cudaStreamDestroy(b->stream); }
  b->stream = (cudaStream_t)s;
  b->own_stream = false;
  return B200MPPI_OK;
}

extern "C" int b200mppi_batch_launch_count(b200mppi_batch* b, int64_t* out) {
  if (!b || !out) return fail(B200MPPI_EINVAL, "null argument");
  *out = b->launches;
  return B200MPPI_OK;
}

extern "C" int b200mppi_batch_share_tdms(b200mppi_batch* b, int32_t enable) {
  if (b && b->loop) return loop_busy("batch_share_tdms");
  if (!b) return fail(B200MPPI_EINVAL, "null batch");
  b->share = enable != 0;
  return B200MPPI_OK;
}

// The TDM groups of the batch's planners [lo, hi) (one kind: the one-map or the MODE_TDM planners) for one call: with
// sharing on, planners with the same (lin, ang) objects form one group (in the order of their first members); otherwise,
// and in barebone batches, every planner is a group of its own.  Group g's planners are members[first[g] .. first[g + 1]),
// in planner order, counted from lo (the index of the kind's launches); per group, plans, launches and commits run once.
struct TdmGroups {
  std::vector<int> of;                 // planner -> group
  std::vector<int> first;              // G + 1 offsets into members
  std::vector<int> members;
  int size() const { return (int)first.size() - 1; }
  int count(int g) const { return first[g + 1] - first[g]; }
  int lead(int g) const { return members[first[g]]; }
  bool shared() const { return (int)members.size() > size(); }
};

static TdmGroups batch_groups(const b200mppi_batch* b, int lo, int hi) {
  b200mppi_planner* const* pl = b->pl.data() + lo;
  const int K = hi - lo;
  TdmGroups gr;
  gr.of.assign(K, -1);
  std::vector<std::vector<int>> g;
  for (int i = 0; i < K; ++i) {
    const b200mppi_planner* p = pl[i];
    if (b->share && b->mode != B200MPPI_MODE_BAREBONE)
      for (int j = 0; j < i && gr.of[i] < 0; ++j)
        if (pl[j]->lin == p->lin && pl[j]->ang == p->ang) gr.of[i] = gr.of[j];
    if (gr.of[i] < 0) { gr.of[i] = (int)g.size(); g.emplace_back(); }
    g[gr.of[i]].push_back(i);
  }
  gr.first.push_back(0);
  for (const std::vector<int>& m : g) {
    gr.members.insert(gr.members.end(), m.begin(), m.end());
    gr.first.push_back((int)gr.members.size());
  }
  return gr;
}

static const char* mode_name(int mode) {
  return mode == B200MPPI_MODE_DET_DYN ? "MODE_DET_DYN" : mode == B200MPPI_MODE_SPEED_MAP ? "MODE_SPEED_MAP" :
         mode == B200MPPI_MODE_BAREBONE ? "MODE_BAREBONE" : "MODE_TDM";
}

// Everything a batch solve checks before it issues any work.
static int batch_validate(b200mppi_batch* b) {
  const int K = (int)b->pl.size();
  for (int i = 0; i < K; ++i) {
    const int rc = planner_check_ready(b->pl[i]);
    if (rc) return fail(rc, "batch_solve: planner " + std::to_string(i) + ": " + g_err);
  }
  for (int i = 0; i < K; ++i) {
    const b200mppi_planner* p = b->pl[i];
    if (p->prm.num_opt != b->pl[0]->prm.num_opt)
      return fail(B200MPPI_EINVAL, "batch_solve: planner " + std::to_string(i) + " has num_opt " +
                                       std::to_string(p->prm.num_opt) + ", planner 0 num_opt " +
                                       std::to_string(b->pl[0]->prm.num_opt) + " (must be equal)");
  }
  if (b->mode == B200MPPI_MODE_BAREBONE) return B200MPPI_OK;
  // sequential solves would sample a TDM shared by two planners twice, one after the other: those planners are not
  // independent, so the batch refuses them (one planner's lin == ang is fine: its own solve samples it twice too).  With
  // sharing on, planners on the same (lin, ang) pair form a group sampled once; any other overlap is still refused.
  for (int i = 0; i < K; ++i)
    for (int j = 0; j < i; ++j) {
      const b200mppi_planner* p = b->pl[i]; const b200mppi_planner* q = b->pl[j];
      const std::string both = "batch_solve: planners " + std::to_string(j) + " and " + std::to_string(i);
      if (!b->share) {
        if (p->lin == q->lin || p->lin == q->ang || p->ang == q->lin || p->ang == q->ang)
          return fail(B200MPPI_EINVAL, both + " share a TDM (batched planners must be independent)");
        continue;
      }
      if (p->lin == q->ang || p->ang == q->lin)
        return fail(B200MPPI_EINVAL, both + ": a TDM is lin of one and ang of the other (a shared TDM pair must be "
                                            "the same (lin, ang) of every planner on it)");
      if ((p->lin == q->lin) != (p->ang == q->ang))
        return fail(B200MPPI_EINVAL, both + " share " + (p->lin == q->lin ? "lin but not ang" : "ang but not lin") +
                                         " (a shared TDM pair must be the same (lin, ang) of every planner on it)");
      if ((p->lin == q->lin || p->ang == q->ang) && (i < b->nmap) != (j < b->nmap))
        return fail(B200MPPI_EINVAL, both + " share a TDM pair, but planner " + std::to_string(j) + " is " +
                                         mode_name(q->cfg.mode) + " and planner " + std::to_string(i) + " " +
                                         mode_name(p->cfg.mode) + " (a pair is shared by planners of one kind)");
      if (p->lin == q->lin && sample_alpha(p) != sample_alpha(q))
        return fail(B200MPPI_EINVAL, both + " share a TDM pair but have alpha_dyn " + std::to_string(sample_alpha(q)) +
                                         " and " + std::to_string(sample_alpha(p)) +
                                         " (a shared pair is sampled once, at one alpha_dyn)");
    }
  return B200MPPI_OK;
}

// sample_box() after a whole-map sampling
static void last_box_whole_map(b200mppi_planner* p) {
  p->last_box[0] = 0; p->last_box[1] = 0; p->last_box[2] = p->lin->rows; p->last_box[3] = 0; p->last_box[4] = p->lin->cols;
}

// The maps of every planner, as its solve() samples them: the pairs whose plan is fused and whose launch equals the
// first such pair's go into ONE launch; every other pair runs its own plan, in planner order.  One-map modes never
// sample a reach box.
// Planning (host tables, the batched pairs' descriptors) comes before the solve's one upload, the launches after the noise.
constexpr double BATCH_ALPHA = 1.0;   // det / speed-map solves sample with the default alpha_dyn (stage_sample_tdms)

// One plan per TDM group (a shared pair is sampled once: one entry of the batched launch or one plan of its own).
static int batch_plan_sample(b200mppi_batch* b, const TdmGroups& gr, SampleGridsV2Args* h_sg,
                             std::vector<SamplePlan>& plans, std::vector<char>& joined, int* njoined) {
  const int G = gr.size();
  plans.resize(G);
  joined.assign(G, 0);
  int nj = 0;
  for (int g = 0; g < G; ++g) {
    const b200mppi_planner* p = b->pl[gr.lead(g)];
    const int rc = plan_sampling(p->lin, p->ang, BATCH_ALPHA, b->stream, &plans[g]);
    if (rc) return rc;
    if (!plans[g].fused || (nj > 0 && !sample_grids_v2_same_launch(h_sg[0], plans[g].a[0]))) continue;
    h_sg[nj++] = plans[g].a[0];
    joined[g] = 1;
  }
  *njoined = nj;
  return B200MPPI_OK;
}

static int batch_run_sample(b200mppi_batch* b, const TdmGroups& gr, const SampleGridsV2Args* h_sg,
                            const SampleGridsV2Args* d_sg, std::vector<SamplePlan>& plans,
                            const std::vector<char>& joined, int nj) {
  if (nj > 0) {
    const SampleGridsV2Args* g0 = h_sg;
    launch_sample_grids_v2_batch(sample_class_launch(&g0, 1), d_sg, nj, nullptr, nullptr, b->stream);
    b->launches++;
    CHECK_LAUNCH();
  }
  for (int g = 0; g < gr.size(); ++g) {
    if (joined[g]) {
      plan_commit(plans[g], 0);
      plan_commit(plans[g], 1);
    } else {
      const int rc = plan_launch(plans[g], false, b->stream, &b->launches);
      if (rc) return rc;
    }
    for (int j = gr.first[g]; j < gr.first[g + 1]; ++j) last_box_whole_map(b->pl[gr.members[j]]);
  }
  return B200MPPI_OK;
}

// start after everything already issued on the members' streams (idle streams need no event)
static int batch_wait_members(b200mppi_batch* b) {
  for (b200mppi_planner* p : b->pl) {
    if (p->stream == b->stream) continue;
    const cudaError_t q = cudaStreamQuery(p->stream);
    if (q == cudaSuccess) continue;
    if (q != cudaErrorNotReady) CU(q);
    CU(cudaEventRecord(b->ev, p->stream));
    CU(cudaStreamWaitEvent(b->stream, b->ev, 0));
  }
  return B200MPPI_OK;
}

// planner p's batched update: UPD_TAIL_APPLY also stores the new u at u_out (the batch's (K, T, 2)) and u_prev if set
static void fill_update_apply(b200mppi_planner* p, UpdateBatchDesc& u, float* u_out, float* u_prev) {
  fill_update_args(p, u.a, nullptr);
  u.tl = UpdateTail{};
  u.tl.counter = p->upd_counter_d;
  u.tl.mode = UPD_TAIL_APPLY;
  u.tl.u_prev = u_prev;
  u.tl.u_out = u_out;
}

// The one-map planners' noise, rollout and update descriptors at byte offset 0 of `h` (b->h_desc's layout)
static void onemap_descs(b200mppi_batch* b, unsigned char* h) {
  NoiseDesc* hn = reinterpret_cast<NoiseDesc*>(h);
  RolloutArgs* hr = reinterpret_cast<RolloutArgs*>(h + b->off_roll);
  UpdateBatchDesc* hu = reinterpret_cast<UpdateBatchDesc*>(h + b->off_upd);
  for (int i = 0; i < b->nmap; ++i) {
    b200mppi_planner* p = b->pl[i];
    hn[i] = NoiseDesc{p->states, p->noise, p->prm.u_std[0], p->prm.u_std[1]};
    fill_rollout_args(p, hr[i]);
    // self.u_prev_d = self.u_cur_d (alias, mppi.py:292,362)
    fill_update_apply(p, hu[i], b->u_d + (size_t)i * b->T * 2, p->u_prev);
  }
}

// A solve's one-map part (planners [0, nmap)): per iteration ONE noise launch, [first iteration: the maps,
// batch_run_sample] and ONE rollout launch
struct OnemapSolve {
  TdmGroups gr;
  std::vector<SamplePlan> plans;
  std::vector<char> joined;
  int nj = 0;
};

// the descriptors and sampler plans, before the solve's one upload
static int onemap_solve_plan(b200mppi_batch* b, OnemapSolve& os) {
  onemap_descs(b, b->h_desc);
  if (b->mode == B200MPPI_MODE_BAREBONE) return B200MPPI_OK;
  os.gr = batch_groups(b, 0, b->nmap);
  return batch_plan_sample(b, os.gr, reinterpret_cast<SampleGridsV2Args*>(b->h_desc + b->off_sample), os.plans,
                           os.joined, &os.nj);
}

static int onemap_solve_sample(b200mppi_batch* b, OnemapSolve& os) {
  if (b->mode == B200MPPI_MODE_BAREBONE) return B200MPPI_OK;
  return batch_run_sample(b, os.gr, reinterpret_cast<const SampleGridsV2Args*>(b->h_desc + b->off_sample),
                          reinterpret_cast<const SampleGridsV2Args*>(b->d_desc + b->off_sample), os.plans, os.joined,
                          os.nj);
}

static int onemap_solve_iteration(b200mppi_batch* b, OnemapSolve& os, int k) {
  const int K1 = b->nmap;
  launch_sample_noise_batch(reinterpret_cast<const NoiseDesc*>(b->d_desc), K1, b->N, b->T, nullptr, b->stream);
  b->launches++;
  CHECK_LAUNCH();
  for (int i = 0; i < K1; ++i) b->pl[i]->prepared = false;
  int rc;
  if (k == 0 && (rc = onemap_solve_sample(b, os))) return rc;
  launch_rollout_batch(reinterpret_cast<const RolloutArgs*>(b->d_desc + b->off_roll), K1, b->mode, b->N, b->T, nullptr,
                       b->stream);
  b->launches++;
  CHECK_LAUNCH();
  for (int i = 0; i < K1; ++i) b->pl[i]->pushed_direct = false;
  return B200MPPI_OK;
}

// The windowed rollout of every MODE_TDM planner of a batch (its kernel and its encoded tensor maps at the batch's
// window geometry WW x WH), checked before any work is issued; `fn` prefixes the messages.
static int stochastic_validate(b200mppi_batch* b, const char* fn, int* WW, int* WH) {
  size_t smem;
  rollout_win_geometry(b->T, WW, WH, &smem);
  *WH = rollout_win_batch_height(b->T);
  CU(cudaSetDevice(b->device));
  for (int i = b->nmap; i < (int)b->pl.size(); ++i) {
    b200mppi_planner* p = b->pl[i];
    const std::string who = std::string(fn) + ": planner " + std::to_string(i);
    // the generic rollout kernel's costs differ from the windowed kernel's in the last bit: no stand-in
    if (!planner_uses_window(p))
      return fail(B200MPPI_EINVAL, who + " does not take the windowed rollout kernel (B200MPPI_NO_WINDOW is set or its "
                                         "window does not fit shared memory)");
    if (!planner_tensor_maps(p, *WW, *WH))
      return fail(B200MPPI_EINVAL, who + ": the tensor maps of its sampled maps / masks could not be encoded");
  }
  return B200MPPI_OK;
}

// The MODE_TDM planners' (pl[nmap ..]) descriptors of the noise + controls, windowed rollout (+ tensor maps), CVaR and
// update launches at byte offset 0 of `h` (the layout of b->h_desc), indexed from nmap except the update's; *masks01:
// every planner's masks are 0 / 1.
static void stochastic_descs(b200mppi_batch* b, unsigned char* h, int WW, int WH, bool* masks01) {
  const int K1 = b->nmap, K2 = (int)b->pl.size() - K1, T = b->T;
  NoisePrepDesc* hn = reinterpret_cast<NoisePrepDesc*>(h + b->off_nprep);
  RolloutWinArgs* hw = reinterpret_cast<RolloutWinArgs*>(h + b->off_win);
  unsigned char* ht = h + b->off_tm;
  CvarDesc* hc = reinterpret_cast<CvarDesc*>(h + b->off_cvar);
  UpdateBatchDesc* hu = reinterpret_cast<UpdateBatchDesc*>(h + b->off_upd);
  *masks01 = true;
  for (int i = 0; i < K2; ++i) {
    b200mppi_planner* p = b->pl[K1 + i];
    const b200mppi_params& q = p->prm;
    hn[i] = NoisePrepDesc{p->states, p->noise, p->u_cur, p->noiseT, p->ctrl, p->reach_d, p->reach_slot ^ 1,
                          q.u_std[0], q.u_std[1], q.lambda_weight, q.u_std[0] * q.u_std[0], q.u_std[1] * q.u_std[1],
                          q.vrange[0], q.vrange[1], q.wrange[0], q.wrange[1]};
    hw[i] = RolloutWinArgs{};
    fill_rollout_params(p, hw[i].p);
    fill_win_args(p, WW, WH, hw[i]);
    fill_cost_dst(p, hw[i].dst, false);
    *masks01 = *masks01 && hw[i].masks01;
    std::memcpy(ht + (size_t)i * sizeof(b200mppi_planner::tmaps), p->tmaps, sizeof(b200mppi_planner::tmaps));
    hc[i] = CvarDesc{p->costs_nm, p->costs, p->n_local, p->n_local, p->M, cvar_numel(p->M, q.cvar_alpha), nullptr};
    // u_prev stays null: a stochastic solve does not alias it
    fill_update_apply(p, hu[K1 + i], b->u_d + (size_t)(K1 + i) * T * 2, nullptr);
  }
}

// A solve's stochastic part (planners [nmap, K)): per iteration ONE noise + controls launch, [first iteration: every TDM
// group's map sampling with the decisions of stage_sample_tdms], ONE windowed rollout launch over all (planner, map)
// units and ONE CVaR launch.  The reach statistics of all planners are read back behind one event, so the host waits
// once.
struct StochasticSolve {
  int WW = 0, WH = 0;                                  // the window geometry (stochastic_validate)
  bool masks01 = true;
  TdmGroups gr;
  std::vector<SamplePlan> plans;
  std::vector<b200mppi_planner*> ps;                   // planners by group
};

// the descriptors and sampler plans, one per TDM group (their host preparation may synchronise the stream), before the
// solve's one upload
static int stochastic_solve_plan(b200mppi_batch* b, StochasticSolve& ss) {
  b200mppi_planner* const* sp = b->pl.data() + b->nmap;
  const int K2 = (int)b->pl.size() - b->nmap;
  stochastic_descs(b, b->h_desc, ss.WW, ss.WH, &ss.masks01);
  ss.gr = batch_groups(b, b->nmap, (int)b->pl.size());
  const int G = ss.gr.size();
  ss.plans.resize(G);
  ss.ps.resize(K2);
  for (int j = 0; j < K2; ++j) ss.ps[j] = sp[ss.gr.members[j]];
  for (int g = 0; g < G; ++g) {
    const b200mppi_planner* p = sp[ss.gr.lead(g)];
    const int rc = plan_sampling(p->lin, p->ang, sample_alpha(p), b->stream, &ss.plans[g]);
    if (rc) return rc;
  }
  return B200MPPI_OK;
}

// the sampling of num_opt <= 0: the reference samples before its (empty) loop
static int stochastic_solve_presample(b200mppi_batch* b, StochasticSolve& ss) {
  const TdmGroups& gr = ss.gr;
  std::vector<const float*> reach(ss.ps.size(), nullptr);
  for (int g = 0; g < gr.size(); ++g) {
    const int rc = sample_finish_group(&ss.ps[gr.first[g]], &reach[gr.first[g]], gr.count(g), ss.plans[g], false,
                                       b->stream, &b->launches);
    if (rc) return rc;
  }
  return B200MPPI_OK;
}

static int stochastic_solve_iteration(b200mppi_batch* b, StochasticSolve& ss, int k) {
  b200mppi_planner* const* sp = b->pl.data() + b->nmap;
  const int K2 = (int)b->pl.size() - b->nmap, G = ss.gr.size();
  const TdmGroups& gr = ss.gr;
  cudaStream_t st = b->stream;
  int rc;
  launch_noise_prepare_batch(reinterpret_cast<const NoisePrepDesc*>(b->d_desc + b->off_nprep), K2, b->N, b->T,
                             sp[0]->npad, k, nullptr, st);
  b->launches++;
  CHECK_LAUNCH();
  for (int i = 0; i < K2; ++i) {                       // stage_noise
    sp[i]->reach_slot ^= 1;
    sp[i]->prepared = true;
    sp[i]->reach_valid = true;
  }
  if (k == 0) {                                        // stage_sample_tdms of every TDM group, one host wait
    std::vector<char> reads(K2), advanced(G);
    std::vector<const float*> reach(K2, nullptr);      // by group, as ps
    bool any = false;
    for (int i = 0; i < K2; ++i) {
      b200mppi_planner* p = sp[i];
      if (!(reads[i] = sample_reads_reach(p))) continue;
      CU(cudaMemcpyAsync(sample_reach_host(p), p->reach_d + p->reach_slot, sizeof(float), cudaMemcpyDeviceToHost, st));
      any = true;
    }
    if (any) CU(cudaEventRecord(b->ev, st));
    for (int g = 0; g < G; ++g) {                      // a fused group's advance, if any member waits for its reach
      bool wait = false;
      for (int j = gr.first[g]; j < gr.first[g + 1]; ++j) wait = wait || reads[gr.members[j]];
      if (!wait || !ss.plans[g].fused) continue;
      launch_plan_advance(ss.plans[g], 0, st);
      CHECK_LAUNCH();
      b->launches++;
      advanced[g] = 1;
    }
    if (any) CU(cudaEventSynchronize(b->ev));
    for (int j = 0; j < K2; ++j) reach[j] = reads[gr.members[j]] ? sample_reach_host(ss.ps[j]) : nullptr;
    for (int g = 0; g < G; ++g)
      if ((rc = sample_finish_group(&ss.ps[gr.first[g]], &reach[gr.first[g]], gr.count(g), ss.plans[g],
                                    advanced[g] != 0, st, &b->launches)))
        return rc;
  }
  CU(launch_rollout_win_batch(*reinterpret_cast<const RolloutWinArgs*>(b->h_desc + b->off_win),
                              reinterpret_cast<const RolloutWinArgs*>(b->d_desc + b->off_win), b->d_desc + b->off_tm,
                              K2, ss.masks01, nullptr, st));
  b->launches++;
  for (int i = 0; i < K2; ++i) { sp[i]->prepared = false; sp[i]->pushed_direct = false; }
  launch_cvar_batch(reinterpret_cast<const CvarDesc*>(b->d_desc + b->off_cvar), K2, b->N, b->M, st);
  b->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

// Every batch's solve: num_opt x (the one-map part's launches, the stochastic part's, then ONE update launch over all K
// planners), each part as described above; a batch of one kind issues only that kind's.  The descriptors of both parts
// are built on the host for this solve and uploaded with ONE copy from pinned staging before the first launch.
static int batch_solve_parts(b200mppi_batch* b) {
  const int K = (int)b->pl.size(), K1 = b->nmap;
  OnemapSolve os;
  StochasticSolve ss;
  int rc;
  if (K1 < K && (rc = stochastic_validate(b, "batch_solve", &ss.WW, &ss.WH))) return rc;
  CU(cudaSetDevice(b->device));
  cudaStream_t st = b->stream;
  if ((rc = batch_wait_members(b))) return rc;
  if (K1 > 0 && (rc = onemap_solve_plan(b, os))) return rc;
  if (K1 < K && (rc = stochastic_solve_plan(b, ss))) return rc;
  CU(cudaMemcpyAsync(b->d_desc, b->h_desc, b->desc_bytes, cudaMemcpyHostToDevice, st));
  const int num_opt = b->pl[0]->prm.num_opt;
  if (num_opt <= 0) {                                  // the reference samples before its (empty) loop
    if (K1 > 0 && (rc = onemap_solve_sample(b, os))) return rc;
    if (K1 < K && (rc = stochastic_solve_presample(b, ss))) return rc;
  }
  const UpdateBatchDesc* du = reinterpret_cast<const UpdateBatchDesc*>(b->d_desc + b->off_upd);
  for (int k = 0; k < num_opt; ++k) {
    if (K1 > 0 && (rc = onemap_solve_iteration(b, os, k))) return rc;
    if (K1 < K && (rc = stochastic_solve_iteration(b, ss, k))) return rc;
    launch_update_partial_batch(du, K, b->pl[0]->num_ctas, nullptr, st);
    b->launches++;
    CHECK_LAUNCH();
  }
  return B200MPPI_OK;
}

extern "C" int b200mppi_batch_solve(b200mppi_batch* b, float* u_out) {
  if (b && b->loop) return loop_busy("batch_solve");
  if (!b) return fail(B200MPPI_EINVAL, "null batch");
  int rc = batch_validate(b);
  if (rc) return rc;
  if ((rc = batch_solve_parts(b))) return rc;
  const size_t n = (size_t)b->T * 2, ubytes = b->pl.size() * n * sizeof(float);
  if (b->pl[0]->prm.num_opt <= 0)                      // u unchanged
    for (size_t i = 0; i < b->pl.size(); ++i)
      CU(cudaMemcpyAsync(b->u_d + i * n, b->pl[i]->u_cur, n * sizeof(float), cudaMemcpyDeviceToDevice, b->stream));
  CU(cudaMemcpyAsync(b->h_u, b->u_d, ubytes, cudaMemcpyDeviceToHost, b->stream));
  // the host waits for the whole batch: work issued afterwards on any member's stream sees its results
  CU(cudaStreamSynchronize(b->stream));
  if (u_out) std::memcpy(u_out, b->h_u, ubytes);
  return B200MPPI_OK;
}

// --------------------------------------------------------------------------------------------- visualisation rollouts
static int vis_count(const b200mppi_planner* p) {
  return p->cfg.num_vis_state_rollouts < 1 ? 1 : p->cfg.num_vis_state_rollouts;
}

// The batch's V, checked before any work is issued: every planner ready (what get_state_rollout checks), equal V, and V
// within each planner's sampled maps (MODE_TDM) or control rollouts.  `fn` prefixes the messages.
static int batch_vis_validate(b200mppi_batch* b, const std::string& fn, int* V) {
  const int V0 = vis_count(b->pl[0]);
  for (int i = 0; i < (int)b->pl.size(); ++i) {
    b200mppi_planner* p = b->pl[i];
    const std::string who = fn + ": planner " + std::to_string(i);
    const int rc = planner_check_ready(p);
    if (rc) return fail(rc, who + ": " + g_err);
    const int v = vis_count(p);
    if (v != V0)
      return fail(B200MPPI_EINVAL, who + " has num_vis_state_rollouts " + std::to_string(v) + ", planner 0 " +
                                       std::to_string(V0) + " (V must be equal)");
    const bool tdm = p->cfg.mode == B200MPPI_MODE_TDM;
    if (tdm ? v > p->lin->num_maps : v > p->n_local)
      return fail(B200MPPI_EINVAL, who + " has num_vis_state_rollouts " + std::to_string(v) + ", more than its " +
                                       std::to_string(tdm ? p->lin->num_maps : p->n_local) +
                                       (tdm ? " sampled maps" : " control rollouts"));
  }
  *V = V0;
  return B200MPPI_OK;
}

// planner p's visualisation rollouts with its RolloutParams at dp (device) into out (device, (V, T+1, 3))
static VisBatchDesc vis_desc(const b200mppi_planner* p, const RolloutParams* dp, float* out) {
  VisBatchDesc v{};
  v.p = dp;
  v.mode = p->cfg.mode; v.V = vis_count(p);
  if (p->cfg.mode != B200MPPI_MODE_BAREBONE) { v.lin_grid = p->lin->grid; v.ang_grid = p->ang->grid; }
  v.noise = p->noise; v.u_cur = p->u_cur; v.u_prev = p->u_prev; v.out = out;
  return v;
}

extern "C" int b200mppi_batch_get_state_rollout(b200mppi_batch* b, float* out, size_t bytes) {
  if (b && b->loop) return loop_busy("batch_get_state_rollout");
  if (!b) return fail(B200MPPI_EINVAL, "null batch");
  if (!out) return fail(B200MPPI_EINVAL, "batch_get_state_rollout: null output");
  int V = 0;
  int rc = batch_vis_validate(b, "batch_get_state_rollout", &V);
  if (rc) return rc;
  const int K = (int)b->pl.size();
  const size_t per = (size_t)V * (b->T + 1) * 3;
  if (bytes != (size_t)K * per * sizeof(float))
    return fail(B200MPPI_EINVAL, "batch_get_state_rollout: size mismatch (" + std::to_string(bytes) + " bytes, (K, V, "
                                 "T+1, 3) float32 is " + std::to_string((size_t)K * per * sizeof(float)) + ")");
  CU(cudaSetDevice(b->device));
  cudaStream_t st = b->stream;
  if ((rc = batch_wait_members(b))) return rc;
  RolloutParams* hp = reinterpret_cast<RolloutParams*>(b->h_desc + b->off_vis);
  VisBatchDesc* hv = reinterpret_cast<VisBatchDesc*>(b->h_desc + b->off_visd);
  const RolloutParams* dp = reinterpret_cast<const RolloutParams*>(b->d_desc + b->off_vis);
  for (int i = 0; i < K; ++i) {
    b200mppi_planner* p = b->pl[i];
    if (p->cfg.mode != B200MPPI_MODE_BAREBONE) {   // as get_state_rollout: the maps of a boxed solve are completed
      if ((rc = tdm_complete_grid(p->lin, st))) return rc;
      if ((rc = tdm_complete_grid(p->ang, st))) return rc;
    }
    hp[i] = RolloutParams{};
    fill_rollout_params(p, hp[i]);
    hv[i] = vis_desc(p, dp + i, p->state_rollout);
  }
  CU(cudaMemcpyAsync(b->d_desc + b->off_vis, b->h_desc + b->off_vis, b->vis_bytes, cudaMemcpyHostToDevice, st));
  launch_state_rollout_batch(reinterpret_cast<const VisBatchDesc*>(b->d_desc + b->off_visd), K, V, nullptr, 0, st);
  b->launches++;
  CHECK_LAUNCH();
  for (int i = 0; i < K; ++i)
    CU(cudaMemcpyAsync(out + (size_t)i * per, b->pl[i]->state_rollout, per * sizeof(float), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return B200MPPI_OK;
}

// --------------------------------------------------------------------------------------------- closed-loop trials
// A batch's planners run whole receding-horizon episodes on the device.  Only x0 (written by the plant kernel into the
// rollout descriptors) and the parity of the TDMs' generator-state double buffers change from step to step: every
// running planner has sampled its maps exactly s times before step s, so two sampler descriptor sets, one per parity,
// serve all steps.  Stopped planners are gated out of every launch by `active`; the host polls the count of running
// planners through pinned memory POLL steps behind the GPU and stops issuing once it reads zero.
constexpr int TRIAL_POLL = 4;

// one-map (MODE_DET_DYN, MODE_SPEED_MAP), stochastic (MODE_TDM), barebone (MODE_BAREBONE, no map) and mixed (one-map
// and MODE_TDM planners of a b200mppi_batch_create_mixed batch) trials
enum class TrialKind { onemap, stochastic, barebone, mixed };

// first: planner i's descriptors are tr[first[i] .. first[i + 1]): one each, or (seq) its episodes in a trial sequence
static int trial_validate(b200mppi_batch* b, TrialKind kind, const b200mppi_trial_desc* tr, int32_t max_steps,
                          const char* fn, const std::vector<int>& first, bool seq, std::vector<char>& in_place) {
  if (!tr) return fail(B200MPPI_EINVAL, std::string(fn) + ": null trial descriptors");
  if (max_steps < 1) return fail(B200MPPI_EINVAL, std::string(fn) + ": max_steps < 1");
  if (kind != TrialKind::barebone && b->mode == B200MPPI_MODE_BAREBONE)
    return fail(B200MPPI_EINVAL, "run_trials: planner 0 is MODE_BAREBONE (trials need traction maps: MODE_DET_DYN or "
                                 "MODE_SPEED_MAP batches)");
  int rc = batch_validate(b);
  if (rc) return rc;
  in_place.assign(first.back(), 0);
  for (int j = 0; j < first.back(); ++j) {
    const int i = (int)(std::upper_bound(first.begin(), first.end(), j) - first.begin()) - 1;
    const std::string who = std::string(fn) + ": planner " + std::to_string(i) +
                            (seq ? ", episode " + std::to_string(j - first[i]) : std::string());
    const b200mppi_trial_desc& d = tr[j];
    if (b->pl[i]->prm.num_opt < 1) return fail(B200MPPI_EINVAL, who + " has num_opt < 1");
    if (kind == TrialKind::barebone) {
      if (d.lin || d.ang)
        return fail(B200MPPI_EINVAL, who + ": traction grids given (barebone trials step the nominal unicycle: lin and "
                                           "ang must be NULL)");
      bool finite = std::isfinite(d.goal_tolerance);
      for (int c = 0; c < 3; ++c) finite = finite && std::isfinite(d.x0[c]);
      for (int c = 0; c < 2; ++c) finite = finite && std::isfinite(d.xgoal[c]);
      if (!finite) return fail(B200MPPI_EINVAL, who + ": start pose, goal or goal_tolerance not finite");
      if (!(d.dt > 0.0) || !std::isfinite(d.dt)) return fail(B200MPPI_EINVAL, who + ": dt not finite and positive");
      continue;
    }
    if (!d.lin || !d.ang || d.height < 1 || d.width < 1)
      return fail(B200MPPI_EINVAL, who + ": empty or missing traction grid");
    if (!(d.res > 0.0) || !std::isfinite(d.res) || !std::isfinite(d.xlo) || !std::isfinite(d.ylo) || !(d.dt > 0.0) ||
        !std::isfinite(d.dt))
      return fail(B200MPPI_EINVAL, who + ": grid res / limits or dt not finite and positive");
    if (!(d.x0[0] >= d.pxlim[0] && d.x0[0] <= d.pxlim[1] && d.x0[1] >= d.pylim[0] && d.x0[1] <= d.pylim[1]) ||
        !std::isfinite(d.x0[2]))
      return fail(B200MPPI_EINVAL, who + ": start pose outside the padded map limits");
    bool dev = false;
    if ((rc = trial_grid_source(d, b->device, who, &dev))) return rc;
    in_place[j] = dev;
  }
  return B200MPPI_OK;
}

// The launch classes of a trial batch's TDM groups: groups whose fused pairs share what one batched sampler launch fixes
// in its kernel variant and block shape -- the padded bins of both TDMs (the NW instantiation), the thread tile tx x ty
// and num_maps -- form one class, in the order of their first group.  Everything else (rows, cols, pitch, row segments,
// jump tables, boxes) each pair's CTAs read from its own descriptor, so a batch on one map geometry is one class.  A step
// issues one sampler launch per class (stochastic: and one state advance).
struct LaunchClasses {
  std::vector<int> groups;              // class c: groups[first[c] .. first[c + 1]), ascending
  std::vector<int> first;
  int size() const { return (int)first.size() - 1; }
  int count(int c) const { return first[c + 1] - first[c]; }
};

static LaunchClasses launch_classes(const std::vector<SamplePlan>& plans) {
  const int G = (int)plans.size();
  auto same = [](const SampleGridsV2Args& a, const SampleGridsV2Args& b) {
    return a.t[0].bpad == b.t[0].bpad && a.t[1].bpad == b.t[1].bpad && a.tx == b.tx && a.ty == b.ty &&
           a.num_maps == b.num_maps;
  };
  std::vector<int> of(G, -1), lead;
  for (int g = 0; g < G; ++g) {
    for (int c = 0; c < (int)lead.size() && of[g] < 0; ++c)
      if (same(plans[lead[c]].a[0], plans[g].a[0])) of[g] = c;
    if (of[g] < 0) { of[g] = (int)lead.size(); lead.push_back(g); }
  }
  LaunchClasses lc;
  lc.first.push_back(0);
  for (int c = 0; c < (int)lead.size(); ++c) {
    for (int g = 0; g < G; ++g)
      if (of[g] == c) lc.groups.push_back(g);
    lc.first.push_back((int)lc.groups.size());
  }
  return lc;
}

// One class's sampler launches in a trial: its shape, and (stochastic) the launch's tile rows and columns
struct TrialClass {
  SampleClassLaunch L{};
  int mrows = 0, ncact = 0;
};

// The planners of one kind in a trial call: the one-map planners pl[0 .. nmap) or the MODE_TDM planners pl[nmap .. K).
// Each kind's launches index its planners, groups and classes from lo (`active` too: active + lo).
struct TrialPart {
  int lo = 0, n = 0;
  TdmGroups gr;
  std::vector<SamplePlan> plans;
  std::vector<SampleGridsV2Args> set0;                 // parity 0, one per TDM group
  LaunchClasses lc;
  std::vector<TrialClass> cls;
  int G = 0, C = 0;                                    // groups whose pairs are sampled, sampler launch classes
  bool grouped = false;                                // shared pairs: the group-aware sampler launches
  // in the call's device buffer: the sampler sets of each parity, class c's pairs cls_d + lc.first[c], and the group
  // descriptors and members (null: no shared pair)
  const SampleGridsV2Args* set_d[2] = {};
  const SampleGridsV2Args* set_cur_d = nullptr;        // a loop's current set (LoopArgs::set_cur), read at every solve
  const int* cls_d = nullptr;
  const SampleGroupDesc* grp_d = nullptr;
  const int* mem_d = nullptr;
};

// A kind's trial sampler plans, one per TDM group (set0: parity 0, each pair's whole-map plan), and their launch classes.
// Every pair must be fused (identical generator streams, well-formed PMF at its alpha, lin != ang): its samplings join
// its class's one sampler launch.
static int trial_plans(b200mppi_batch* b, TrialPart& q, bool stochastic, const std::string& fn) {
  b200mppi_planner* const* pl = b->pl.data() + q.lo;
  q.G = q.gr.size();
  q.plans.resize(q.G);
  q.set0.resize(q.G);
  for (int g = 0; g < q.G; ++g) {
    const b200mppi_planner* p = pl[q.gr.lead(g)];
    const int rc = plan_sampling(p->lin, p->ang, stochastic ? sample_alpha(p) : BATCH_ALPHA, b->stream, &q.plans[g]);
    if (rc) return rc;
    if (!q.plans[g].fused)
      return fail(B200MPPI_EINVAL, fn + ": planner " + std::to_string(q.lo + q.gr.lead(g)) + ": its TDM pair cannot join "
                                   "the batch's one sampler launch (" + (stochastic ? "lin == ang, or " : "") +
                                   "map geometry, PMF or generator streams differ from planner 0's)");
    q.set0[g] = q.plans[g].a[0];
  }
  q.lc = launch_classes(q.plans);
  q.C = q.lc.size();
  q.grouped = q.gr.shared();
  q.cls.assign(q.C, TrialClass{});
  return B200MPPI_OK;
}

// The MODE_TDM planners' per-class launch sizes, and their parity-0 sets made the boxed launch's.
static int stochastic_trial_classes(b200mppi_batch* b, TrialPart& q, const std::string& fn) {
  b200mppi_planner* const* sp = b->pl.data() + q.lo;
  const TdmGroups& gr = q.gr;
  const LaunchClasses& lc = q.lc;
  // a class's sampler launch is sized for the largest box the static bound allows (reach_box_decide: at most 2 R / res + 5
  // cells a side) over its planners that sample a box: mrows tile rows x ncact tile columns with the boxed launch's maps
  // per CTA, each the largest over the class's pairs of what the pair's own tile size needs.  Whole-map steps loop over
  // such groups.  x0 moves during a trial, so R's rounding terms take their bounds from the padded map's limits (a box
  // exists only for an x0 inside them).
  std::vector<double> span(q.G, -1.0);                // per pair: cells a side + margin (-1: no planner gets a box)
  for (int i = 0; i < q.n; ++i) {
    ReachBoxConst c;
    fill_reach_const(sp[i], q.plans[gr.of[i]], &c);
    if (c.mode == 0) continue;
    const double w = (double)c.cols * (double)c.res, h = (double)c.rows * (double)c.res;
    const double A = std::fmax(std::fabs((double)c.pxl), std::fabs((double)c.pxl + w)) +
                     std::fmax(std::fabs((double)c.pyl), std::fabs((double)c.pyl + h));
    const double R = reach_radius(c, (double)c.T * std::fmax(std::fabs((double)c.vr0), std::fabs((double)c.vr1)), A,
                                  w + h);
    if (!(R >= 0.0)) continue;                        // that planner never gets a box
    span[gr.of[i]] = std::fmax(span[gr.of[i]], 2.0 * R / (double)c.res + 8.0);
  }
  for (int c = 0; c < q.C; ++c) {
    TrialClass& tc = q.cls[c];
    const SampleGridsV2Args& sg0 = q.plans[lc.groups[lc.first[c]]].a[0];
    for (int j = lc.first[c]; j < lc.first[c + 1]; ++j) {
      const int g = lc.groups[j];
      if (span[g] < 0.0) continue;
      const SampleGridsV2Args& sg = q.plans[g].a[0];
      const int nrow = (sg.rows + sg.tx - 1) / sg.tx, ncol = (sg.cols + sg.ty - 1) / sg.ty;
      const bool small = span[g] < (double)(sg.rows + sg.cols);
      tc.mrows = std::max(tc.mrows, small ? std::min(sg.tx, (int)span[g] / nrow + 2) : sg.tx);
      tc.ncact = std::max(tc.ncact, small ? std::min(sg.ty, (int)span[g] / ncol + 2) : sg.ty);
    }
    if (tc.mrows == 0) { tc.mrows = sg0.tx; tc.ncact = sg0.ty; }
    int gm_b = 128 / tc.ncact;                        // apply_box's maps per CTA for that many tile columns
    gm_b = std::max(1, std::min(std::min(gm_b, SG_GM_MAX), sg0.num_maps));
    // the boxed launch's row segments over the whole-map plan
    std::vector<const SampleGridsV2Args*> mem;
    for (int j = lc.first[c]; j < lc.first[c + 1]; ++j) {
      const int g = lc.groups[j];
      const b200mppi_tdm* l = sp[gr.lead(g)]->lin;
      SampleGridsV2Args& s0 = q.set0[g];
      s0.segs = l->box_segs; s0.seg_rows = l->box_seg_rows; s0.jump = l->jump_box_d;
      s0.write_states = 0;
      s0.gm = gm_b;
      if (!sample_box_batch_fits(s0, tc.ncact))
        return fail(B200MPPI_EINVAL, fn + ": planner " + std::to_string(q.lo + gr.lead(lc.groups[lc.first[c]])) +
                                     ": the batched sampler launch (" + std::to_string(tc.ncact) + " tile columns x " +
                                     std::to_string(gm_b) + " maps per CTA) does not fit a CTA");
      mem.push_back(&s0);
    }
    tc.L = sample_box_class_launch(mem.data(), (int)mem.size(), tc.mrows, tc.ncact);
  }
  return B200MPPI_OK;
}

// The one-map planners' per-class launch shapes over their whole-map plans
static void onemap_trial_classes(TrialPart& q) {
  for (int c = 0; c < q.C; ++c) {
    std::vector<const SampleGridsV2Args*> mem;
    for (int j = q.lc.first[c]; j < q.lc.first[c + 1]; ++j) mem.push_back(&q.set0[q.lc.groups[j]]);
    q.cls[c].L = sample_class_launch(mem.data(), (int)mem.size());
  }
}

// Byte offsets into a trial call's one device allocation, in the order trial_layout takes them
struct TrialLayout {
  struct Part { size_t set[2] = {}, grp = 0, mem = 0, cls = 0, cur = 0; };   // a kind's sampler sets (by parity),
  Part part[2];                                                     // group descriptors, members, class lists and
                                                                    // (loop) current set
  size_t box = 0, rec = 0, grec = 0, state = 0, con = 0, res = 0, loop = 0, clock = 0, task = 0, obs64 = 0, res_end = 0,
         tr = 0, act = 0, seq = 0, start = 0, slot0 = 0;
  size_t vis = 0, rflag = 0, head = 0;                 // head: the sections staged and uploaded with one copy
  std::vector<size_t> grid;                            // per slot
  size_t vrec = 0, xh = 0, uh = 0, lu = 0, obs = 0, total = 0;
};

// One trial call passed through its phases: the request, both kinds' parts, the layout and the buffers
struct TrialCall {
  // the request: batch_run_trials' arguments (S: max_steps; episodes null: one episode per planner)
  b200mppi_batch* b; TrialKind kind; const b200mppi_trial_desc* trials; int S;
  double* xhist; float* uhist; b200mppi_trial_result* results; int32_t* contact_steps;
  int record_every; float* rollouts; size_t rollout_bytes; const int32_t* episodes; bool reset_x0;
  std::string fn;                                      // prefixes the refusals
  bool barebone = false, seq = false, record = false, rec_seq = false;
  int K = 0, K1 = 0, K2 = 0, nslot = 0, max_episodes = 1;   // the one-map planners, then the MODE_TDM planners
  std::vector<int> first;                              // planner i's slots: first[i] .. first[i + 1]
  std::vector<char> in_place;                          // slots whose grids are realisation planes, read where they are
  int V = 0, R = 0;                                    // recording: rollouts per record, records per slot
  size_t per = 0, rec_bytes = 0;                       // floats of one record, bytes of the device's records
  int WW = 0, WH = 0;                                  // the stochastic planners' window geometry
  bool masks01 = true;
  TrialPart P[2];                                      // one-map, stochastic
  TrialLayout L;
  unsigned char* d = nullptr;                          // the device buffer (L)
  unsigned char* h = nullptr;                          // its pinned staging: the head, then the histories
  PlantArgs pa{};
  SeqArgs sa{};
  RolloutWinArgs g0{};                                 // the stochastic planners' first windowed rollout descriptor
  // a device loop (b200mppi_batch_loop_open) instead of a trial: no descriptors, grids, histories or plant step; per
  // planner its padded limits (K x 4, null for barebone) and its row in the caller's arrays (null: its index)
  bool loop = false;
  const double* limits = nullptr;
  const int32_t* rows = nullptr;
  int O = 0;                                           // a loop's obstacle capacity per planner (barebone)
};

// What a device loop checks in place of trial_validate: a batch that can solve, num_opt >= 1, padded limits for every
// planner that has a map, and rows that are a permutation of 0 .. K-1
static int loop_validate(TrialCall& t) {
  b200mppi_batch* b = t.b;
  if (!t.barebone && b->mode == B200MPPI_MODE_BAREBONE)
    return fail(B200MPPI_EINVAL, t.fn + ": planner 0 is MODE_BAREBONE (its loops are of kind B200MPPI_TRIALS_BAREBONE)");
  int rc = batch_validate(b);
  if (rc) return rc;
  if (!t.barebone && !t.limits) return fail(B200MPPI_EINVAL, t.fn + ": null padded limits");
  std::vector<char> seen(t.K, 0);
  for (int i = 0; i < t.K; ++i) {
    const std::string who = t.fn + ": planner " + std::to_string(i);
    if (b->pl[i]->prm.num_opt < 1) return fail(B200MPPI_EINVAL, who + " has num_opt < 1");
    for (int c = 0; c < 4 && !t.barebone; ++c)
      if (std::isnan(t.limits[4 * i + c])) return fail(B200MPPI_EINVAL, who + ": padded limit is NaN");
    const int r = t.rows ? t.rows[i] : i;
    if (r < 0 || r >= t.K || seen[r]) return fail(B200MPPI_EINVAL, who + ": row " + std::to_string(r) + " out of range "
                                                                 "or taken twice (rows must be a permutation of 0 .. K-1)");
    seen[r] = 1;
  }
  return B200MPPI_OK;
}

// Everything a trial call checks before it allocates or issues anything
static int trial_call_validate(TrialCall& t) {
  b200mppi_batch* b = t.b;
  const bool stochastic = t.kind == TrialKind::stochastic, mixed = t.kind == TrialKind::mixed;
  t.barebone = t.kind == TrialKind::barebone;
  t.seq = t.episodes != nullptr;
  t.fn = t.loop ? "loop_open" : t.seq ? (t.barebone ? "run_barebone_trial_sequences" : "run_trial_sequences") : stochastic ? "run_stochastic_trials"
         : t.barebone ? "run_barebone_trials" : mixed ? "run_mixed_trials" : "run_trials";
  const std::string& fn = t.fn;
  t.K = (int)b->pl.size();
  t.K1 = b->nmap;
  t.K2 = t.K - t.K1;
  t.first.assign(t.K + 1, 0);
  for (int i = 0; i < t.K; ++i) {
    const int E = t.seq ? t.episodes[i] : 1;
    if (E < 1)
      return fail(B200MPPI_EINVAL, fn + ": planner " + std::to_string(i) + ": episode count " + std::to_string(E) + " < 1");
    if ((int64_t)t.first[i] + E > (1 << 24))
      return fail(B200MPPI_EINVAL, fn + ": more than 2^24 episodes in all");
    t.first[i + 1] = t.first[i] + E;
    t.max_episodes = std::max(t.max_episodes, E);
  }
  if ((int64_t)t.max_episodes * t.S > INT32_MAX)
    return fail(B200MPPI_EINVAL, fn + ": max_steps x the largest episode count exceeds 2^31 - 1 steps");
  if (b->mixed && !mixed)
    return fail(B200MPPI_EINVAL, fn + ": a mixed batch (b200mppi_batch_create_mixed) runs its trials with "
                                 "b200mppi_batch_run_mixed_trials (kind B200MPPI_TRIALS_MIXED)");
  if (!b->mixed && mixed)
    return fail(B200MPPI_EINVAL, fn + ": planner 0 is " + mode_name(b->mode) + " in a batch that is not mixed (mixed "
                                 "trials run batches made by b200mppi_batch_create_mixed)");
  if (t.barebone && b->mode != B200MPPI_MODE_BAREBONE)
    return fail(B200MPPI_EINVAL, fn + ": planner 0 is " + mode_name(b->mode) + " (barebone trials run MODE_BAREBONE "
                                 "batches; b200mppi_batch_run_trials and b200mppi_batch_run_stochastic_trials run the "
                                 "others)");
  if (b->stochastic && t.kind == TrialKind::onemap)
    return fail(B200MPPI_EINVAL, "run_trials: planner 0 is MODE_TDM (trials run det-dynamics or speed-map batches: a "
                                 "stochastic solve sizes each planner's map-sampling box on the host)");
  if (!b->stochastic && stochastic)
    return fail(B200MPPI_EINVAL, fn + ": planner 0 is " + mode_name(b->mode) +
                                     " (stochastic trials run MODE_TDM batches; b200mppi_batch_run_trials runs the others)");
  int rc = t.loop ? loop_validate(t) : trial_validate(b, t.kind, t.trials, t.S, fn.c_str(), t.first, t.seq, t.in_place);
  if (rc) return rc;
  if (!t.loop && (!t.xhist || !t.uhist || !t.results || (t.barebone && !t.contact_steps)))
    return fail(B200MPPI_EINVAL, fn + ": null output buffer");
  t.nslot = t.first[t.K];
  t.record = t.record_every > 0;
  t.rec_seq = t.record && t.seq;                       // records gated per planner on the device (SeqArgs::rec_flag)
  if (t.record) {
    // bytes of the device's records (per slot) and of the caller's (K, max_episodes) slabs, so a sequence's records
    // need no re-layout on the host (one episode per planner: the same two sizes)
    if ((rc = batch_vis_validate(b, fn, &t.V))) return rc;
    t.R = (t.S + t.record_every - 1) / t.record_every;
    t.per = (size_t)t.V * (b->T + 1) * 3;
    if ((double)t.K * t.max_episodes * t.R * t.per * sizeof(float) > 4e18)
      return fail(B200MPPI_EINVAL, fn + ": the records exceed 4e18 bytes");
    t.rec_bytes = (size_t)t.nslot * t.R * t.per * sizeof(float);
    const size_t out_bytes = (size_t)t.K * t.max_episodes * t.R * t.per * sizeof(float);
    if (!t.rollouts || t.rollout_bytes != out_bytes)
      return fail(B200MPPI_EINVAL, fn + ": rollouts buffer of " + std::to_string(t.rollout_bytes) + " bytes, the records " +
                                   (t.seq ? "(K, Emax" : "(K") + ", R, V, T+1, 3) float32 need " + std::to_string(out_bytes));
  }
  if (t.K2 > 0 && (rc = stochastic_validate(b, fn.c_str(), &t.WW, &t.WH))) return rc;
  return B200MPPI_OK;
}

// The sampler plans and launch classes of both kinds (their host preparation may synchronise the stream): every TDM
// group's pair must join the one launch of its class.  Groups of more than one planner (shared pairs) take the
// group-aware sampler launches.
static int trial_call_plan(TrialCall& t) {
  b200mppi_batch* b = t.b;
  CU(cudaSetDevice(b->device));
  t.P[0].n = t.K1; t.P[1].lo = t.K1; t.P[1].n = t.K2;
  for (TrialPart& q : t.P) q.gr = batch_groups(b, q.lo, q.lo + q.n);
  int rc;
  if (t.K2 > 0 && ((rc = trial_plans(b, t.P[1], true, t.fn)) || (rc = stochastic_trial_classes(b, t.P[1], t.fn))))
    return rc;
  if (t.K1 > 0 && !t.barebone) {
    if ((rc = trial_plans(b, t.P[0], false, "run_trials"))) return rc;
    onemap_trial_classes(t.P[0]);
  }
  return batch_wait_members(b);
}

static TrialLayout trial_layout(const TrialCall& t) {
  const size_t K = t.K, K2 = t.K2, nslot = t.nslot, S = t.S, szs = sizeof(SampleGridsV2Args);
  const size_t nres = t.seq ? nslot : 0;               // sequence-only sections: per-slot results and start poses
  const TrialPart* P = t.P;
  TrialLayout L;
  TrialLayout::Part& om = L.part[0];
  TrialLayout::Part& sto = L.part[1];
  // the batch's descriptors in b->h_desc's layout, where the one-map parity-0 sampler set is a section of its own
  Sections s{t.b->desc_bytes};
  om.set[0] = t.b->off_sample;
  sto.set[0] = s.take(P[1].G * szs);
  sto.set[1] = s.take(P[1].G * szs);
  om.set[1] = s.take(P[0].G * szs);
  L.box = s.take(K2 * sizeof(SampleBoxDesc));
  L.rec = s.take(K2 * 5 * sizeof(int));
  L.grec = s.take((P[1].grouped ? P[1].G : 0) * 5 * sizeof(int));   // stochastic shared pairs' group records
  // one section each of group descriptors, members and class lists, the one-map kind's entries first
  const size_t ngrp0 = P[0].grouped ? P[0].G : 0, nmem0 = P[0].grouped ? P[0].n : 0;
  om.grp = s.take((ngrp0 + (P[1].grouped ? P[1].G : 0)) * sizeof(SampleGroupDesc));
  om.mem = s.take((nmem0 + (P[1].grouped ? P[1].n : 0)) * sizeof(int));
  om.cls = s.take((size_t)(P[0].G + P[1].G) * sizeof(int));
  sto.grp = om.grp + ngrp0 * sizeof(SampleGroupDesc);
  sto.mem = om.mem + nmem0 * sizeof(int);
  sto.cls = om.cls + P[0].G * sizeof(int);
  L.state = s.take(K * sizeof(TrialState));
  L.con = s.take((t.barebone ? nslot : 0) * sizeof(int));   // barebone contacts, per slot
  L.res = s.take(nres * sizeof(TrialState));
  L.loop = s.take((t.loop ? K : 0) * sizeof(LoopState));   // a loop's per-planner counters and poses
  L.clock = s.take((t.loop ? 2 : 0) * sizeof(int));   // a loop's solve clock (LoopClock)
  L.task = s.take((t.loop ? K : 0) * sizeof(LoopTask));   // a loop's task updates (LoopTaskArgs) and their float64
  L.obs64 = s.take((t.loop ? K * t.O * 3 : 0) * sizeof(double));   // obstacle triples: read back at close
  L.res_end = s.end;
  L.tr = s.take(nslot * sizeof(TrialDev));
  L.act = s.take((K + 1) * sizeof(int));               // active (K), the count of running planners
  L.seq = s.take((t.seq ? 2 * K + 1 : 0) * sizeof(int));     // first (K + 1), episode (K)
  L.start = s.take(nres * 3 * sizeof(double));
  L.vis = s.take((t.record ? K : 0) * sizeof(VisBatchDesc));
  L.rflag = s.take((t.rec_seq ? K : 0) * sizeof(int));
  om.cur = s.take((t.loop ? P[0].G : 0) * szs);        // a loop's current sampler sets and staged reach slots
  sto.cur = s.take((t.loop ? P[1].G : 0) * szs);
  L.slot0 = s.take((t.loop ? 2 * K2 : 0) * sizeof(int));
  L.head = s.end;
  // The pinned staging holds the head and the histories only.  The float64 ground-truth grids (tens of MB for a batch
  // of large maps) are copied straight from the caller's arrays, and a slot whose grids are planes of a realisation set
  // has no grid section: the plant reads the planes.  The written records (of K * R * V * (T+1) * 12 bytes, 145 MB for
  // K 8, 150 steps, V 100, T 100) are copied straight into the caller's array.
  L.grid.resize(nslot);
  for (size_t j = 0; j < nslot; ++j)
    L.grid[j] = s.take(t.barebone || t.loop || t.in_place[j] ? 0 : 2 * (size_t)t.trials[j].height * t.trials[j].width * sizeof(double));
  L.vrec = s.take(t.rec_bytes);                        // (slots, R, V, T+1, 3)
  L.xh = s.take((t.loop ? 0 : nslot * (S + 1) * 3) * sizeof(double));
  L.uh = s.take(nslot * S * 2 * sizeof(float));
  L.lu = s.take((t.loop ? K * t.b->T * 2 : 0) * sizeof(float));   // a loop's own (K, T, 2) controls
  L.obs = s.take((t.loop ? K * t.O * 3 : 0) * sizeof(float));      // the obstacles a barebone loop's rollouts read
  L.total = s.end;
  return L;
}

// A barebone loop's (O, 3) obstacle slice of planner i
static float* loop_obstacles(const TrialCall& t, int i) {
  return reinterpret_cast<float*>(t.d + t.L.obs) + (size_t)i * t.O * 3;
}

// Fills the pinned staging's head (the batch's descriptors, per-planner and per-slot trial state, box, vis and sequence
// descriptors, both parities' sampler sets, group descriptors and members) and uploads it and the host grids.
static int trial_call_stage(TrialCall& t) {
  b200mppi_batch* b = t.b;
  const TrialLayout& L = t.L;
  unsigned char* d = t.d;
  unsigned char* h = t.h;
  const int K = t.K, K1 = t.K1, R = t.R;
  const std::vector<int>& first = t.first;
  const b200mppi_trial_desc* trials = t.trials;
  if (K1 > 0) onemap_descs(b, h);
  if (t.K2 > 0) stochastic_descs(b, h, t.WW, t.WH, &t.masks01);
  SampleBoxDesc* hb = reinterpret_cast<SampleBoxDesc*>(h + L.box);
  TrialState* hst = reinterpret_cast<TrialState*>(h + L.state);
  TrialDev* ht = reinterpret_cast<TrialDev*>(h + L.tr);
  int* hact = reinterpret_cast<int*>(h + L.act);
  int* dact = reinterpret_cast<int*>(d + L.act);
  // the rollout descriptors whose x0 the plant step writes: RolloutArgs (one-map), RolloutWinArgs (stochastic)
  RolloutArgs* dr = reinterpret_cast<RolloutArgs*>(d + b->off_roll);
  RolloutWinArgs* dw = reinterpret_cast<RolloutWinArgs*>(d + b->off_win);
  int* hcon = reinterpret_cast<int*>(h + L.con);
  VisBatchDesc* hv = reinterpret_cast<VisBatchDesc*>(h + L.vis);
  float* drec = reinterpret_cast<float*>(d + L.vrec);
  for (int i = 0; i < K; ++i) {
    b200mppi_planner* p = b->pl[i];
    const bool sto = i >= K1;
    const int r = i - K1;                              // a stochastic planner's index in its kind's launches
    if (t.record)                                      // x0 from the record the plant step writes; record 0 of slot 0
      hv[i] = vis_desc(p, sto ? &dw[r].p : &dr[i].p, drec + (size_t)first[i] * R * t.per);
    if (t.rec_seq) reinterpret_cast<int*>(h + L.rflag)[i] = 1;
    hst[i] = TrialState{};
    for (int c = 0; c < 3; ++c) hst[i].x[c] = t.loop ? (double)p->prm.x0[c] : trials[first[i]].x0[c];
    hact[i] = 1;
    if (t.loop) {                                      // from the pose of the params the batch's descriptors were built from
      LoopState& ls = reinterpret_cast<LoopState*>(h + L.loop)[i];
      ls = LoopState{};
      for (int c = 0; c < 3; ++c) { ls.x[c] = p->prm.x0[c]; ls.x0[c] = p->prm.x0[c]; }
      ls.bounded = !t.barebone;
      if (ls.bounded) {
        const double* lim = t.limits + 4 * i;
        ls.pxlim[0] = lim[0]; ls.pxlim[1] = lim[1]; ls.pylim[0] = lim[2]; ls.pylim[1] = lim[3];
      }
      ls.row = t.rows ? t.rows[i] : i;
      TrialDev& td = ht[i];                            // what the loop kernels read: the shift, the next x0 and window
      td = TrialDev{};
      td.u_cur = p->u_cur;
      td.x0_out = sto ? dw[r].p.x0 : dr[i].p.x0;
      if (sto) {
        const b200mppi_tdm* l = p->lin;
        td.win = &dw[r].WW;
        td.win_pxl = l->pxl[0]; td.win_pyl = l->pyl[0]; td.win_res = l->res; td.win_rows = l->rows; td.win_cols = l->cols;
      }
      // where the goal and obstacle calls write; a barebone planner reads its obstacles from its slice of the loop's
      // buffer, filled with its current ones below (no capacity: the descriptor is left as it is, with no obstacles)
      LoopTask& lt = reinterpret_cast<LoopTask*>(h + L.task)[i];
      lt = LoopTask{};
      lt.xgoal_out = sto ? dw[r].p.xgoal : dr[i].p.xgoal;
      if (t.barebone) {
        lt.num_obstacles_out = &dr[i].num_obstacles;
        if (t.O > 0) reinterpret_cast<RolloutArgs*>(h + b->off_roll)[i].obstacles = loop_obstacles(t, i);
      }
    }
    for (int j = first[i]; j < first[i + 1] && !t.loop; ++j) {    // the planner's episodes: one, or its sequence
      const b200mppi_trial_desc& q = trials[j];
      if (t.barebone) hcon[j] = 0;
      TrialDev& td = ht[j];
      td = TrialDev{};
      td.dt = q.dt; td.xgoal[0] = q.xgoal[0]; td.xgoal[1] = q.xgoal[1]; td.tol = q.goal_tolerance;
      td.u_cur = p->u_cur;
      if (t.barebone) {                                // lin null: nominal unicycle, no map; contacts counted
        td.x0_out = dr[i].p.x0;
        td.obstacles = p->obstacles; td.num_obstacles = p->num_obstacles;
        continue;
      }
      const double* dg = reinterpret_cast<const double*>(d + L.grid[j]);
      td.lin = t.in_place[j] ? q.lin : dg;
      td.ang = t.in_place[j] ? q.ang : dg + (size_t)q.height * q.width;
      td.H = q.height; td.W = q.width;
      td.xlo = q.xlo; td.ylo = q.ylo; td.res = q.res;
      td.pxlim[0] = q.pxlim[0]; td.pxlim[1] = q.pxlim[1]; td.pylim[0] = q.pylim[0]; td.pylim[1] = q.pylim[1];
      if (!sto) {
        td.x0_out = dr[i].p.x0;                        // win stays null: one-map rollouts have no window
        continue;
      }
      const b200mppi_tdm* l = p->lin;
      td.x0_out = dw[r].p.x0;
      td.win = &dw[r].WW;
      td.win_pxl = l->pxl[0]; td.win_pyl = l->pyl[0]; td.win_res = l->res; td.win_rows = l->rows; td.win_cols = l->cols;
    }
    if (!sto) continue;
    reinterpret_cast<CvarDesc*>(h + b->off_cvar)[r].active = dact + i;
    hb[r] = SampleBoxDesc{{}, dw[r].p.x0, p->reach_d, p->reach_slot ^ 1, reinterpret_cast<int*>(d + L.rec) + 5 * r,
                          p->lin->jump_tile_d};
    fill_reach_const(p, t.P[1].plans[t.P[1].gr.of[r]], &hb[r].c);
  }
  if (t.seq) {                                         // slots that never run keep NOT_RUN and 0 steps
    int* hseq = reinterpret_cast<int*>(h + L.seq);
    double* hstart = reinterpret_cast<double*>(h + L.start);
    TrialState* hres = reinterpret_cast<TrialState*>(h + L.res);
    std::copy(first.begin(), first.end(), hseq);
    std::fill(hseq + K + 1, hseq + 2 * K + 1, 0);
    for (int j = 0; j < t.nslot; ++j) {
      hres[j] = TrialState{};
      hres[j].status = B200MPPI_TRIAL_NOT_RUN;
      for (int c = 0; c < 3; ++c) hstart[3 * j + c] = trials[j].x0[c];
    }
    int* dseq = reinterpret_cast<int*>(d + L.seq);
    t.sa = SeqArgs{dseq, dseq + K + 1, reinterpret_cast<const double*>(d + L.start),
                   reinterpret_cast<TrialState*>(d + L.res), t.reset_x0 ? 1 : 0};
    if (t.rec_seq) {
      static_assert(sizeof(VisBatchDesc) % sizeof(float*) == 0, "rec_stride counts float* slots");
      t.sa.rec_flag = reinterpret_cast<int*>(d + L.rflag);
      t.sa.rec_out = &reinterpret_cast<VisBatchDesc*>(d + L.vis)->out;
      t.sa.rec = drec;
      t.sa.rec_per = (long long)t.per;
      t.sa.rec_every = t.record_every; t.sa.rec_R = R; t.sa.rec_stride = (int)(sizeof(VisBatchDesc) / sizeof(float*));
    }
  }
  for (int k = 0; k < 2; ++k) {
    TrialPart& q = t.P[k];
    const TrialLayout::Part& o = L.part[k];
    SampleGridsV2Args* hs0 = reinterpret_cast<SampleGridsV2Args*>(h + o.set[0]);
    SampleGridsV2Args* hs1 = reinterpret_cast<SampleGridsV2Args*>(h + o.set[1]);
    for (int g = 0; g < q.G; ++g) {
      // parity 1: the pair samples from the buffers parity 0 wrote into
      hs0[g] = hs1[g] = q.set0[g];
      for (SampleTdm& td : hs1[g].t) {
        uint64_t* in = td.states_out;
        td.states_out = const_cast<uint64_t*>(td.states);
        td.states = in;
      }
    }
    SampleGroupDesc* hg = reinterpret_cast<SampleGroupDesc*>(h + o.grp);
    for (int g = 0; g < q.G && q.grouped; ++g)
      hg[g] = SampleGroupDesc{q.gr.first[g], q.gr.count(g), k == 1 ? reinterpret_cast<int*>(d + L.grec) + 5 * g : nullptr};
    if (q.grouped) std::copy(q.gr.members.begin(), q.gr.members.end(), reinterpret_cast<int*>(h + o.mem));
    std::copy(q.lc.groups.begin(), q.lc.groups.end(), reinterpret_cast<int*>(h + o.cls));
    q.set_d[0] = reinterpret_cast<const SampleGridsV2Args*>(d + o.set[0]);
    q.set_d[1] = reinterpret_cast<const SampleGridsV2Args*>(d + o.set[1]);
    if (t.loop) {                                      // the current set of solve 0: parity 0
      std::copy(hs0, hs0 + q.G, reinterpret_cast<SampleGridsV2Args*>(h + o.cur));
      q.set_cur_d = reinterpret_cast<const SampleGridsV2Args*>(d + o.cur);
    }
    q.cls_d = reinterpret_cast<const int*>(d + o.cls);
    q.grp_d = q.grouped ? reinterpret_cast<const SampleGroupDesc*>(d + o.grp) : nullptr;
    q.mem_d = q.grouped ? reinterpret_cast<const int*>(d + o.mem) : nullptr;
  }
  hact[K] = K;
  if (t.loop) {                                        // the clock at 0, and the staged slots the clock rewrites from
    std::fill_n(reinterpret_cast<int*>(h + L.clock), 2, 0);
    int* slot0 = reinterpret_cast<int*>(h + L.slot0);
    const NoisePrepDesc* hn = reinterpret_cast<const NoisePrepDesc*>(h + b->off_nprep);
    for (int r = 0; r < t.K2; ++r) { slot0[r] = hn[r].slot; slot0[t.K2 + r] = hb[r].slot; }
    std::memset(h + L.obs64, 0, (size_t)K * t.O * 3 * sizeof(double));
  }
  if (t.K2 > 0) t.g0 = *reinterpret_cast<const RolloutWinArgs*>(h + b->off_win);
  cudaStream_t st = b->stream;
  CU(cudaMemcpyAsync(d, h, L.head, cudaMemcpyHostToDevice, st));
  for (int i = 0; i < K && t.loop && t.O > 0; ++i) {
    const b200mppi_planner* p = b->pl[i];
    if (p->num_obstacles > 0)
      CU(cudaMemcpyAsync(loop_obstacles(t, i), p->obstacles, (size_t)p->num_obstacles * 3 * sizeof(float),
                         cudaMemcpyDeviceToDevice, st));
  }
  for (int j = 0; j < t.nslot && !t.barebone && !t.loop; ++j) {  // pageable sources: staged by the driver before the call returns
    if (t.in_place[j]) continue;
    const size_t bytes = (size_t)trials[j].height * trials[j].width * sizeof(double);
    CU(cudaMemcpyAsync(d + L.grid[j], trials[j].lin, bytes, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d + L.grid[j] + bytes, trials[j].ang, bytes, cudaMemcpyHostToDevice, st));
  }
  t.pa = PlantArgs{reinterpret_cast<const TrialDev*>(d + L.tr), reinterpret_cast<TrialState*>(d + L.state), dact,
                   dact + K, reinterpret_cast<double*>(d + L.xh), reinterpret_cast<float*>(d + L.uh), K, b->T, t.S, 0,
                   t.barebone ? reinterpret_cast<int*>(d + L.con) : nullptr};
  CU(cudaStreamSynchronize(st));                      // the staging is read by the upload above
  return B200MPPI_OK;
}

// The launches of step s but its plant step (trial_call_plant; a device loop runs the caller's plant), each counted where
// it is issued
static int trial_call_step(TrialCall& t, int s) {
  b200mppi_batch* b = t.b;
  const unsigned char* d = t.d;
  cudaStream_t st = b->stream;
  const int K = t.K, K1 = t.K1, K2 = t.K2, N = b->N, T = b->T, num_opt = b->pl[0]->prm.num_opt;
  const TrialPart& om = t.P[0];
  const TrialPart& sto = t.P[1];
  const int* dact = t.pa.active;
  const int* dact2 = dact + K1;                        // the stochastic launches' active flags
  const RolloutWinArgs* dw = reinterpret_cast<const RolloutWinArgs*>(d + b->off_win);
  const SampleBoxDesc* db = reinterpret_cast<const SampleBoxDesc*>(d + t.L.box);
  // a loop's solves read the current sets and slots its solve clock prepares (LoopClock): nothing of solve s is
  // passed by value, so a captured solve replays as any later one
  const SampleGridsV2Args* om_set = t.loop ? om.set_cur_d : om.set_d[s & 1];
  const SampleGridsV2Args* sto_set = t.loop ? sto.set_cur_d : sto.set_d[s & 1];
  for (int k = 0; k < num_opt; ++k) {
    if (K1 > 0) {
      launch_sample_noise_batch(reinterpret_cast<const NoiseDesc*>(d), K1, N, T, dact, st);
      b->launches++;
      CHECK_LAUNCH();
      for (int c = 0; c < om.C && k == 0; ++c) {
        launch_sample_grids_v2_batch(om.cls[c].L, om_set, om.lc.count(c), om.cls_d + om.lc.first[c], dact, st,
                                     om.grp_d, om.mem_d);
        b->launches++;
        CHECK_LAUNCH();
      }
      launch_rollout_batch(reinterpret_cast<const RolloutArgs*>(d + b->off_roll), K1, b->mode, N, T, dact, st);
      b->launches++;
      CHECK_LAUNCH();
    }
    if (K2 > 0) {
      const int iter = (t.loop ? 0 : s * num_opt) + k;   // every planner's reach slot toggles once per iteration
      launch_noise_prepare_batch(reinterpret_cast<const NoisePrepDesc*>(d + b->off_nprep), K2, N, T, b->pl[0]->npad,
                                 iter, dact2, st);
      b->launches++;
      CHECK_LAUNCH();
      for (int c = 0; c < sto.C && k == 0; ++c) {
        const TrialClass& tc = sto.cls[c];
        const SampleGridsV2Args& g0c = sto.set0[sto.lc.groups[sto.lc.first[c]]];
        const int* cls = sto.cls_d + sto.lc.first[c];
        launch_sample_grids_v2_box_batch(tc.L, sto_set, db, sto.lc.count(c), cls, dact2, iter, tc.mrows,
                                         tc.ncact, st, sto.grp_d, sto.mem_d);
        b->launches++;
        CHECK_LAUNCH();
        launch_advance_states_batch(sto_set, db, sto.lc.count(c), cls, g0c.tx, g0c.ty, g0c.num_maps, dact2, st,
                                    sto.grp_d, sto.mem_d);
        b->launches++;
        CHECK_LAUNCH();
      }
      CU(launch_rollout_win_batch(t.g0, dw, d + b->off_tm, K2, t.masks01, dact2, st));
      b->launches++;
      launch_cvar_batch(reinterpret_cast<const CvarDesc*>(d + b->off_cvar), K2, N, b->M, st);
      b->launches++;
      CHECK_LAUNCH();
    }
    launch_update_partial_batch(reinterpret_cast<const UpdateBatchDesc*>(d + b->off_upd), K, b->pl[0]->num_ctas, dact,
                                st);
    b->launches++;
    CHECK_LAUNCH();
  }
  // a sequence's episodes start at steps only the device knows: a recording sequence issues the record launches at
  // every step, gated per planner by the flags the previous plant step set, each writing where its descriptor points
  if (t.record && (t.seq || s % t.record_every == 0)) {
    const int* rflag = t.seq ? t.sa.rec_flag : dact;
    for (int c = 0; c < sto.C; ++c) {                 // from the pre-call states this step's sampling read
      const TrialClass& tc = sto.cls[c];
      launch_sample_grids_v2_complete_batch(tc.L, sto.set_d[s & 1], db, sto.lc.count(c), sto.cls_d + sto.lc.first[c],
                                            rflag + K1, t.V, tc.mrows, tc.ncact, st, sto.grp_d, sto.mem_d);
      b->launches++;
      CHECK_LAUNCH();
    }
    launch_state_rollout_batch(reinterpret_cast<const VisBatchDesc*>(d + t.L.vis), K, t.V, rflag,
                               t.seq ? 0 : (size_t)(s / t.record_every) * t.per, st);
    b->launches++;
    CHECK_LAUNCH();
  }
  return B200MPPI_OK;
}

// The plant step that ends trial step s
static int trial_call_plant(TrialCall& t, int s) {
  cudaStream_t st = t.b->stream;
  t.pa.step = s;
  if (t.seq) launch_plant_step_seq(t.pa, t.sa, st);
  else launch_plant_step(t.pa, st);
  t.b->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

// Leaves every planner and every TDM group's pair as after the host loop in which planner i solved ran[i] times, the
// last time from x0[3 i ..]; t.h holds the box records read back.  A planner that never solved is left as it was.
static void trial_commit_planners(TrialCall& t, const std::vector<int>& ran, const std::vector<float>& x0) {
  const TrialLayout& L = t.L;
  const unsigned char* h = t.h;
  const int K1 = t.K1, num_opt = t.b->pl[0]->prm.num_opt;
  const int* hrec = reinterpret_cast<const int*>(h + L.rec);
  for (int i = 0; i < t.K; ++i) {
    // host state as after ran[i] solves: the reach slot toggled once per iteration, the last solve's box and x0 (the
    // samplings of the pair below)
    b200mppi_planner* p = t.b->pl[i];
    const int n = ran[i];
    p->prepared = false;
    p->pushed_direct = false;
    if (n == 0) continue;
    if (i >= K1) {
      const int* rec = hrec + 5 * (i - K1);
      p->reach_slot ^= (n * num_opt) & 1;
      p->reach_valid = true;
      for (int c = 0; c < 5; ++c) p->last_box[c] = rec[c];
    } else if (!t.barebone) {
      last_box_whole_map(p);
    }
    for (int c = 0; c < 3; ++c) p->prm.x0[c] = x0[3 * i + c];
  }
  // each TDM group's pair as after the samplings of its longest-running member (a group samples at every solve while any
  // member runs), a stochastic pair's last kind from the group's record (a group of one: its planner's)
  for (int k = 0; k < 2; ++k) {
    TrialPart& q = t.P[k];
    for (int g = 0; g < q.G; ++g) {
      int n = 0;
      for (int j = q.gr.first[g]; j < q.gr.first[g + 1]; ++j) n = std::max(n, ran[q.lo + q.gr.members[j]]);
      if (n == 0) continue;
      if (k == 1) {
        const int* rec = q.grouped ? reinterpret_cast<const int*>(h + L.grec) + 5 * g : hrec + 5 * q.gr.lead(g);
        q.plans[g].boxed[0] = q.plans[g].boxed[1] = rec[0] != 0;
      }
      for (int s = 0; s < n; ++s) { plan_commit(q.plans[g], 0); plan_commit(q.plans[g], 1); }
    }
  }
}

// Reads back the states and histories, and leaves the caller's outputs, every planner and every TDM group's pair as
// after the host loop
static int trial_call_commit(TrialCall& t) {
  b200mppi_batch* b = t.b;
  const TrialLayout& L = t.L;
  const unsigned char* d = t.d;
  unsigned char* h = t.h;
  cudaStream_t st = b->stream;
  const int K = t.K, S = t.S, R = t.R;
  const size_t per = t.per;
  const std::vector<int>& first = t.first;
  b200mppi_trial_result* results = t.results;
  // the box records (stochastic) through the results (sequences), then the histories
  CU(cudaMemcpyAsync(h + L.rec, d + L.rec, L.res_end - L.rec, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(h + L.head, d + L.xh, L.total - L.xh, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const TrialState* hst = reinterpret_cast<const TrialState*>(h + L.state);
  const TrialState* hres = reinterpret_cast<const TrialState*>(h + L.res);
  const int* hcon = reinterpret_cast<const int*>(h + L.con);
  const double* hx = reinterpret_cast<const double*>(h + L.head);
  const float* hu = reinterpret_cast<const float*>(h + L.head + (L.uh - L.xh));
  const double dnan = std::nan("");
  const float fnan = std::nanf("");
  std::vector<int> ran(K, 0);                          // steps each planner ran, over all its episodes
  std::vector<float> x0(3 * (size_t)K);                // the x0 of each planner's last solve
  for (int i = 0; i < K; ++i) {
    int last = first[i];                               // the planner's last slot that ran
    for (int j = first[i]; j < first[i + 1]; ++j) {
      const TrialState& r = t.seq ? hres[j] : hst[i];
      const int n = r.steps;                           // 0: an episode of a sequence that never ran
      double* xo = t.xhist + (size_t)j * (S + 1) * 3;
      float* uo = t.uhist + (size_t)j * S * 2;
      if (n > 0) {
        for (int c = 0; c < 3; ++c) xo[c] = t.trials[j].x0[c];
        last = j;
      }
      std::memcpy(xo + 3, hx + ((size_t)j * (S + 1) + 1) * 3, (size_t)n * 3 * sizeof(double));
      for (size_t q = (size_t)(n > 0 ? n + 1 : 0) * 3; q < (size_t)(S + 1) * 3; ++q) xo[q] = dnan;
      std::memcpy(uo, hu + (size_t)j * S * 2, (size_t)n * 2 * sizeof(float));
      for (size_t q = (size_t)n * 2; q < (size_t)S * 2; ++q) uo[q] = fnan;
      results[j] = b200mppi_trial_result{r.cum_obj, r.cum_dist, r.dist, n, r.status};
      ran[i] += n;
      if (t.barebone) t.contact_steps[j] = hcon[j];
    }
    // the last solve planned from the pose before the last step -- or, when a later episode of a sequence without
    // reset_x0 took one step, from the previous episode's final pose
    const double* xl = t.xhist + ((size_t)last * (S + 1) + results[last].steps - 1) * 3;
    if (results[last].steps == 1 && last > first[i] && !t.reset_x0)
      xl = t.xhist + ((size_t)(last - 1) * (S + 1) + results[last - 1].steps) * 3;
    for (int c = 0; c < 3; ++c) x0[3 * i + c] = (float)xl[c];
  }
  trial_commit_planners(t, ran, x0);
  if (!t.record) return B200MPPI_OK;
  // record r of a slot belongs to step r * record_every of its episode; slot first[i] + e goes to the caller's slab
  // (i, e).  Only the written ones are copied (records past an episode's last step are never written, and an early
  // stop leaves most of them so): the rest is NaN, as are the slabs of episodes a planner does not have.  The last one
  // of a planner's last run episode is what its state_rollout buffer holds after the host loop's last
  // get_state_rollout.
  const float* drec = reinterpret_cast<const float*>(d + L.vrec);
  for (int i = 0; i < K; ++i) {
    int last = first[i], last_done = 0;
    float* planner_out = t.rollouts + (size_t)i * t.max_episodes * R * per;
    std::fill(planner_out + (size_t)(first[i + 1] - first[i]) * R * per,
              planner_out + (size_t)t.max_episodes * R * per, fnan);
    for (int j = first[i]; j < first[i + 1]; ++j) {
      const int done = (results[j].steps + t.record_every - 1) / t.record_every;
      float* slab = planner_out + (size_t)(j - first[i]) * R * per;
      CU(cudaMemcpyAsync(slab, drec + (size_t)j * R * per, (size_t)done * per * sizeof(float), cudaMemcpyDeviceToHost,
                         st));
      std::fill(slab + (size_t)done * per, slab + (size_t)R * per, fnan);
      if (done > 0) { last = j; last_done = done; }
    }
    CU(cudaMemcpyAsync(b->pl[i]->state_rollout, drec + ((size_t)last * R + last_done - 1) * per, per * sizeof(float),
                       cudaMemcpyDeviceToDevice, st));
  }
  CU(cudaStreamSynchronize(st));
  return B200MPPI_OK;
}

// The closed-loop trials of every kind of batch.  Stochastic trials also move each planner's reach box with the robot;
// with box_mode 2 and num_opt 1 it depends on the controls drawn, so the batched boxed sampler decides it on the device
// (reach_box_decide, the function sample_finish calls) and a step needs no host round trip (trial_call_step lists a
// step's launches).  The plant step also moves stochastic planners' rollout windows and counts barebone contacts.
// record_every = n > 0 records the visualisation rollouts of every step s with s % n == 0, after the step's last update
// and before the plant step (which shifts u_cur and overwrites x0); stochastic planners first complete maps [0, V) of
// every pair whose step sampled a box (the maps the rollouts read).
// Trial sequences (episodes non-null, b200mppi_batch_run_trial_sequences): planner i runs episodes[i] episodes back to
// back, descriptors, histories and results per slot (planner-major: planner i's are slots first[i] .. first[i + 1]),
// through the same step loop for up to max_i episodes[i] * max_steps steps; the plant step (plant_step_seq_kernel)
// moves a planner to its next episode without a launch, and the commit follows each planner's total steps.
// A recording sequence records at each episode's own steps t with t % record_every == 0: the plant step sets each
// planner's record flag and record pointer for the next step (SeqArgs).
static int batch_run_trials(b200mppi_batch* b, TrialKind kind, const b200mppi_trial_desc* trials, int32_t max_steps,
                            double* xhist, float* uhist, b200mppi_trial_result* results, int32_t* contact_steps,
                            int32_t record_every, float* rollouts, size_t rollout_bytes, int32_t* steps_issued,
                            const int32_t* episodes, int32_t reset_x0) {
  if (!b) return fail(B200MPPI_EINVAL, "null batch");
  if (b->loop) return loop_busy("run_trials");
  TrialCall t{b, kind, trials, max_steps, xhist, uhist, results, contact_steps, record_every, rollouts, rollout_bytes,
              episodes, reset_x0 != 0};
  int rc;
  if ((rc = trial_call_validate(t)) || (rc = trial_call_plan(t))) return rc;
  t.L = trial_layout(t);
  struct Buffers {                                     // freed on every return
    unsigned char* d = nullptr;
    unsigned char* h = nullptr;
    cudaEvent_t ev[TRIAL_POLL] = {};
    ~Buffers() {
      cudaFree(d);
      if (h) cudaFreeHost(h);
      for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    }
  } buf;
  if (cudaMalloc(&buf.d, t.L.total) != cudaSuccess) {
    buf.d = nullptr;
    cudaGetLastError();                                // not sticky: later calls start clean
    return fail(B200MPPI_ECUDA, t.fn + ": cudaMalloc of " + std::to_string(t.L.total) + " bytes");
  }
  if (cudaMallocHost(&buf.h, t.L.head + (t.L.total - t.L.xh)) != cudaSuccess) {
    buf.h = nullptr;
    return fail(B200MPPI_ECUDA, t.fn + ": cudaMallocHost");
  }
  t.d = buf.d;
  t.h = buf.h;
  if ((rc = trial_call_stage(t))) return rc;
  int* hcount = reinterpret_cast<int*>(t.h);           // the polled counts, in the no longer needed head of the staging
  for (cudaEvent_t& e : buf.ev) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  int issued = 0;
  for (int s = 0; s < t.S * t.max_episodes; ++s) {
    if (s >= TRIAL_POLL) {                            // the count after step s - POLL
      CU(cudaEventSynchronize(buf.ev[s % TRIAL_POLL]));
      if (hcount[s % TRIAL_POLL] == 0) break;
    }
    if ((rc = trial_call_step(t, s)) || (rc = trial_call_plant(t, s))) return rc;
    ++issued;
    CU(cudaMemcpyAsync(hcount + s % TRIAL_POLL, t.pa.active_count, sizeof(int), cudaMemcpyDeviceToHost, b->stream));
    CU(cudaEventRecord(buf.ev[s % TRIAL_POLL], b->stream));
  }
  if ((rc = trial_call_commit(t))) return rc;
  if (steps_issued) *steps_issued = issued;
  return B200MPPI_OK;
}

extern "C" int b200mppi_batch_run_trials(b200mppi_batch* b, const b200mppi_trial_desc* trials, int32_t max_steps,
                                         double* xhist, float* uhist, b200mppi_trial_result* results,
                                         int32_t* steps_issued) {
  return batch_run_trials(b, TrialKind::onemap, trials, max_steps, xhist, uhist, results, nullptr, 0, nullptr, 0,
                          steps_issued, nullptr, 0);
}

extern "C" int b200mppi_batch_run_stochastic_trials(b200mppi_batch* b, const b200mppi_trial_desc* trials,
                                                    int32_t max_steps, double* xhist, float* uhist,
                                                    b200mppi_trial_result* results, int32_t* steps_issued) {
  return batch_run_trials(b, TrialKind::stochastic, trials, max_steps, xhist, uhist, results, nullptr, 0, nullptr, 0,
                          steps_issued, nullptr, 0);
}

extern "C" int b200mppi_batch_run_mixed_trials(b200mppi_batch* b, const b200mppi_trial_desc* trials, int32_t max_steps,
                                               double* xhist, float* uhist, b200mppi_trial_result* results,
                                               int32_t* steps_issued) {
  return batch_run_trials(b, TrialKind::mixed, trials, max_steps, xhist, uhist, results, nullptr, 0, nullptr, 0,
                          steps_issued, nullptr, 0);
}

// the trial kind of B200MPPI_TRIALS_* `kind`
static TrialKind trial_kind(int32_t kind) {
  return kind == B200MPPI_TRIALS_STOCHASTIC ? TrialKind::stochastic : kind == B200MPPI_TRIALS_BAREBONE ?
         TrialKind::barebone : kind == B200MPPI_TRIALS_MIXED ? TrialKind::mixed : TrialKind::onemap;
}

extern "C" int b200mppi_batch_run_barebone_trials(b200mppi_batch* b, const b200mppi_trial_desc* trials,
                                                  int32_t max_steps, double* xhist, float* uhist,
                                                  b200mppi_trial_result* results, int32_t* contact_steps,
                                                  int32_t* steps_issued) {
  return batch_run_trials(b, TrialKind::barebone, trials, max_steps, xhist, uhist, results, contact_steps, 0, nullptr,
                          0, steps_issued, nullptr, 0);
}

extern "C" int b200mppi_batch_run_trials_recorded(b200mppi_batch* b, int32_t kind, const b200mppi_trial_desc* trials,
                                                  int32_t max_steps, double* xhist, float* uhist,
                                                  b200mppi_trial_result* results, int32_t* contact_steps,
                                                  int32_t record_every, float* rollouts, size_t rollout_bytes,
                                                  int32_t* steps_issued) {
  if (!b) return fail(B200MPPI_EINVAL, "null batch");
  if (kind != B200MPPI_TRIALS_MAP && kind != B200MPPI_TRIALS_STOCHASTIC && kind != B200MPPI_TRIALS_BAREBONE &&
      kind != B200MPPI_TRIALS_MIXED)
    return fail(B200MPPI_EINVAL, "run_trials_recorded: unknown trial kind " + std::to_string(kind));
  if (record_every < 1)
    return fail(B200MPPI_EINVAL, "run_trials_recorded: record_every " + std::to_string(record_every) + " < 1");
  return batch_run_trials(b, trial_kind(kind), trials, max_steps, xhist, uhist, results, contact_steps, record_every, rollouts,
                          rollout_bytes, steps_issued, nullptr, 0);
}

extern "C" int b200mppi_batch_run_trial_sequences(b200mppi_batch* b, int32_t kind, const b200mppi_trial_desc* trials,
                                                  const int32_t* episodes, int32_t max_steps, int32_t reset_x0,
                                                  double* xhist, float* uhist, b200mppi_trial_result* results,
                                                  int32_t* steps_issued) {
  if (!b) return fail(B200MPPI_EINVAL, "null batch");
  if (kind != B200MPPI_TRIALS_MAP && kind != B200MPPI_TRIALS_STOCHASTIC && kind != B200MPPI_TRIALS_MIXED)
    return fail(B200MPPI_EINVAL, "run_trial_sequences: trial kind " + std::to_string(kind) + " (sequences run "
                                 "B200MPPI_TRIALS_MAP, B200MPPI_TRIALS_STOCHASTIC or B200MPPI_TRIALS_MIXED batches)");
  if (!episodes) return fail(B200MPPI_EINVAL, "run_trial_sequences: null episode counts");
  return batch_run_trials(b, trial_kind(kind), trials,
                          max_steps, xhist, uhist, results, nullptr, 0, nullptr, 0, steps_issued, episodes, reset_x0);
}

extern "C" int b200mppi_batch_run_trial_sequences_ex(b200mppi_batch* b, int32_t kind, const b200mppi_trial_desc* trials,
                                                     const int32_t* episodes, int32_t max_steps, int32_t reset_x0,
                                                     double* xhist, float* uhist, b200mppi_trial_result* results,
                                                     int32_t* contact_steps, int32_t record_every, float* rollouts,
                                                     size_t rollout_bytes, int32_t* steps_issued) {
  if (!b) return fail(B200MPPI_EINVAL, "null batch");
  if (kind != B200MPPI_TRIALS_MAP && kind != B200MPPI_TRIALS_STOCHASTIC && kind != B200MPPI_TRIALS_BAREBONE &&
      kind != B200MPPI_TRIALS_MIXED)
    return fail(B200MPPI_EINVAL, "run_trial_sequences_ex: unknown trial kind " + std::to_string(kind));
  if (!episodes) return fail(B200MPPI_EINVAL, "run_trial_sequences_ex: null episode counts");
  if (record_every < 0)
    return fail(B200MPPI_EINVAL, "run_trial_sequences_ex: record_every " + std::to_string(record_every) + " < 0");
  if (kind != B200MPPI_TRIALS_BAREBONE && contact_steps)
    return fail(B200MPPI_EINVAL, "run_trial_sequences_ex: contact_steps given for a trial kind other than "
                                 "B200MPPI_TRIALS_BAREBONE");
  return batch_run_trials(b, trial_kind(kind), trials, max_steps, xhist, uhist, results, contact_steps, record_every,
                          rollouts, rollout_bytes, steps_issued, episodes, reset_x0);
}

// --------------------------------------------------------------------------------------------- device loops
// A trial call without its plant step, driven one call at a time: the phases of batch_run_trials (validation, plans,
// layout, staging, step and the planner and TDM commit) over one device buffer that lives while the loop is open.  The
// caller's plant runs between the calls on the batch's stream; the loop kernels (reduce.cu) take its poses and stops.
// The loop's solve clock lives on the device (LoopClock) and no call passes anything that changes from one call
// to the next, so the calls may be captured into a CUDA graph and replayed, mixed freely with eager calls.  Every call
// a loop call makes while the batch's stream captures is legal under cudaStreamCaptureModeGlobal; close refuses.
struct b200mppi_loop {
  TrialCall t{};
  LoopArgs la{};
  LoopClock lc{};
  LoopTaskArgs ta{};
  cudaEvent_t ev = nullptr;            // orders the batch's stream after work on the stream of a caller's array
  ~b200mppi_loop() {
    cudaFree(t.d);
    if (t.h) cudaFreeHost(t.h);
    if (ev) cudaEventDestroy(ev);
  }
};

// a caller's array at p must lie in device memory of the batch's device
static int loop_device_ptr(const b200mppi_loop* lp, const void* p, const char* fn, const char* what) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    return fail(B200MPPI_EINVAL, std::string(fn) + ": " + what + " is not a CUDA pointer");
  }
  if ((at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) || at.device != lp->t.b->device)
    return fail(B200MPPI_EINVAL, std::string(fn) + ": " + what + " is not in memory of device " +
                                 std::to_string(lp->t.b->device));
  return B200MPPI_OK;
}

constexpr int LOOP_MAX_OBSTACLES = 1 << 24;

extern "C" int b200mppi_batch_loop_open_ex(b200mppi_batch* b, int32_t kind, const double* padded_limits,
                                           const int32_t* rows, int32_t max_obstacles, b200mppi_loop** out) {
  if (!b || !out) return fail(B200MPPI_EINVAL, "loop_open: null argument");
  if (b->loop) return loop_busy("loop_open");
  if (kind != B200MPPI_TRIALS_MAP && kind != B200MPPI_TRIALS_STOCHASTIC && kind != B200MPPI_TRIALS_BAREBONE &&
      kind != B200MPPI_TRIALS_MIXED)
    return fail(B200MPPI_EINVAL, "loop_open: unknown trial kind " + std::to_string(kind));
  if (max_obstacles < 0 || max_obstacles > LOOP_MAX_OBSTACLES)
    return fail(B200MPPI_EINVAL, "loop_open: max_obstacles " + std::to_string(max_obstacles) + " outside [0, 2^24]");
  if (max_obstacles > 0 && kind != B200MPPI_TRIALS_BAREBONE)
    return fail(B200MPPI_EINVAL, "loop_open: max_obstacles " + std::to_string(max_obstacles) + " for a loop that is not "
                                 "barebone (only barebone planners take obstacles)");
  std::unique_ptr<b200mppi_loop> lp(new b200mppi_loop());
  TrialCall& t = lp->t;
  t.b = b; t.kind = trial_kind(kind); t.S = 0;
  t.loop = true; t.limits = padded_limits; t.rows = rows;
  int rc;
  if ((rc = trial_call_validate(t)) || (rc = trial_call_plan(t))) return rc;
  // the capacity: a barebone loop can always set again as many obstacles as any of its planners has now
  t.O = max_obstacles;
  for (int i = 0; i < t.K && t.barebone; ++i) t.O = std::max(t.O, b->pl[i]->num_obstacles);
  t.L = trial_layout(t);
  if (cudaMalloc(&t.d, t.L.total) != cudaSuccess) {
    t.d = nullptr;
    cudaGetLastError();
    return fail(B200MPPI_ECUDA, "loop_open: cudaMalloc of " + std::to_string(t.L.total) + " bytes");
  }
  if (cudaMallocHost(&t.h, t.L.head) != cudaSuccess) {
    t.h = nullptr;
    return fail(B200MPPI_ECUDA, "loop_open: cudaMallocHost");
  }
  if ((rc = trial_call_stage(t))) return rc;
  CU(cudaEventCreateWithFlags(&lp->ev, cudaEventDisableTiming));
  lp->la = LoopArgs{reinterpret_cast<const TrialDev*>(t.d + t.L.tr), reinterpret_cast<LoopState*>(t.d + t.L.loop),
                    t.pa.active, t.pa.active_count, t.K, b->T};
  LoopClock& lc = lp->lc;
  lc.clock = reinterpret_cast<int*>(t.d + t.L.clock);
  for (int k = 0; k < 2; ++k) {
    lc.set_cur[k] = reinterpret_cast<SampleGridsV2Args*>(t.d + t.L.part[k].cur);
    lc.set_par[k][0] = t.P[k].set_d[0];
    lc.set_par[k][1] = t.P[k].set_d[1];
    lc.G[k] = t.P[k].G;
  }
  lc.nprep = reinterpret_cast<NoisePrepDesc*>(t.d + b->off_nprep);
  lc.box = reinterpret_cast<SampleBoxDesc*>(t.d + t.L.box);
  lc.slot0 = reinterpret_cast<const int*>(t.d + t.L.slot0);
  lc.K2 = t.K2;
  lc.num_opt = b->pl[0]->prm.num_opt;
  lp->ta = LoopTaskArgs{reinterpret_cast<LoopTask*>(t.d + t.L.task), reinterpret_cast<float*>(t.d + t.L.obs),
                        reinterpret_cast<double*>(t.d + t.L.obs64), t.O};
  b->loop = lp.get();
  for (b200mppi_planner* p : b->pl) p->loop = lp.get();
  *out = lp.release();
  return B200MPPI_OK;
}

extern "C" int b200mppi_batch_loop_open(b200mppi_batch* b, int32_t kind, const double* padded_limits,
                                        const int32_t* rows, b200mppi_loop** out) {
  return b200mppi_batch_loop_open_ex(b, kind, padded_limits, rows, 0, out);
}

extern "C" int b200mppi_loop_obstacle_capacity(b200mppi_loop* lp, int32_t* capacity) {
  if (!lp || !capacity) return fail(B200MPPI_EINVAL, "loop_obstacle_capacity: null argument");
  *capacity = lp->t.O;
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_controls(b200mppi_loop* lp, float** u_dev, void** stream) {
  if (!lp || !u_dev || !stream) return fail(B200MPPI_EINVAL, "loop_controls: null argument");
  *u_dev = reinterpret_cast<float*>(lp->t.d + lp->t.L.lu);
  *stream = lp->t.b->stream;
  return B200MPPI_OK;
}

// The capture sequence id of stream s (0: s is not capturing)
static int capture_id(cudaStream_t s, unsigned long long* id) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  *id = 0;
  CU(cudaStreamGetCaptureInfo(s, &cs, id));
  if (cs != cudaStreamCaptureStatusActive) *id = 0;
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_wait_stream(b200mppi_loop* lp, void* stream) {
  if (!lp) return fail(B200MPPI_EINVAL, "loop_wait_stream: null loop");
  cudaStream_t s = (cudaStream_t)stream, st = lp->t.b->stream;
  if (s == st) return B200MPPI_OK;
  CU(cudaSetDevice(lp->t.b->device));
  // while the batch's stream captures, an event recorded on a stream outside that capture would invalidate it (the
  // legacy default stream is never part of one, and is not even queried then)
  unsigned long long id_st = 0, id_s = 0;
  int rc;
  if ((rc = capture_id(st, &id_st))) return rc;
  if (id_st && s != nullptr && s != cudaStreamLegacy && (rc = capture_id(s, &id_s))) return rc;
  if (id_st && id_s != id_st)
    return fail(B200MPPI_EINVAL, "loop_wait_stream: the batch's stream is capturing a CUDA graph and the stream is not "
                                 "part of that capture");
  CU(cudaEventRecord(lp->ev, s));
  CU(cudaStreamWaitEvent(st, lp->ev, 0));
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_solve(b200mppi_loop* lp, float* u_dev) {
  if (!lp || !u_dev) return fail(B200MPPI_EINVAL, "loop_solve: null argument");
  int rc;
  if ((rc = loop_device_ptr(lp, u_dev, "loop_solve", "u_dev"))) return rc;
  b200mppi_batch* b = lp->t.b;
  CU(cudaSetDevice(b->device));
  if ((rc = trial_call_step(lp->t, 0))) return rc;   // s unused: the loop's solves read what its clock prepared
  launch_loop_export(lp->la, lp->lc, u_dev, b->stream);
  b->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_shift_and_update(b200mppi_loop* lp, const void* x_dev, int32_t dtype,
                                              int64_t row_stride_bytes) {
  if (!lp || !x_dev) return fail(B200MPPI_EINVAL, "loop_shift_and_update: null argument");
  if (dtype != B200MPPI_POSE_F64 && dtype != B200MPPI_POSE_F32)
    return fail(B200MPPI_EINVAL, "loop_shift_and_update: unknown pose dtype " + std::to_string(dtype));
  const int64_t e = dtype == B200MPPI_POSE_F64 ? 8 : 4;
  if (row_stride_bytes < 3 * e || row_stride_bytes % e != 0 || reinterpret_cast<uintptr_t>(x_dev) % e != 0)
    return fail(B200MPPI_EINVAL, "loop_shift_and_update: row stride of " + std::to_string(row_stride_bytes) +
                                 " bytes or a pointer not aligned to the element (rows of 3 contiguous elements)");
  int rc;
  if ((rc = loop_device_ptr(lp, x_dev, "loop_shift_and_update", "x_dev"))) return rc;
  b200mppi_batch* b = lp->t.b;
  CU(cudaSetDevice(b->device));
  launch_loop_ingest(lp->la, x_dev, dtype, row_stride_bytes, b->stream);
  b->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_stop(b200mppi_loop* lp, const void* mask_dev, int32_t elem_bytes) {
  if (!lp || !mask_dev) return fail(B200MPPI_EINVAL, "loop_stop: null argument");
  if (elem_bytes != 1 && elem_bytes != 4)
    return fail(B200MPPI_EINVAL, "loop_stop: mask elements of " + std::to_string(elem_bytes) + " bytes (1 or 4)");
  if (reinterpret_cast<uintptr_t>(mask_dev) % elem_bytes != 0)
    return fail(B200MPPI_EINVAL, "loop_stop: mask not aligned to its elements");
  int rc;
  if ((rc = loop_device_ptr(lp, mask_dev, "loop_stop", "mask_dev"))) return rc;
  b200mppi_batch* b = lp->t.b;
  CU(cudaSetDevice(b->device));
  launch_loop_stop(lp->la, mask_dev, elem_bytes, b->stream);
  b->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

// A caller's (count, n) array of dtype B200MPPI_POSE_F64 / _F32, rows row_stride_bytes apart: the stride holds a row
// and is a whole number of elements, and the pointer is aligned to the element
static int loop_rows_ok(const void* p, int32_t dtype, int64_t n, int64_t row_stride_bytes, const char* fn,
                        const char* what) {
  if (dtype != B200MPPI_POSE_F64 && dtype != B200MPPI_POSE_F32)
    return fail(B200MPPI_EINVAL, std::string(fn) + ": unknown " + what + " dtype " + std::to_string(dtype));
  const int64_t e = dtype == B200MPPI_POSE_F64 ? 8 : 4;
  if (row_stride_bytes < n * e || row_stride_bytes % e != 0 || reinterpret_cast<uintptr_t>(p) % e != 0)
    return fail(B200MPPI_EINVAL, std::string(fn) + ": row stride of " + std::to_string(row_stride_bytes) + " bytes or a " +
                                 "pointer not aligned to the element (rows of " + std::to_string(n) +
                                 " contiguous elements)");
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_set_goals(b200mppi_loop* lp, const void* g_dev, int32_t dtype, int64_t row_stride_bytes) {
  if (!lp || !g_dev) return fail(B200MPPI_EINVAL, "loop_set_goals: null argument");
  int rc;
  if ((rc = loop_rows_ok(g_dev, dtype, 2, row_stride_bytes, "loop_set_goals", "goal"))) return rc;
  if ((rc = loop_device_ptr(lp, g_dev, "loop_set_goals", "g_dev"))) return rc;
  b200mppi_batch* b = lp->t.b;
  CU(cudaSetDevice(b->device));
  launch_loop_goal(lp->la, lp->ta, g_dev, dtype, row_stride_bytes, b->stream);
  b->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_set_obstacles(b200mppi_loop* lp, const void* obs_dev, int32_t dtype, int32_t count,
                                           int64_t row_stride_bytes, const int32_t* counts_dev) {
  if (!lp || (!obs_dev && count > 0)) return fail(B200MPPI_EINVAL, "loop_set_obstacles: null argument");
  if (!lp->t.barebone)
    return fail(B200MPPI_EINVAL, "loop_set_obstacles: the loop is not barebone (only barebone planners take obstacles)");
  if (count < 0 || count > lp->t.O)
    return fail(B200MPPI_EINVAL, "loop_set_obstacles: " + std::to_string(count) + " obstacles per planner, the loop's "
                                 "capacity is " + std::to_string(lp->t.O) + " (b200mppi_batch_loop_open_ex's "
                                 "max_obstacles)");
  int rc;
  if ((rc = loop_rows_ok(obs_dev, dtype, 3 * (int64_t)count, row_stride_bytes, "loop_set_obstacles", "obstacle")))
    return rc;
  if (count > 0 && (rc = loop_device_ptr(lp, obs_dev, "loop_set_obstacles", "obs_dev"))) return rc;
  if (counts_dev) {
    if (reinterpret_cast<uintptr_t>(counts_dev) % 4 != 0)
      return fail(B200MPPI_EINVAL, "loop_set_obstacles: counts not aligned to its int32 elements");
    if ((rc = loop_device_ptr(lp, counts_dev, "loop_set_obstacles", "counts_dev"))) return rc;
  }
  b200mppi_batch* b = lp->t.b;
  CU(cudaSetDevice(b->device));
  launch_loop_obstacles(lp->la, lp->ta, obs_dev, dtype, count, row_stride_bytes, counts_dev, b->stream);
  b->launches++;
  CHECK_LAUNCH();
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_active(b200mppi_loop* lp, const int32_t** dev) {
  if (!lp || !dev) return fail(B200MPPI_EINVAL, "loop_active: null argument");
  *dev = lp->t.pa.active;
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_close_ex(b200mppi_loop* lp, b200mppi_loop_summary* per_planner,
                                      b200mppi_loop_task* tasks, double* obstacles) {
  if (!lp) return fail(B200MPPI_EINVAL, "loop_close: null loop");
  TrialCall& t = lp->t;
  b200mppi_batch* b = t.b;
  // close waits for the stream, which a capture forbids: refused with the loop left open and usable
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(b->stream, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone)
    return fail(B200MPPI_EINVAL, "loop_close: the batch's stream is capturing a CUDA graph (close the loop after the "
                                 "capture ends)");
  std::unique_ptr<b200mppi_loop> own(lp);
  b->loop = nullptr;                                   // closed whatever follows: the batch and planners are free again
  for (b200mppi_planner* p : b->pl) p->loop = nullptr;
  CU(cudaSetDevice(b->device));
  // the box records through the loop's counters, poses, solve clock and task updates, in one copy
  CU(cudaMemcpyAsync(t.h + t.L.rec, t.d + t.L.rec, t.L.res_end - t.L.rec, cudaMemcpyDeviceToHost, b->stream));
  CU(cudaStreamSynchronize(b->stream));
  if (reinterpret_cast<const int*>(t.h + t.L.clock)[1]) {
    for (b200mppi_planner* p : b->pl) { p->prepared = false; p->pushed_direct = false; }
    return fail(B200MPPI_ESTATE, "loop_close: more than 2^31 - 1 solves issued; the planners' counts are not committed");
  }
  const LoopState* ls = reinterpret_cast<const LoopState*>(t.h + t.L.loop);
  std::vector<int> ran(t.K);
  std::vector<float> x0(3 * (size_t)t.K);
  for (int i = 0; i < t.K; ++i) {
    ran[i] = ls[i].solves;
    for (int c = 0; c < 3; ++c) x0[3 * i + c] = ls[i].x0[c];
    if (per_planner) {
      b200mppi_loop_summary& s = per_planner[i];
      s.solves = ls[i].solves; s.shifts = ls[i].shifts; s.status = ls[i].status;
      for (int c = 0; c < 3; ++c) s.x[c] = ls[i].x[c];
    }
  }
  trial_commit_planners(t, ran, x0);
  // the C-side params and obstacles as set_params and set_obstacles of the last goal and obstacle set would leave them
  const LoopTask* lt = reinterpret_cast<const LoopTask*>(t.h + t.L.task);
  const double* o64 = reinterpret_cast<const double*>(t.h + t.L.obs64);
  bool copied = false;
  for (int i = 0; i < t.K; ++i) {
    b200mppi_planner* p = b->pl[i];
    if (tasks) {
      tasks[i] = b200mppi_loop_task{lt[i].took_goal, lt[i].took_obstacles, lt[i].num_obstacles, 0,
                                    {lt[i].goal[0], lt[i].goal[1]}};
    }
    if (lt[i].took_goal)
      for (int c = 0; c < 2; ++c) p->prm.xgoal[c] = (float)lt[i].goal[c];
    if (!lt[i].took_obstacles) continue;
    const int n = lt[i].num_obstacles;
    if (n > p->obstacles_cap) {
      cudaFree(p->obstacles); p->obstacles = nullptr; p->obstacles_cap = 0; p->num_obstacles = 0;
      CU(cudaMalloc(&p->obstacles, (size_t)n * 3 * sizeof(float)));
      p->obstacles_cap = n;
    }
    if (n > 0) {
      CU(cudaMemcpyAsync(p->obstacles, loop_obstacles(t, i), (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToDevice,
                         b->stream));
      copied = true;
    }
    p->num_obstacles = n;
  }
  if (obstacles) std::memcpy(obstacles, o64, (size_t)t.K * t.O * 3 * sizeof(double));
  if (copied) CU(cudaStreamSynchronize(b->stream));   // before the loop's buffer is freed
  return B200MPPI_OK;
}

extern "C" int b200mppi_loop_close(b200mppi_loop* lp, b200mppi_loop_summary* per_planner) {
  return b200mppi_loop_close_ex(lp, per_planner, nullptr, nullptr);
}
