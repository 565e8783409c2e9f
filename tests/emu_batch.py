"""Host emulation of the batched one-map kernels (TEST INFRASTRUCTURE; tests/emu_core.py).  The kernel text of the
noise, rollout, update and sampler regions of csrc/*.cu -- the single-planner kernels AND their batched wrappers
(``[emu:... *_batch]``) -- is compiled with g++ with a launch over blockIdx.y / blockIdx.z.  Each library runs either K
single launches or ONE batched launch of the same emulated code, so the CPU suite checks the descriptor plumbing and
the grid-coordinate indexing of the batched kernels bit for bit."""
from tests import emu_sampler, emu_update
from tests.emu_core import build as _build
from tests.emu_core import cell_index_rzi, extern_shared, region

# ----------------------------------------------------------------------------- noise
NOISE_HARNESS = r'''
using namespace b200;
// K planners: batched != 0 -> ONE launch over blockIdx.y, else K single launches of sample_noise_kernel
extern "C" void emu_noise(int K, int batched, uint64_t** states, float** noise, const float* std, long long count) {
  std::vector<NoiseDesc> d(K);
  for (int i = 0; i < K; ++i) d[i] = NoiseDesc{states[i], noise[i], std[2 * i], std[2 * i + 1]};
  const unsigned blocks = (unsigned)((count + 255) / 256);
  if (batched) {
    emu::launch_serial({blocks, (unsigned)K, 1}, 256, [&] { sample_noise_batch_kernel(d.data(), count); });
    return;
  }
  for (int i = 0; i < K; ++i)
    emu::launch_serial({blocks, 1, 1}, 256, [&] {
      sample_noise_kernel(states[i], reinterpret_cast<float2*>(noise[i]), count, std[2 * i], std[2 * i + 1], nullptr);
    });
}
'''


def noise_kernels():
    """sample_noise_kernel and sample_noise_batch_kernel with the generator and its descriptor."""
    return [region("common.cuh", "xoro"), region("common.cuh", "normal"), region("reduce.cu", "noise"),
            region("kernels.h", "noise_desc"), region("reduce.cu", "noise_batch")]


def build_noise(out_dir, extra=""):
    return _build(out_dir, "noise_batch_emu", noise_kernels(), NOISE_HARNESS + extra)


# ----------------------------------------------------------------------------- rollout (modes 1, 2, 3)
ROLLOUT_HARNESS = r'''
using namespace b200;
// planner i: f[23 i ..], g[9 i ..] as tests/emu_rollout.py (one map: M = 1), ratios[2 i ..]; per-planner buffers as
// pointer arrays
extern "C" void emu_rollout(int K, int batched, int mode, const float* f, const int* g, const double* ratios,
                            const int8_t** lin, const int8_t** ang, const int8_t** obs, const int8_t** unk,
                            const int8_t** risk, const float** noise, const float** u_cur, float** costs,
                            const float** obstacles, const int* num_obstacles) {
  std::vector<RolloutArgs> d(K);
  for (int i = 0; i < K; ++i) {
    RolloutArgs a{};
    emu::params(a.p, f + 23 * i, g + 9 * i, ratios + 2 * i, 1);
    a.mode = mode; a.lin_grid = lin[i]; a.ang_grid = ang[i]; a.obstacle = obs[i]; a.unknown = unk[i]; a.risk = risk[i];
    a.noise = noise[i]; a.u_cur = u_cur[i]; a.costs = costs[i]; a.obstacles = obstacles[i];
    a.num_obstacles = num_obstacles[i];
    d[i] = a;
  }
  const int threads = 128;
  const unsigned gx = (unsigned)((d[0].p.N + threads - 1) / threads);
  if (batched) {
    const EmuDim3 grid{gx, (unsigned)K, 1};
    if (mode == 1) emu::launch(grid, threads, [&] { rollout_batch_kernel<1>(d.data()); });
    else if (mode == 2) emu::launch(grid, threads, [&] { rollout_batch_kernel<2>(d.data()); });
    else emu::launch(grid, threads, [&] { rollout_batch_kernel<3>(d.data()); });
    return;
  }
  for (int i = 0; i < K; ++i) {
    const RolloutArgs a = d[i];
    if (mode == 1) emu::launch({gx, 1, 1}, threads, [&] { rollout_kernel<1>(a); });
    else if (mode == 2) emu::launch({gx, 1, 1}, threads, [&] { rollout_kernel<2>(a); });
    else emu::launch({gx, 1, 1}, threads, [&] { rollout_barebone_kernel(a); });
  }
}
'''


def build_rollout(out_dir, extra=""):
    parts = [region("common.cuh", "params"), cell_index_rzi(region("common.cuh", "cell_index")),
             region("kernels.h", "cost_dst"), region("kernels.h", "rollout_args"),
             extern_shared(region("rollout.cu", "rollout") + region("rollout.cu", "rollout_batch"), 2)]
    return _build(out_dir, "rollout_batch_emu", parts, ROLLOUT_HARNESS + extra)


# ----------------------------------------------------------------------------- update (UPD_TAIL_APPLY)
UPDATE_HARNESS = r'''
using namespace b200;
// planner i: costs / noise / w_raw / cta_partials / rank_partial / u_cur / weights / u_prev / u_out buffers, lambda[i],
// ranges vr[2 i], wr[2 i]; batched: ONE launch over blockIdx.y, else K single launches (u_prev / u_out unset: the
// single-planner path's tail, whose u_prev the caller then copies as after_u_update does).  Returns the sum of the
// ticket counters left behind (0: every planner's counter is reset for the next launch).
extern "C" int emu_update(int K, int batched, const float** costs, const float** noise, float** w_raw, float** parts,
                          float** rank_partial, float** u_cur, float** weights, float** u_prev, float** u_out, int N,
                          int T, const float* lambda, const float* vr, const float* wr) {
  std::vector<UpdateBatchDesc> d(K);
  std::vector<unsigned> counters(K, 0);
  int ctas, rows_per_cta;
  emu::update_geometry(N, ctas, rows_per_cta);
  for (int i = 0; i < K; ++i) {
    UpdateArgs a{};
    a.costs = costs[i]; a.noise = noise[i]; a.w_raw = w_raw[i]; a.cta_partials = parts[i]; a.rank_partial = rank_partial[i];
    a.u_cur = u_cur[i]; a.weights = weights[i]; a.N = N; a.T = T; a.num_ctas = ctas; a.rows_per_cta = rows_per_cta;
    a.lambda = lambda[i]; a.vrange[0] = vr[2 * i]; a.vrange[1] = vr[2 * i + 1]; a.wrange[0] = wr[2 * i]; a.wrange[1] = wr[2 * i + 1];
    UpdateTail tl{};
    tl.counter = &counters[i]; tl.mode = UPD_TAIL_APPLY;
    if (batched) { tl.u_prev = u_prev[i]; tl.u_out = u_out[i]; }
    d[i] = UpdateBatchDesc{a, tl};
  }
  if (batched) {
    emu::launch({(unsigned)ctas, (unsigned)K, 1}, UPD_THREADS, [&] { update_partial_batch_kernel(d.data()); });
  } else {
    for (int i = 0; i < K; ++i) {
      const UpdateArgs a = d[i].a;
      const UpdateTail tl = d[i].tl;
      emu::launch({(unsigned)ctas, 1, 1}, UPD_THREADS, [&] { update_partial_kernel(a, tl); });
    }
  }
  int left = 0;
  for (unsigned c : counters) left += (int)c;
  return left;
}
'''


def build_update(out_dir, extra=""):
    return _build(out_dir, "update_batch_emu", emu_update.kernels("update_batch"), UPDATE_HARNESS + extra)


# ----------------------------------------------------------------------------- sampler (fused lin + ang, whole maps)
SAMPLER_HARNESS = r'''
using namespace b200;
// pair i: grids g0[i] / g1[i] (grid_rows, pitch), cumulative tables c0[i] / c1[i], ONE set of generator states st[i]
// (fused: both TDMs hold the same states) -> so0[i] / so1[i], value tables q0[i] / q1[i]; one geometry for all pairs
extern "C" int emu_sampler(int K, int batched, int8_t** g0, int8_t** g1, const int8_t** c0, const int8_t** c1,
                           const uint64_t** st, uint64_t** so0, uint64_t** so1, const int8_t** q0, const int8_t** q1,
                           int bpad, int rows, int cols, int grid_rows, int pitch, int tx, int ty, int segs, double alpha,
                           int q_cap) {
  std::vector<uint64_t> T(SAMPLE_TABLE_WORDS);
  if (!build_sample_thresholds(alpha, q_cap, T.data())) return 1;
  const int nrow = (rows + tx - 1) / tx;
  int seg_rows;
  std::vector<uint64_t> J;
  emu::segment_jumps(rows, cols, tx, ty, segs, seg_rows, J);
  std::vector<SampleGridsV2Args> d(K);
  for (int i = 0; i < K; ++i) {
    SampleGridsV2Args a{};
    a.t[0] = SampleTdm{g0[i], c0[i], st[i], so0[i], q0[i], bpad};
    a.t[1] = SampleTdm{g1[i], c1[i], st[i], so1[i], q1[i], bpad};
    a.thresholds = T.data(); a.jump = J.empty() ? nullptr : J.data();
    a.rows = rows; a.cols = cols; a.grid_rows = grid_rows; a.pitch = pitch; a.tx = tx; a.ty = ty; a.num_maps = 1;
    a.segs = segs; a.seg_rows = seg_rows;
    sample_box_full(a);
    if (a.ty * a.gm > 256) a.gm = 256 / a.ty;
    d[i] = a;
  }
  const int threads = ((d[0].nact * d[0].gm + 31) / 32) * 32;
  if (threads > 256 || d[0].gm < 1) return 3;
  const int tix_hi = std::min(tx - 1, (rows - 1) / nrow);               // launch_v2_nt (sample.cu)
  const unsigned gx = (unsigned)((tix_hi + 1) * segs), gy = (unsigned)((1 + d[0].gm - 1) / d[0].gm);
  emu::sampler_nw(bpad, [&](auto NW) {
    if (batched) {
      emu::launch({gx, gy, (unsigned)K}, threads, [&] { sample_grids_v2_batch_kernel<2, decltype(NW)::value>(d.data()); });
      return;
    }
    for (int i = 0; i < K; ++i) {
      const SampleGridsV2Args a = d[i];
      emu::launch({gx, gy, 1}, threads, [&] { sample_grids_v2_kernel<2, decltype(NW)::value>(a); });
    }
  });
  return 0;
}
'''


def build_sampler(out_dir, extra=""):
    return _build(out_dir, "sampler_batch_emu", emu_sampler.kernels(None, "sampler_batch"), SAMPLER_HARNESS + extra,
                  link_engine=True)
