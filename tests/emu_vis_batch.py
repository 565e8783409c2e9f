"""Host emulation of the batched visualisation rollouts and of the map completion of recording stochastic trials (TEST
INFRASTRUCTURE; tests/emu_core.py).

``build``: state_rollout_batch_kernel (csrc/rollout.cu, ``[emu:... vis_batch]``) next to the single-planner
state_rollout_kernel it wraps, with its descriptor (csrc/kernels.h, ``vis_args``): K single launches or ONE batched
launch of the same emulated code, with the trials' ``active`` gate and record offset.

``build_complete``: sample_grids_v2_complete_batch_kernel (csrc/sample.cu, ``[emu:... sampler_box_batch]``) launched as
run_stochastic_trials launches it, next to tests/emu_sampler.py's single-planner sampler as the whole-map reference."""
from tests import emu_sampler
from tests.emu_core import build as _build
from tests.emu_core import cell_index_rzi, extern_shared, region

HARNESS = r'''
using namespace b200;
// planner i: mode modes[i], f[23 i ..], g[9 i ..] (g[9 i + 8] = its M), ratios[2 i ..] as tests/emu_rollout.py, its own
// grids / noise / u_cur / u_prev.  batched: ONE launch over blockIdx.y into out[i] + out_off (active may be null), else
// K single launches into out[i].
extern "C" void emu_vis(int K, int batched, const int* modes, int V, const float* f, const int* g, const double* ratios,
                        const int8_t** lin, const int8_t** ang, const float** noise, const float** u_cur,
                        const float** u_prev, float** out, const int* active, size_t out_off) {
  std::vector<VisArgs> a(K);
  std::vector<RolloutParams> ps(K);
  std::vector<VisBatchDesc> d(K);
  for (int i = 0; i < K; ++i) {
    a[i] = VisArgs{};
    emu::params(a[i].p, f + 23 * i, g + 9 * i, ratios + 2 * i, g[9 * i + 8]);
    a[i].mode = modes[i]; a[i].V = V; a[i].lin_grid = lin[i]; a[i].ang_grid = ang[i];
    a[i].noise = noise[i]; a[i].u_cur = u_cur[i]; a[i].u_prev = u_prev[i]; a[i].out = out[i];
    ps[i] = a[i].p;
    d[i] = VisBatchDesc{&ps[i], modes[i], V, lin[i], ang[i], noise[i], u_cur[i], u_prev[i], out[i]};
  }
  const unsigned gx = (unsigned)((V + 31) / 32);
  if (batched) {
    emu::launch_serial({gx, (unsigned)K, 1}, 32, [&] { state_rollout_batch_kernel(d.data(), active, out_off); });
    return;
  }
  for (int i = 0; i < K; ++i) {
    const VisArgs ai = a[i];
    emu::launch_serial({gx, 1, 1}, 32, [&] { state_rollout_kernel(ai); });
  }
}
'''

COMPLETE_HARNESS = r'''
// K fused pairs of one geometry (shared cum / qvals / thresholds; own maps and pre-call states): ONE completion launch
// over maps [0, V) as run_stochastic_trials issues it after a step's boxed sampling, with the box launch's geometry
// (mrows tile rows x segs, ncact tile columns, gm maps per CTA).  rec[k]: the pair's box record (rec[k][0] = how).
// grid0 / grid1: K x (M, grid_rows, pitch); states: K x (ngen, 2), read; out0 / out1: K x (ngen, 2), the other buffers.
extern "C" int emu_complete(int K, int8_t* grid0, int8_t* grid1, const int8_t* cum0, const int8_t* cum1,
                            const uint64_t* states, uint64_t* out0, uint64_t* out1, const int8_t* qv0, const int8_t* qv1,
                            int bpad, int rows, int cols, int grid_rows, int pitch, int tx, int ty, int M, int segs,
                            double alpha, int q_cap, int* rec, const int* active, int V, int mrows, int ncact, int gm) {
  std::vector<uint64_t> T(SAMPLE_TABLE_WORDS);
  if (!build_sample_thresholds(alpha, q_cap, T.data())) return 1;
  int seg_rows;
  std::vector<uint64_t> J;
  emu::segment_jumps(rows, cols, tx, ty, segs, seg_rows, J);
  const size_t ngen = (size_t)tx * ty * M, gsz = (size_t)M * grid_rows * pitch;
  std::vector<SampleGridsV2Args> d(K);
  std::vector<SampleBoxDesc> bx(K);
  for (int k = 0; k < K; ++k) {
    SampleGridsV2Args& a = d[k];
    a = SampleGridsV2Args{};
    a.t[0] = SampleTdm{grid0 + k * gsz, cum0, states + k * ngen * 2, out0 + k * ngen * 2, qv0, bpad};
    a.t[1] = SampleTdm{grid1 + k * gsz, cum1, states + k * ngen * 2, out1 + k * ngen * 2, qv1, bpad};
    a.thresholds = T.data(); a.jump = J.empty() ? nullptr : J.data();
    a.rows = rows; a.cols = cols; a.grid_rows = grid_rows; a.pitch = pitch; a.tx = tx; a.ty = ty; a.num_maps = M;
    a.segs = segs; a.seg_rows = seg_rows;
    sample_box_full(a);
    a.gm = gm; a.write_states = 0;
    bx[k] = SampleBoxDesc{};
    bx[k].record = rec + 5 * k;
  }
  const int threads = ((ncact * gm + 31) / 32) * 32;
  emu::sampler_nw(bpad, [&](auto NW) {
    emu::launch({(unsigned)(mrows * segs), (unsigned)((V + gm - 1) / gm), (unsigned)K}, threads, [&] {
      sample_grids_v2_complete_batch_kernel<decltype(NW)::value>(d.data(), bx.data(), active, V, mrows, ncact);
    });
  });
  return 0;
}
'''


def build(out_dir, extra=""):
    parts = [region("common.cuh", "params"), cell_index_rzi(region("common.cuh", "cell_index")),
             region("kernels.h", "cost_dst"), region("kernels.h", "rollout_args"), region("kernels.h", "vis_args"),
             extern_shared(region("rollout.cu", "rollout"), 2), region("rollout.cu", "vis"),
             region("rollout.cu", "vis_batch")]
    return _build(out_dir, "vis_batch_emu", parts, HARNESS + extra)


def build_complete(out_dir, extra=""):
    """The completion launch and, compiled into the same library, emu_sample_v2 (tests/emu_sampler.py)."""
    return _build(out_dir, "complete_batch_emu", emu_sampler.kernels(None, "sampler_box_batch"),
                  emu_sampler.HARNESS + COMPLETE_HARNESS + extra, link_engine=True)
