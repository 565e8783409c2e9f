"""Host emulation of the generic rollout kernels and the visualisation kernel (TEST INFRASTRUCTURE; tests/emu_core.py).
The kernels' text (csrc/rollout.cu between the ``[emu:... rollout]`` / ``[emu:... vis]`` markers, cell_index* and the
parameter structs from csrc/common.cuh / kernels.h) is compiled with g++.  The arithmetic helpers of common.cuh have
their IEEE meaning and the MUFU approximations and approximate divisions are libm's correctly rounded ones
(tests/emu_cuda.h) -- which is what the oracle and the reference's simulator goldens use, so the comparison tolerance
is a few ulp, tighter than on the GPU."""
from tests.emu_core import build as _build
from tests.emu_core import cell_index_rzi, extern_shared, region

HARNESS = r'''
using namespace b200;
// as launch_rollout (csrc/rollout.cu): mode 0 / 1 / 2 generic kernels, mode 3 the barebone kernel
extern "C" void emu_rollout(int mode, const float* f, const int* g, const double* ratios, const int8_t* lin,
                            const int8_t* ang, const int8_t* obs, const int8_t* unk, const int8_t* risk,
                            const float* noise, const float* u_cur, float* costs_nm, float* costs,
                            const float* obstacles, int num_obstacles) {
  RolloutArgs a{};
  emu::params(a.p, f, g, ratios, g[8]);
  a.mode = mode; a.lin_grid = lin; a.ang_grid = ang; a.obstacle = obs; a.unknown = unk; a.risk = risk;
  a.noise = noise; a.u_cur = u_cur; a.costs = costs; a.obstacles = obstacles;
  a.num_obstacles = num_obstacles;
  std::vector<float> mn((size_t)std::max(a.p.M, 1) * std::max(a.p.N, 1), 0.0f);      // map-major device layout (kernels.h, CostDst)
  a.dst.base[0] = mn.data(); a.dst.n_per = std::max(a.p.N, 1); a.dst.ld = a.p.N; a.dst.row0 = 0;
  const int threads = 128;
  const unsigned gx = (unsigned)((a.p.N + threads - 1) / threads);
  if (mode == 3) emu::launch({gx, 1, 1}, threads, [&] { rollout_barebone_kernel(a); });
  else if (mode == 0) emu::launch({gx, (unsigned)a.p.M, 1}, threads, [&] { rollout_kernel<0>(a); });
  else if (mode == 1) emu::launch({gx, 1, 1}, threads, [&] { rollout_kernel<1>(a); });
  else emu::launch({gx, 1, 1}, threads, [&] { rollout_kernel<2>(a); });
  if (mode == 0 && costs_nm)                                      // hand back the logical (N, M) array
    for (int n = 0; n < a.p.N; ++n)
      for (int m = 0; m < a.p.M; ++m) costs_nm[(size_t)n * a.p.M + m] = mn[(size_t)m * a.p.N + n];
}

extern "C" void emu_state_rollout(int mode, int V, const float* f, const int* g, const double* ratios, const int8_t* lin,
                                  const int8_t* ang, const float* noise, const float* u_cur, const float* u_prev,
                                  float* out) {
  VisArgs a{};
  emu::params(a.p, f, g, ratios, g[8]);
  a.mode = mode; a.V = V; a.lin_grid = lin; a.ang_grid = ang; a.noise = noise; a.u_cur = u_cur; a.u_prev = u_prev;
  a.out = out;
  emu::launch({(unsigned)((V + 31) / 32), 1, 1}, 32, [&] { state_rollout_kernel(a); });
}
'''


def build(out_dir, extra=""):
    parts = [region("common.cuh", "params"), cell_index_rzi(region("common.cuh", "cell_index")),
             region("kernels.h", "cost_dst"), region("kernels.h", "rollout_args"), region("kernels.h", "vis_args"),
             extern_shared(region("rollout.cu", "rollout"), 2), region("rollout.cu", "vis")]
    return _build(out_dir, "rollout_emu", parts, HARNESS + extra)
