"""Host emulation of the closed-loop plant-step kernel (TEST INFRASTRUCTURE; tests/emu_core.py): the kernel text of
csrc/reduce.cu between the ``[emu:... trial]`` markers and its argument structs from kernels.h, compiled with g++ with
the CUDA rounding intrinsics replaced by the IEEE operations they name and one thread per lane of each planner's warp
(``__syncwarp`` = a barrier of the 32 threads)."""
from tests.emu_core import build as _build
from tests.emu_core import region

HARNESS = r'''
using namespace b200;
// planner i: grids lin[i] / ang[i] (H[i], W[i]) float64, g[11 i ..] = xlo, ylo, res, dt, xgoal[2], tol, pxlim[2],
// pylim[2]; u_cur[i] (T, 2) shifted in place, x0_out[i] (3 floats); state: K TrialStates of 7 doubles: x[3], cum_obj,
// cum_dist, dist, then steps and status as two int32
extern "C" void emu_plant(int K, int T, int max_steps, int step, const double** lin, const double** ang, const int* H,
                          const int* W, const double* g, float** u_cur, float** x0_out, void* state, int* active,
                          int* count, double* xhist, float* uhist) {
  std::vector<TrialDev> d(K);
  for (int i = 0; i < K; ++i) {
    const double* q = g + 11 * i;
    d[i] = TrialDev{lin[i], ang[i], H[i], W[i], q[0], q[1], q[2], q[3], {q[4], q[5]}, q[6], {q[7], q[8]}, {q[9], q[10]},
                    u_cur[i], x0_out[i]};
  }
  PlantArgs a{d.data(), reinterpret_cast<TrialState*>(state), active, count, xhist, uhist, K, T, max_steps, step};
  emu::launch({(unsigned)K, 1, 1}, 32, [&] { plant_step_body(a, (int)blockIdx.x, (int)threadIdx.x); });
}
extern "C" int emu_state_bytes() { return (int)sizeof(b200::TrialState); }
'''


def kernels():
    """plant_step_body with its argument structs."""
    return [region("kernels.h", "trial_args"), region("reduce.cu", "trial")]


def build(out_dir, extra=""):
    return _build(out_dir, "trial_emu", kernels(), HARNESS + extra)
