"""Host emulation of the closed-loop plant-step kernel (TEST INFRASTRUCTURE; technique of tests/emu_batch.py): the
kernel text of csrc/reduce.cu between the ``[emu:... trial]`` markers and its argument structs from kernels.h, compiled
with g++ (-ffp-contract=off) with the CUDA rounding intrinsics replaced by the IEEE operations they name and one thread
per lane of each planner's warp (``__syncwarp`` = a barrier of the 32 threads)."""
import ctypes as C
import os

from tests.emu_batch import _compile, _src

PRELUDE = r'''
#include <barrier>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <thread>
#include <vector>
struct EmuDim3 { unsigned x, y, z; };
static thread_local EmuDim3 threadIdx, blockIdx, blockDim;
static std::barrier<>* g_bar = nullptr;
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __restrict__
static inline void __syncwarp() { g_bar->arrive_and_wait(); }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __dsqrt_rn(double a) { return std::sqrt(a); }
static inline float __double2float_rn(double a) { return (float)a; }
static inline int atomicSub(int* p, int v) { int o = *p; *p = o - v; return o; }
using std::cos; using std::sin; using std::fmod; using std::floor; using std::copysign;
namespace b200 {
'''

HARNESS = r'''
}  // namespace b200
// planner i: grids lin[i] / ang[i] (H[i], W[i]) float64, g[11 i ..] = xlo, ylo, res, dt, xgoal[2], tol, pxlim[2],
// pylim[2]; u_cur[i] (T, 2) shifted in place, x0_out[i] (3 floats); state: K TrialStates of 7 doubles: x[3], cum_obj,
// cum_dist, dist, then steps and status as two int32
extern "C" void emu_plant(int K, int T, int max_steps, int step, const double** lin, const double** ang, const int* H,
                          const int* W, const double* g, float** u_cur, float** x0_out, void* state, int* active,
                          int* count, double* xhist, float* uhist) {
  using namespace b200;
  std::vector<TrialDev> d(K);
  for (int i = 0; i < K; ++i) {
    const double* q = g + 11 * i;
    d[i] = TrialDev{lin[i], ang[i], H[i], W[i], q[0], q[1], q[2], q[3], {q[4], q[5]}, q[6], {q[7], q[8]}, {q[9], q[10]},
                    u_cur[i], x0_out[i]};
  }
  PlantArgs a{d.data(), reinterpret_cast<TrialState*>(state), active, count, xhist, uhist, K, T, max_steps, step};
  for (int k = 0; k < K; ++k) {
    std::barrier<> bar(32);
    g_bar = &bar;
    std::vector<std::thread> th;
    for (int lane = 0; lane < 32; ++lane) th.emplace_back([&, lane] { plant_step_body(a, k, lane); });
    for (auto& t : th) t.join();
  }
}
extern "C" int emu_state_bytes() { return (int)sizeof(b200::TrialState); }
'''


def build(out_dir):
    src = PRELUDE + _src("kernels.h", "trial_args") + _src("reduce.cu", "trial") + HARNESS
    lib = _compile(out_dir, "trial_emu", src)
    P, I = C.c_void_p, C.c_int
    lib.emu_plant.restype = None
    lib.emu_plant.argtypes = [I, I, I, I] + [P] * 12
    lib.emu_state_bytes.restype = I
    return lib
