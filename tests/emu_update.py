"""Host emulation of the control-update kernels (TEST INFRASTRUCTURE; technique of tests/emu_sampler.py): the text of
update_partial_kernel / merge_partials / update_rank_kernel / update_apply_kernel (csrc/reduce.cu between the
``[emu:... update]`` markers) compiled with g++, one std::thread per CUDA thread.  Float arithmetic follows the
kernel's own order; ``exp`` is libm's instead of CUDA's (both within an ulp), so results are compared within the
bounds of tests/reduce_bounds.py."""
import ctypes as C
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mppi_numba_b200", "csrc")

PRELUDE = r'''
#include <algorithm>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>
struct EmuDim3 { unsigned x, y, z; };
static thread_local EmuDim3 threadIdx, blockIdx, blockDim, gridDim;
static std::barrier<>* g_bar = nullptr;
struct EmuWarp { std::barrier<> bar{32}; float fbuf[32]; };
static thread_local EmuWarp* g_warp = nullptr;
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__
static inline void __syncthreads() { g_bar->arrive_and_wait(); }
static inline float __shfl_xor_sync(unsigned, float v, int o) {
  const int lane = threadIdx.x & 31;
  g_warp->fbuf[lane] = v;
  g_warp->bar.arrive_and_wait();
  const float r = g_warp->fbuf[lane ^ o];
  g_warp->bar.arrive_and_wait();
  return r;
}
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void __threadfence_system() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void st_flag_sys(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
struct FlagWait { const uint32_t* flags; int ws; uint32_t epoch; unsigned long long timeout_ns; int* status; };
static inline void flag_wait(const FlagWait&) {}          // blocks run one after the other: nothing to wait for
static inline float __double2float_rn(double d) { return (float)d; }
struct float2 { float x, y; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
using std::min;
using std::max;
namespace b200 {
static inline float fsub(float a, float b) { return a - b; }      // common.cuh: sub.rn.ftz.f32
'''

HARNESS = r'''
template <class K>
static void run(K kernel, int threads, unsigned blocks) {
  for (unsigned bx = 0; bx < blocks; ++bx) {
    std::barrier<> bar(threads);
    g_bar = &bar;
    std::vector<std::unique_ptr<EmuWarp>> warps;
    for (int w = 0; w < threads / 32; ++w) warps.emplace_back(new EmuWarp());
    std::vector<std::thread> th;
    for (int t = 0; t < threads; ++t)
      th.emplace_back([&, t] {
        threadIdx = {(unsigned)t, 0, 0}; blockIdx = {bx, 0, 0}; blockDim = {(unsigned)threads, 1, 1}; gridDim = {blocks, 1, 1};
        g_warp = warps[t / 32].get();
        kernel();
      });
    for (auto& x : th) x.join();
  }
}
static UpdateArgs make(const float* costs, const float* noise, float* w_raw, float* cta_partials, float* rank_partial,
                       float* u_cur, float* weights, int N, int T, float lambda, const float* vr, const float* wr) {
  UpdateArgs a{};
  a.costs = costs; a.noise = noise; a.w_raw = w_raw; a.cta_partials = cta_partials; a.rank_partial = rank_partial;
  a.u_cur = u_cur; a.weights = weights; a.N = N; a.T = T; a.lambda = lambda;
  a.vrange[0] = vr[0]; a.vrange[1] = vr[1]; a.wrange[0] = wr[0]; a.wrange[1] = wr[1];
  int ctas = (N + 31) / 32;                       // update_num_ctas + the planner's rows_per_cta rule (api.cu)
  if (ctas > 296) ctas = 296;
  if (ctas < 1) ctas = 1;
  a.rows_per_cta = (N + ctas - 1) / ctas;
  a.num_ctas = (N + a.rows_per_cta - 1) / a.rows_per_cta;
  return a;
}
}  // namespace b200

extern "C" int emu_update_num_ctas(int N) {
  float z[2] = {0, 0};
  return b200::make(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, N, 1, 1.0f, z, z).num_ctas;
}

// launch_update_partial with UPD_TAIL_RANK: CTA partials + (last CTA) this rank's partial (2T+2 floats)
extern "C" void emu_update_partial(const float* costs, const float* noise, float* w_raw, float* cta_partials,
                                   float* rank_partial, int N, int T, float lambda) {
  using namespace b200;
  float z[2] = {0, 0};
  const UpdateArgs a = make(costs, noise, w_raw, cta_partials, rank_partial, nullptr, nullptr, N, T, lambda, z, z);
  unsigned counter = 0;
  UpdateTail tl{};
  tl.counter = &counter; tl.mode = UPD_TAIL_RANK;
  run([&] { update_partial_kernel(a, tl); }, UPD_THREADS, (unsigned)a.num_ctas);
}

// UPD_TAIL_APPLY: the whole one-rank update in ONE launch (partials, merge and apply by the last CTA)
extern "C" int emu_update_one_rank(const float* costs, const float* noise, float* w_raw, float* cta_partials,
                                   float* rank_partial, float* u_cur, float* weights, int N, int T, float lambda,
                                   const float* vr, const float* wr) {
  using namespace b200;
  const UpdateArgs a = make(costs, noise, w_raw, cta_partials, rank_partial, u_cur, weights, N, T, lambda, vr, wr);
  unsigned counter = 0;
  UpdateTail tl{};
  tl.counter = &counter; tl.mode = UPD_TAIL_APPLY;
  run([&] { update_partial_kernel(a, tl); }, UPD_THREADS, (unsigned)a.num_ctas);
  return counter == 0 ? 0 : 1;                    // the ticket counter is left at zero for the next launch
}

// UPD_TAIL_BCAST: the rank partial goes into slot `rank` of every peer's gather buffer (ws, 2T+2), flags raised
extern "C" int emu_update_bcast(const float* costs, const float* noise, float* w_raw, float* cta_partials,
                                float* rank_partial, int N, int T, float lambda, int ws, int rank, float* gather_all,
                                uint32_t* flags_all, uint32_t epoch) {
  using namespace b200;
  float z[2] = {0, 0};
  const UpdateArgs a = make(costs, noise, w_raw, cta_partials, rank_partial, nullptr, nullptr, N, T, lambda, z, z);
  unsigned counter = 0;
  UpdateTail tl{};
  tl.counter = &counter; tl.mode = UPD_TAIL_BCAST; tl.ws = ws; tl.rank = rank; tl.epoch = epoch;
  for (int q = 0; q < ws; ++q) {
    tl.peer_gather[q] = gather_all + (size_t)q * ws * (2 * T + 2);
    tl.peer_flags[q] = flags_all + (size_t)q * ws;
  }
  run([&] { update_partial_kernel(a, tl); }, UPD_THREADS, (unsigned)a.num_ctas);
  return counter == 0 ? 0 : 1;
}

// launch_update_finish: combine `count` gathered rank partials into u_cur and this rank's normalised weights
extern "C" void emu_update_finish(const float* gathered, int count, const float* w_raw, const float* cta_partials,
                                  float* u_cur, float* weights, int N, int T, float lambda, const float* vr,
                                  const float* wr) {
  using namespace b200;
  const UpdateArgs a = make(nullptr, nullptr, const_cast<float*>(w_raw), const_cast<float*>(cta_partials), nullptr, u_cur,
                            weights, N, T, lambda, vr, wr);
  int ctas = a.num_ctas < 32 ? a.num_ctas : 32;
  if (ctas < 1) ctas = 1;
  run([&] { update_apply_kernel(a, gathered, count, FlagWait{}); }, UPD_THREADS, (unsigned)ctas);
}
'''


def _region(path, name):
    text = open(path).read()
    m = re.search(r"// \[emu:begin %s\][^\n]*\n(.*?)// \[emu:end %s\]" % (name, name), text, re.S)
    assert m, "marker %s not found in %s" % (name, path)
    return m.group(1)


def build(out_dir):
    kernels = _region(os.path.join(CSRC, "reduce.cu"), "update")
    kernels = re.sub(r"(?m)^(\s*)__shared__ ", r"\1static ", kernels)      # block-shared arrays: one instance
    kernels = kernels.replace("int update_num_ctas(int N) {", "static int update_num_ctas_unused(int N) {")
    src = (PRELUDE + "constexpr int P2P_MAX_PEERS = 16;\n" + _region(os.path.join(CSRC, "kernels.h"), "update_args") +
           _region(os.path.join(CSRC, "kernels.h"), "update_tail") +
           _region(os.path.join(CSRC, "common.cuh"), "warp_min") + _region(os.path.join(CSRC, "common.cuh"), "warp_sum") +
           kernels + HARNESS)
    cpp = os.path.join(out_dir, "update_emu.cpp")
    so = os.path.join(out_dir, "libupdate_emu.so")
    open(cpp, "w").write(src)
    r = subprocess.run(["g++", "-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-Wno-unknown-pragmas",
                        "-ffp-contract=off", cpp, "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    lib = C.CDLL(so)
    P, I, F = C.c_void_p, C.c_int, C.c_float
    lib.emu_update_num_ctas.restype = I
    lib.emu_update_num_ctas.argtypes = [I]
    lib.emu_update_partial.restype = None
    lib.emu_update_partial.argtypes = [P, P, P, P, P, I, I, F]
    lib.emu_update_one_rank.restype = I
    lib.emu_update_one_rank.argtypes = [P, P, P, P, P, P, P, I, I, F, P, P]
    lib.emu_update_bcast.restype = I
    lib.emu_update_bcast.argtypes = [P, P, P, P, P, I, I, F, I, I, P, P, C.c_uint32]
    lib.emu_update_finish.restype = None
    lib.emu_update_finish.argtypes = [P, I, P, P, P, P, I, I, F, P, P]
    return lib
