"""Host emulation of the sampler kernel (TEST INFRASTRUCTURE).

The text of sample_grids_v2_kernel and the device helpers it uses is lifted verbatim from the CUDA sources (the
regions between ``[emu:begin ...]`` / ``[emu:end ...]`` markers in csrc/sample.cu, csrc/common.cuh and
csrc/kernels.h) and compiled with g++ against a few shims: the thread / block indices are thread-local variables,
``__syncthreads()`` is a std::barrier over the block's threads (one std::thread per CUDA thread, blocks run one
after the other), ``__shared__`` memory is one static buffer, ``__popc`` / ``__byte_perm`` / ``__ldg`` are
functions.  The host-side table builders (threshold buckets, GF(2) jump matrices) are the library's own, linked
from libb200mppi.so.  This lets the CPU test-suite run the REAL kernel source on small maps and compare it bit
for bit with the oracle -- no GPU needed."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mppi_numba_b200", "csrc")

PRELUDE = r'''
#include <algorithm>
#include <barrier>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>
#include <cmath>
struct EmuDim3 { unsigned x, y, z; };
static thread_local EmuDim3 threadIdx, blockIdx, blockDim, gridDim;
static std::barrier<>* g_bar = nullptr;
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __align__(n)
#define __shared__
static inline void __syncthreads() { g_bar->arrive_and_wait(); }
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned s) {        // default mode, no msb replication
  const unsigned long long src = ((unsigned long long)b << 32) | a;
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) r |= (unsigned)((src >> (8 * ((s >> (4 * i)) & 7))) & 0xffu) << (8 * i);
  return r;
}
struct ulonglong2 { unsigned long long x, y; };
static inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { return ulonglong2{x, y}; }
struct uint4 { unsigned x, y, z, w; };
using std::min;
using std::max;
namespace b200 {
alignas(16) unsigned char smem[1 << 20];
'''

HARNESS = r'''
bool build_sample_thresholds(double alpha, int q_cap, uint64_t* table);

template <int NT, int NW>
static void run(const SampleGridsV2Args& a, int threads, unsigned gx, unsigned gy) {
  for (unsigned by = 0; by < gy; ++by)
    for (unsigned bx = 0; bx < gx; ++bx) {
      std::barrier<> bar(threads);
      g_bar = &bar;
      std::vector<std::thread> th;
      for (int t = 0; t < threads; ++t)
        th.emplace_back([&, t] {
          threadIdx = {(unsigned)t, 0, 0}; blockIdx = {bx, by, 0}; blockDim = {(unsigned)threads, 1, 1}; gridDim = {gx, gy, 1};
          sample_grids_v2_kernel<NT, NW>(a);
        });
      for (auto& x : th) x.join();
    }
}
}  // namespace b200

// nt TDMs (1 or 2) sampled from the generator states `states` (numba layout, gen = tix*(ty*M)+m*ty+tiy).
// cum: (nt)(rows, cols, bpad) int8 running sums; grids: (nt)(M, grid_rows, pitch); qvals: (nt)(128).
// disc = {cx, cy, r} (cells) or null: the reach disc inside the box (per-CTA narrowing of the tile columns).
// box = {row_lo, row_hi, col_lo, col_hi} (cells) or null: with a box the launch is restricted as apply_box (api.cu)
// does it and the states come from advance_states_kernel -- what plan_launch does for a boxed solve.
extern "C" int emu_sample_v2(int nt, int8_t* grid0, int8_t* grid1, const int8_t* cum0, const int8_t* cum1,
                             const uint64_t* states, uint64_t* states_out, const int8_t* qv0, const int8_t* qv1, int bpad,
                             int rows, int cols, int grid_rows, int pitch, int tx, int ty, int num_maps, int segs,
                             double alpha, int q_cap, const int* box, const float* disc) {
  using namespace b200;
  SampleGridsV2Args a{};
  std::vector<uint64_t> out2(states_out ? 0 : 1);
  a.t[0] = SampleTdm{grid0, cum0, states, states_out, qv0, bpad};
  std::vector<uint64_t> alt;
  if (nt == 2) {                       // the second TDM holds identical states (that is the fusion condition)
    alt.resize((size_t)tx * ty * num_maps * 2);
    a.t[1] = SampleTdm{grid1, cum1, states, alt.data(), qv1, bpad};
  }
  std::vector<uint64_t> T(SAMPLE_TABLE_WORDS);
  if (!build_sample_thresholds(alpha, q_cap, T.data())) return 1;
  a.thresholds = T.data();
  const int nrow = (rows + tx - 1) / tx, ncol = (cols + ty - 1) / ty;
  if (segs > nrow) segs = nrow;
  if (segs < 1) segs = 1;
  const int seg_rows = (nrow + segs - 1) / segs;
  std::vector<uint64_t> J;
  if (segs > 1) {                      // as tdm_prepare_jump (api.cu)
    int last_w = cols - (ty - 1) * ncol;
    for (int iy = ty - 1; iy >= 0 && last_w <= 0; --iy) last_w = cols - iy * ncol;
    if (last_w > ncol) last_w = ncol;
    if (last_w < 0) last_w = 0;
    std::vector<int64_t> ks;
    for (int s = 1; s < segs; ++s) { ks.push_back((int64_t)s * seg_rows * ncol); ks.push_back((int64_t)s * seg_rows * last_w); }
    J.resize(ks.size() * 256);
    build_jump_matrices(ks.data(), (int)ks.size(), J.data());
    a.jump = J.data();
  }
  a.rows = rows; a.cols = cols; a.grid_rows = grid_rows; a.pitch = pitch; a.tx = tx; a.ty = ty; a.num_maps = num_maps;
  a.segs = segs; a.seg_rows = seg_rows;
  sample_box_full(a);
  if (a.ty * a.gm > 256) a.gm = 256 / a.ty;
  int tix_hi = tx - 1;
  if (box) {                           // apply_box (api.cu)
    a.row_lo = box[0]; a.row_hi = box[1];
    a.tix_lo = box[0] / nrow;
    a.tiy_lo = box[2] / ncol;
    a.nact = (box[3] - 1) / ncol - a.tiy_lo + 1;
    int gm = 128 / a.nact;
    if (gm > SG_GM_MAX) gm = SG_GM_MAX;
    if (gm > num_maps) gm = num_maps;
    if (gm < 1) gm = 1;
    a.gm = gm;
    a.write_states = 0;
    if (disc) { a.disc_cx = disc[0]; a.disc_cy = disc[1]; a.disc_r = disc[2]; }
    tix_hi = std::min(tx - 1, (std::max(a.row_hi, a.row_lo + 1) - 1) / nrow);       // launch_v2_nt (sample.cu)
  }
  const int threads = ((a.nact * a.gm + 31) / 32) * 32;
  if (threads > 256 || a.gm < 1) return 3;
  const unsigned gx = (unsigned)((tix_hi - a.tix_lo + 1) * segs), gy = (unsigned)((num_maps + a.gm - 1) / a.gm);
  const int nw = bpad / 4;
  if (nt == 1) {
    if (nw == 3) run<1, 3>(a, threads, gx, gy); else if (nw == 8) run<1, 8>(a, threads, gx, gy);
    else if (nw == 1) run<1, 1>(a, threads, gx, gy); else run<1, 0>(a, threads, gx, gy);
  } else {
    if (nw == 3) run<2, 3>(a, threads, gx, gy); else if (nw == 8) run<2, 8>(a, threads, gx, gy);
    else if (nw == 1) run<2, 1>(a, threads, gx, gy); else run<2, 0>(a, threads, gx, gy);
  }
  if (box) {                           // launch_advance_states (sample.cu), one thread at a time
    int64_t ks[4];
    const int nr = (rows + tx - 1) / tx, nc = (cols + ty - 1) / ty;           // sample_tile_draws
    const int last_h = rows % nr ? rows % nr : nr, last_w = cols % nc ? cols % nc : nc;
    ks[0] = (int64_t)nr * nc; ks[1] = (int64_t)nr * last_w; ks[2] = (int64_t)last_h * nc; ks[3] = (int64_t)last_h * last_w;
    std::vector<uint64_t> mats(4 * 256);
    build_jump_matrices(ks, 4, mats.data());
    const int64_t total = (int64_t)tx * ty * num_maps;
    const unsigned nblk = (unsigned)((total + 127) / 128);
    for (unsigned bx = 0; bx < nblk; ++bx) {                   // 128 host threads per block (the kernel stages in shared memory)
      std::barrier<> bar(128);
      g_bar = &bar;
      std::vector<std::thread> th;
      for (int t = 0; t < 128; ++t)
        th.emplace_back([&, t] {
          threadIdx = {(unsigned)t, 0, 0}; blockIdx = {bx, 0, 0}; blockDim = {128, 1, 1}; gridDim = {nblk, 1, 1};
          advance_states_kernel(reinterpret_cast<const ulonglong2*>(states), reinterpret_cast<ulonglong2*>(states_out),
                                nt == 2 ? reinterpret_cast<ulonglong2*>(alt.data()) : nullptr,
                                reinterpret_cast<const ulonglong2*>(mats.data()), rows, cols, tx, ty, num_maps);
        });
      for (auto& x : th) x.join();
    }
  }
  if (nt == 2 && std::memcmp(alt.data(), states_out, alt.size() * 8) != 0) return 2;   // both TDMs advance alike
  return 0;
}
'''


def _region(path, name):
    text = open(path).read()
    m = re.search(r"// \[emu:begin %s\][^\n]*\n(.*?)// \[emu:end %s\]" % (name, name), text, re.S)
    assert m, "marker %s not found in %s" % (name, path)
    return m.group(1)


def build(out_dir, values_in_registers=None, popc_per_word=None):
    """Generate + compile the emulator; returns the loaded ctypes library.  ``values_in_registers`` / ``popc_per_word``
    override the kernel's compile-time switches SG_VALUES_IN_REGISTERS / SG_POPC_PER_WORD (the A/B variants of the
    value lookup and of the byte count)."""
    kernel = _region(os.path.join(CSRC, "sample.cu"), "sampler_v2")
    tag = ""
    for name, val in (("SG_VALUES_IN_REGISTERS", values_in_registers), ("SG_POPC_PER_WORD", popc_per_word)):
        if val is not None:
            kernel, n = re.subn(r"constexpr bool %s = [A-Za-z_0-9]+;" % name,
                                "constexpr bool %s = %s;" % (name, "true" if val else "false"), kernel)
            assert n == 1
            tag += "_%s%d" % (name[3:8].lower(), int(bool(val)))
    src = (PRELUDE + _region(os.path.join(CSRC, "kernels.h"), "sampler_args") +
           _region(os.path.join(CSRC, "common.cuh"), "xoro") + _region(os.path.join(CSRC, "common.cuh"), "threshold") +
           kernel + HARNESS)
    cpp = os.path.join(out_dir, "sampler_emu%s.cpp" % tag)
    so = os.path.join(out_dir, "libsampler_emu%s.so" % tag)
    open(cpp, "w").write(src)
    libdir = os.path.join(ROOT, "mppi_numba_b200")
    cmd = ["g++", "-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-Wno-unknown-pragmas", cpp, "-o", so,
           "-L" + libdir, "-l:libb200mppi.so", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    lib = C.CDLL(so)
    P = C.c_void_p
    lib.emu_sample_v2.restype = C.c_int
    lib.emu_sample_v2.argtypes = [C.c_int, P, P, P, P, P, P, P, P] + [C.c_int] * 9 + [C.c_double, C.c_int, P, P]
    return lib


def cumulative_table(pmf, bpad):
    """csrc/sample.cu build_cum_kernel: (B, rows, cols) -> (rows, cols, bpad) running sums clamped to int8, bins
    beyond B repeat the last sum."""
    B, rows, cols = pmf.shape
    acc = np.cumsum(pmf.astype(np.int64), axis=0)
    acc = np.concatenate([acc, np.repeat(acc[-1:], bpad - B, axis=0)], axis=0)
    return np.ascontiguousarray(np.clip(acc, -128, 127).astype(np.int8).transpose(1, 2, 0))
