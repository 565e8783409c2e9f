"""Host emulation of the sampler kernel (TEST INFRASTRUCTURE; tests/emu_core.py).

The text of sample_grids_v2_kernel and the device helpers it uses is lifted verbatim from the CUDA sources (the
regions between ``[emu:begin ...]`` / ``[emu:end ...]`` markers in csrc/sample.cu, csrc/common.cuh and
csrc/kernels.h) and compiled with g++ against tests/emu_cuda.h: the thread / block indices are thread-local variables,
``__syncthreads()`` is a std::barrier over the block's threads (one std::thread per CUDA thread, blocks run one
after the other), ``__shared__`` memory is one static buffer, ``__popc`` / ``__byte_perm`` / ``__ldg`` are
functions.  The host-side table builders (threshold buckets, GF(2) jump matrices) are the library's own, linked
from libb200mppi.so.  This lets the CPU test-suite run the REAL kernel source on small maps and compare it bit
for bit with the oracle -- no GPU needed."""
import re

import numpy as np

from tests.emu_core import build as _build
from tests.emu_core import extern_shared, region

HARNESS = r'''
using namespace b200;
// nt TDMs (1 or 2) sampled from the generator states `states` (numba layout, gen = tix*(ty*M)+m*ty+tiy).
// cum: (nt)(rows, cols, bpad) int8 running sums; grids: (nt)(M, grid_rows, pitch); qvals: (nt)(128).
// disc = {cx, cy, r} (cells) or null: the reach disc inside the box (per-CTA narrowing of the tile columns).
// box = {row_lo, row_hi, col_lo, col_hi} (cells) or null: with a box the launch is restricted as apply_box (api.cu)
// does it and the states come from advance_states_kernel -- what plan_launch does for a boxed solve.
extern "C" int emu_sample_v2(int nt, int8_t* grid0, int8_t* grid1, const int8_t* cum0, const int8_t* cum1,
                             const uint64_t* states, uint64_t* states_out, const int8_t* qv0, const int8_t* qv1, int bpad,
                             int rows, int cols, int grid_rows, int pitch, int tx, int ty, int num_maps, int segs,
                             double alpha, int q_cap, const int* box, const float* disc) {
  SampleGridsV2Args a{};
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
  std::vector<uint64_t> J;
  emu::segment_jumps(rows, cols, tx, ty, segs, a.seg_rows, J);
  a.jump = J.empty() ? nullptr : J.data();
  a.rows = rows; a.cols = cols; a.grid_rows = grid_rows; a.pitch = pitch; a.tx = tx; a.ty = ty; a.num_maps = num_maps;
  a.segs = segs;
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
  const EmuDim3 grid{(unsigned)((tix_hi - a.tix_lo + 1) * segs), (unsigned)((num_maps + a.gm - 1) / a.gm), 1};
  emu::sampler_nw(bpad, [&](auto NW) {
    if (nt == 1) emu::launch(grid, threads, [&] { sample_grids_v2_kernel<1, decltype(NW)::value>(a); });
    else emu::launch(grid, threads, [&] { sample_grids_v2_kernel<2, decltype(NW)::value>(a); });
  });
  if (box) {                           // launch_advance_states (sample.cu)
    int64_t ks[4];
    const int nr = (rows + tx - 1) / tx, nc = (cols + ty - 1) / ty;           // sample_tile_draws
    const int last_h = rows % nr ? rows % nr : nr, last_w = cols % nc ? cols % nc : nc;
    ks[0] = (int64_t)nr * nc; ks[1] = (int64_t)nr * last_w; ks[2] = (int64_t)last_h * nc; ks[3] = (int64_t)last_h * last_w;
    std::vector<uint64_t> mats(4 * 256);
    build_jump_matrices(ks, 4, mats.data());
    const int64_t total = (int64_t)tx * ty * num_maps;
    emu::launch({(unsigned)((total + 127) / 128), 1, 1}, 128, [&] {   // 128 threads per block: the kernel stages in shared memory
      advance_states_kernel(reinterpret_cast<const ulonglong2*>(states), reinterpret_cast<ulonglong2*>(states_out),
                            nt == 2 ? reinterpret_cast<ulonglong2*>(alt.data()) : nullptr,
                            reinterpret_cast<const ulonglong2*>(mats.data()), rows, cols, tx, ty, num_maps);
    });
  }
  if (nt == 2 && std::memcmp(alt.data(), states_out, alt.size() * 8) != 0) return 2;   // both TDMs advance alike
  return 0;
}
'''

# the completion kernel's entry point (needs the window_complete region)
WINDOW_COMPLETE = r'''// window-first sampling's completion (stage_rollout, api.cu): sample_window_complete_kernel on the fused pair's
// whole-map plan (as emu_sample_v2 without a box) from the pre-call states, write_states = 0, with the reach-box
// decision off (record[0..4] = whole maps).  esc[M]: this solve's flags; clear[M]: the other parity's (zeroed);
// record[6].  Returns the plan's maps per CTA (> 0) or an error (< 0).
extern "C" int emu_window_complete(int8_t* grid0, int8_t* grid1, const int8_t* cum0, const int8_t* cum1,
                                   const uint64_t* states, const int8_t* qv0, const int8_t* qv1, int bpad, int rows,
                                   int cols, int grid_rows, int pitch, int tx, int ty, int num_maps, double alpha,
                                   int q_cap, const unsigned char* esc, unsigned char* clear, int* record) {
  SampleGridsV2Args a{};
  a.t[0] = SampleTdm{grid0, cum0, states, nullptr, qv0, bpad};
  a.t[1] = SampleTdm{grid1, cum1, states, nullptr, qv1, bpad};
  std::vector<uint64_t> T(SAMPLE_TABLE_WORDS);
  if (!build_sample_thresholds(alpha, q_cap, T.data())) return -1;
  a.thresholds = T.data();
  std::vector<uint64_t> J;
  int segs = 1;
  emu::segment_jumps(rows, cols, tx, ty, segs, a.seg_rows, J);
  a.jump = nullptr;
  a.rows = rows; a.cols = cols; a.grid_rows = grid_rows; a.pitch = pitch; a.tx = tx; a.ty = ty; a.num_maps = num_maps;
  a.segs = segs;
  sample_box_full(a);
  if (a.ty * a.gm > 256) a.gm = 256 / a.ty;
  a.write_states = 0;
  const ReachBoxConst c{};
  const float reach = 0.0f;
  const int threads = ((a.nact * a.gm + 31) / 32) * 32;              // v2_threads
  if (threads > 256 || a.gm < 1) return -3;
  const EmuDim3 grid{(unsigned)(tx * segs), (unsigned)((num_maps + a.gm - 1) / a.gm), 1};
  emu::sampler_nw(bpad, [&](auto NW) {
    emu::launch(grid, threads, [&] {
      sample_window_complete_kernel<decltype(NW)::value>(a, c, 0.0f, 0.0f, &reach, record, esc, clear);
    });
  });
  return a.gm;
}
'''


def kernels(kernel=None, *more):
    """The sampler's text (``kernel``: the sampler_v2 region, possibly edited; then the named regions of
    csrc/sample.cu) with its argument structs, the generator step and the threshold lookup."""
    kernel = region("sample.cu", "sampler_v2") if kernel is None else kernel
    return [region("kernels.h", "sampler_args"), region("kernels.h", "box_desc"), region("common.cuh", "xoro"),
            region("common.cuh", "threshold"), extern_shared(kernel + "".join(region("sample.cu", r) for r in more), 2)]


def build(out_dir, values_in_registers=None, popc_per_word=None, extra="", more=()):
    """Generate + compile the emulator; returns the loaded ctypes library.  ``values_in_registers`` / ``popc_per_word``
    override the kernel's compile-time switches SG_VALUES_IN_REGISTERS / SG_POPC_PER_WORD (the A/B variants of the
    value lookup and of the byte count); ``more``: further regions of csrc/sample.cu (e.g. ``window_complete``)."""
    kernel = region("sample.cu", "sampler_v2")
    tag = ""
    for name, val in (("SG_VALUES_IN_REGISTERS", values_in_registers), ("SG_POPC_PER_WORD", popc_per_word)):
        if val is not None:
            kernel, n = re.subn(r"constexpr bool %s = [A-Za-z_0-9]+;" % name,
                                "constexpr bool %s = %s;" % (name, "true" if val else "false"), kernel)
            assert n == 1
            tag += "_%s%d" % (name[3:8].lower(), int(bool(val)))
    tag += "".join("_" + m for m in more)
    harness = HARNESS + (WINDOW_COMPLETE if "window_complete" in more else "") + extra
    return _build(out_dir, "sampler_emu" + tag, kernels(kernel, *more), harness, link_engine=True)


def cumulative_table(pmf, bpad):
    """csrc/sample.cu build_cum_kernel: (B, rows, cols) -> (rows, cols, bpad) running sums clamped to int8, bins
    beyond B repeat the last sum."""
    B, rows, cols = pmf.shape
    acc = np.cumsum(pmf.astype(np.int64), axis=0)
    acc = np.concatenate([acc, np.repeat(acc[-1:], bpad - B, axis=0)], axis=0)
    return np.ascontiguousarray(np.clip(acc, -128, 127).astype(np.int8).transpose(1, 2, 0))
