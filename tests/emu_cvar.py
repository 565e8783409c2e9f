"""Host emulation of the CVaR kernels (TEST INFRASTRUCTURE; tests/emu_core.py): the kernels' text (csrc/rollout.cu
between the ``[emu:... cvar]`` markers, ``warp_sum`` from csrc/common.cuh) is compiled with g++; one std::thread per
CUDA thread, ``__syncthreads()`` = a barrier over the block, the warp collectives (``__reduce_add_sync``,
``__shfl_xor_sync``) = exchanges through a per-warp buffer between two warp barriers."""
from tests.emu_core import build as _build
from tests.emu_core import extern_shared, region, shared_static

HARNESS = r'''
using namespace b200;
// as launch_cvar (csrc/rollout.cu): which kernel, which PER, which grid.  costs_nm: the logical (N, M) array; the
// kernels get the map-major (M, ld) device layout, ld >= N (a row stride larger than the row exercises `ld`).
extern "C" int emu_cvar(const float* costs_nm, float* costs, int N, int M, int ld, float cvar_alpha) {
  if (ld < N) return 2;
  std::vector<float> mn((size_t)M * ld, 12345.0f);
  for (int n = 0; n < N; ++n)
    for (int m = 0; m < M; ++m) mn[(size_t)m * ld + n] = costs_nm[(size_t)n * M + m];
  int numel = (int)std::ceil((double)M * (double)cvar_alpha);
  if (numel < 1) numel = 1;
  if (numel > M) numel = M;
  if (M > 32 * CVAR_MAX_PER_LANE) {
    if (M > (1 << 15)) return 1;
    emu::launch({(unsigned)N, 1, 1}, CVAR_LARGE_THREADS, [&] { cvar_large_kernel(mn.data(), costs, N, ld, M, numel, FlagWait{}); });
    return 0;
  }
  const int nb = cvar_block_n(M);
  const unsigned blocks = (unsigned)((N + nb - 1) / nb);
  emu::cvar_per(M, [&](auto P) {
    emu::launch({blocks, 1, 1}, CVAR_THREADS, [&] { cvar_kernel<decltype(P)::value>(mn.data(), costs, N, ld, M, numel, FlagWait{}); });
  });
  return 0;
}
'''


def kernels(*more):
    """The CVaR kernels' text (``cvar`` region, then the named regions of csrc/rollout.cu) with warp_sum and the
    descriptor of the batched kernels."""
    return [region("kernels.h", "cvar_desc"), region("common.cuh", "warp_sum"),
            extern_shared(shared_static("".join(region("rollout.cu", r) for r in ("cvar",) + more), 3), 1)]


def build(out_dir, extra=""):
    return _build(out_dir, "cvar_emu", kernels(), HARNESS + extra)
