"""The batched CTA-wide CVaR kernel (cvar_large_batch_kernel, csrc/rollout.cu: stochastic batches of more than 1024
maps) from its real source on the host, with the technique and hardware stand-ins of tests/emu_cvar.py.  For K planners
of equal N and M, each with its own alpha, one batched launch (grid (N, K)) must equal cvar_large_kernel run once per
planner bit for bit, and each result must lie within the CTA kernel's derived bound around the exact CVaR
(tests/reduce_bounds.py): M from just above the warp kernel's limit to the largest the kernel takes; numel 1, M - 1, M
and the benchmark's alpha 0.2; ties, signed zeros, +-inf and 1e+-30 magnitudes at and around the threshold (the rows of
reduce_bounds.cvar_rows), scattered +inf; a row stride larger than N.  With CvarDesc::active, stopped planners' outputs
stay byte for byte as they were and running planners equal the ungated launch."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tests import emu_cvar
from tests import reduce_bounds as RB
from tests.emu_rollout import _region

F32 = np.float32

HARNESS = r'''
// K planners of equal N and M > 1024, each with its own numel; costs_mn (K, M, ld) map-major.  out_batch: ONE batched
// launch on grid (N, K) (planner blockIdx.y) with each planner's CvarDesc::active = active + k (active null: ungated);
// out_single: cvar_large_kernel once per planner
extern "C" int emu_cvar_large_batch(int K, const float* costs_mn, int N, int M, int ld, const int* numel,
                                    const int* active, float* out_batch, float* out_single) {
  using namespace b200;
  if (M <= 32 * CVAR_MAX_PER_LANE || M > (1 << 15) || ld < N) return 1;
  std::vector<CvarDesc> d(K);
  for (int k = 0; k < K; ++k)
    d[k] = CvarDesc{costs_mn + (size_t)k * M * ld, out_batch + (size_t)k * N, N, ld, M, numel[k],
                    active ? active + k : nullptr};
  if (out_single)
    for (int k = 0; k < K; ++k)
      run([&] { cvar_large_kernel(costs_mn + (size_t)k * M * ld, out_single + (size_t)k * N, N, ld, M, numel[k],
                                  FlagWait{}); }, CVAR_LARGE_THREADS, (unsigned)N);
  for (int k = 0; k < K; ++k)
    run([&] { blockIdx.y = (unsigned)k; cvar_large_batch_kernel(d.data()); }, CVAR_LARGE_THREADS, (unsigned)N);
  return 0;
}
'''


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu_cvar_large_batch"))
    csrc = emu_cvar.CSRC
    rollout = os.path.join(csrc, "rollout.cu")
    kern = _region(rollout, "cvar") + _region(rollout, "cvar_large_batch")
    kern = re.sub(r"(?m)^(\s*)__shared__ ", r"\1static ", kern)
    src = (emu_cvar.PRELUDE + _region(os.path.join(csrc, "kernels.h"), "cvar_desc") +
           _region(os.path.join(csrc, "common.cuh"), "warp_sum") + kern + emu_cvar.HARNESS + HARNESS)
    cpp, so = os.path.join(out, "cvar_large_batch_emu.cpp"), os.path.join(out, "libcvar_large_batch_emu.so")
    open(cpp, "w").write(src)
    r = subprocess.run(["g++", "-O1", "-std=c++20", "-pthread", "-shared", "-fPIC", "-Wno-unknown-pragmas", cpp, "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    lib = C.CDLL(so)
    P, I = C.c_void_p, C.c_int
    lib.emu_cvar_large_batch.restype = I
    lib.emu_cvar_large_batch.argtypes = [I, P, I, I, I, P, P, P, P]
    return lib


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _alpha_for(M, numel):
    """An alpha whose reference count ceil(M * f32(alpha)) is numel."""
    if numel >= M:
        return 1.0
    a = (numel - 0.5) / M
    assert RB.cvar_numel(M, a) == numel
    return a


def planner_rows(M, alphas, seed):
    """Per planner a (N, M) float32 matrix: the value cases of reduce_bounds.cvar_rows for its numel, then two rows of
    scattered +inf (a few, and about a third of the maps)."""
    rng = np.random.default_rng(seed)
    out = []
    for k, a in enumerate(alphas):
        rows = RB.cvar_rows(M, RB.cvar_numel(M, a), seed + k)
        extra = rng.normal(50, 20, (2, M)).astype(F32)
        extra[0, rng.choice(M, 3, replace=False)] = np.inf
        extra[1, rng.choice(M, M // 3, replace=False)] = np.inf
        out.append(np.concatenate([rows, extra]))
    assert len({r.shape for r in out}) == 1
    return out


def map_major(rows, ld):
    """(K, M, ld) float32 from K (N, M) matrices; the columns beyond N hold a value no kernel may read."""
    K, (N, M) = len(rows), rows[0].shape
    mn = np.full((K, M, ld), 12345.0, F32)
    for k, r in enumerate(rows):
        mn[k, :, :N] = r.T
    return np.ascontiguousarray(mn)


@pytest.mark.parametrize("M", [1025, 2048, 4097, 16384])
def test_batched_cta_cvar_equals_single_launches(emu, M):
    alphas = [_alpha_for(M, 1), _alpha_for(M, M - 1), 1.0, 0.2]
    rows = planner_rows(M, alphas, M)
    K, N = len(rows), rows[0].shape[0]
    ld = N + 3
    costs = map_major(rows, ld)
    numel = np.array([RB.cvar_numel(M, a) for a in alphas], np.int32)
    assert numel.tolist() == [1, M - 1, M, int(np.ceil(M * np.float64(F32(0.2))))]
    ob, os_ = np.full((K, N), np.nan, F32), np.full((K, N), -np.nan, F32)
    assert emu.emu_cvar_large_batch(K, _p(costs), N, M, ld, _p(numel), None, _p(ob), _p(os_)) == 0
    assert ob.tobytes() == os_.tobytes()
    for k in range(K):
        RB.check_cvar(ob[k], rows[k], alphas[k], kind="cta", label="M=%d planner %d" % (M, k))
    assert np.isposinf(ob[:, -2:]).all()                  # scattered +inf: every top set holds the largest value
    assert not np.isnan(ob).any()


@pytest.mark.parametrize("M,active", [(1025, [1, 0, 1, 0]), (4097, [0, 1, 1, 0])])
def test_gated_batched_cta_cvar(emu, M, active):
    alphas = [0.5, 0.1, 1.0, 0.2]
    rows = planner_rows(M, alphas, 7 * M)
    K, N = len(rows), rows[0].shape[0]
    costs = map_major(rows, N)
    numel = np.array([RB.cvar_numel(M, a) for a in alphas], np.int32)
    act = np.array(active, np.int32)
    sentinel = np.full((K, N), -3.0, F32)
    gated, full = sentinel.copy(), np.full((K, N), np.nan, F32)
    assert emu.emu_cvar_large_batch(K, _p(costs), N, M, N, _p(numel), _p(act), _p(gated), None) == 0
    assert emu.emu_cvar_large_batch(K, _p(costs), N, M, N, _p(numel), None, _p(full), None) == 0
    for k in range(K):
        want = full[k] if active[k] else sentinel[k]
        assert gated[k].tobytes() == want.tobytes(), "planner %d (active %d)" % (k, active[k])
