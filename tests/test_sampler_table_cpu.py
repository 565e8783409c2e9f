"""The sampler's one-word threshold entries (breakpoint | q at the bucket start, csrc/common.cuh sample_threshold_q) at
the small alphas where most buckets hold no breakpoint and q stays at 0 or 1 over long runs of draws, evaluated on the
host (b200mppi_debug_sample_threshold) against the oracle's float arithmetic."""
import numpy as np
import pytest

from oracle import terrain_ref as TR


@pytest.fixture(scope="module")
def libmod():
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    return _lib


def _oracle_q(raw, alpha):
    u = ((raw >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)).astype(np.float32)
    return TR.sample_thresholds(u, alpha).astype(np.int64)


@pytest.mark.parametrize("alpha", [0.01, 0.004, 1e-6])
def test_small_alpha_tables_match_reference_arithmetic(libmod, alpha):
    rng = np.random.default_rng(11)
    edges = np.arange(256, dtype=np.uint64) << np.uint64(56)
    raw = np.concatenate([rng.integers(0, 2 ** 64, 100000, dtype=np.uint64), edges, edges + np.uint64(2047),
                          edges + np.uint64(2048), edges - np.uint64(1),
                          np.array([0, 1, 2047, 2048, 4095, 4096, 2 ** 64 - 1], dtype=np.uint64)])
    out = np.empty(raw.shape, np.uint8)
    libmod.check(libmod.lib.b200mppi_debug_sample_threshold(alpha, 127, libmod.ptr(raw), raw.size, libmod.ptr(out)))
    assert (out.astype(np.int64) == _oracle_q(raw, alpha)).all()


def test_zero_alpha_is_refused(libmod):
    """q = 0 for every draw cannot be told apart from "below the breakpoint" in the last bucket: generic kernel."""
    r = np.zeros(2, np.uint64)
    out = np.empty(2, np.uint8)
    assert libmod.lib.b200mppi_debug_sample_threshold(0.0, 127, libmod.ptr(r), 2, libmod.ptr(out)) != 0
