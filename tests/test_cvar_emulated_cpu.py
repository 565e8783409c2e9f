"""The CVaR kernels' real source (warp radix select for M <= 1024, CTA-wide select above), executed on the host
by tests/emu_cvar.py, against the exact mean of the numel largest values (tests/reduce_bounds.py) within a bound
derived from each kernel's reduction depth: ties, signed zeros and +inf at the threshold, negatives, magnitudes
1e-30 .. 1e30, M around every PER step and the CTA kernel, the alpha edge cases, the map-major layout with a row
stride.  The numpy oracle's pairwise tree must stay within its own bound on the same rows."""
import ctypes as C

import numpy as np
import pytest

from oracle import mppi_ref as MR
from tests import reduce_bounds as RB
from tests.emu_cvar import build


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build(str(tmp_path_factory.mktemp("emu_cvar")))


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _alpha_for(M, numel):
    """An alpha whose reference count ceil(M * f32(alpha)) is numel."""
    if numel >= M:
        return 1.0
    a = (numel - 0.5) / M
    assert RB.cvar_numel(M, a) == numel
    return a


SHAPES = [1, 31, 32, 33, 63, 64, 65, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 4097, 16384]
CASES = ([(M, a) for M, a in ((6, 0.5), (33, 0.1), (100, 0.999), (256, 0.5), (1000, 0.25), (1024, 1.0), (7, 0.01),
                               (1, 0.5), (1025, 0.5), (3000, 0.1), (2048, 1.0))]
         # alpha = 0.1: float32(0.1) * 1000 is 100.0000015 -- ceil 101 in float64, 100 in float32
         + [(1000, 0.1)]
         + sorted({(M, _alpha_for(M, k)) for M in SHAPES for k in (1, 2, M - 1, M) if 1 <= k <= M}))
CASES = list(dict.fromkeys(CASES))          # (1024, 1.0) is both a listed case and numel = M


@pytest.mark.parametrize("M,alpha", CASES)
def test_cvar_kernel_source_matches_oracle(emu, M, alpha):
    rng = np.random.default_rng(M)
    N = 9
    c = rng.normal(0, 100, (N, M)).astype(np.float32)
    c[:, ::3] = np.round(c[:, ::3])            # many exact ties
    c[5] = 7.0                                  # all equal
    c[6] = -np.abs(c[6])                        # all negative
    numel = RB.cvar_numel(M, alpha)
    c = np.ascontiguousarray(np.concatenate([c, RB.cvar_rows(M, numel, M + numel)]))
    N = c.shape[0]
    out = np.zeros(N, dtype=np.float32)
    assert emu.emu_cvar(_ptr(c), _ptr(out), N, M, N, np.float32(alpha)) == 0
    label = "M=%d alpha=%r" % (M, alpha)
    RB.check_cvar(out, c, alpha, label=label)
    RB.check_cvar(MR.cvar_reduce(c, alpha), c, alpha, kind="tree", label=label + " (numpy oracle)")
    # the gap row: the numel-th and (numel+1)-th values differ by more than 2 numel bounds, so a select of one element
    # too many or too few lands outside the bound
    if numel < M:
        s = np.sort(c[9])[::-1]
        mu, abs_sum, _ = RB.cvar_exact(c[9:10], alpha)[0]
        assert s[numel - 1] - s[numel] > 2 * numel * RB.cvar_bound(M, numel, abs_sum, mu, RB.kernel_kind(M))


def test_cvar_count_uses_the_float64_product():
    assert RB.cvar_numel(1000, 0.1) == 101
    assert int(np.ceil(np.float32(1000) * np.float32(0.1))) == 100


@pytest.mark.parametrize("M,N,ld", [(64, 70, 96), (256, 33, 33), (1000, 19, 40), (1536, 3, 8),
                                    (257, 21, 37), (1023, 9, 13), (4097, 5, 7)])
def test_cvar_kernel_row_stride_and_ragged_blocks(emu, M, N, ld):
    """Map-major input with a row stride larger than the row (the receive buffer of a sharded solve is (M, N/ws)
    with ld = N/ws; a one-rank buffer has ld = N) and control-sequence counts that do not fill the last CTA: the
    same values reach the same lanes, so the result does not depend on ld, and is within the bound."""
    rng = np.random.default_rng(M + N)
    c = rng.normal(50, 20, (N, M)).astype(np.float32)
    out, one = np.zeros(N, dtype=np.float32), np.zeros(N, dtype=np.float32)
    assert emu.emu_cvar(_ptr(c), _ptr(out), N, M, ld, np.float32(0.3)) == 0
    assert emu.emu_cvar(_ptr(c), _ptr(one), N, M, N, np.float32(0.3)) == 0
    assert (out == one).all()
    RB.check_cvar(out, c, 0.3, label="M=%d N=%d ld=%d" % (M, N, ld))
