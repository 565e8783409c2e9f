"""xoroshiro128+ exactly as numba.cuda.random implements it (numba 0.65.0,
numba/cuda/random.py:47-197) -- the third-party generator behind the reference's
``sample_noise_numba`` (mppi.py:1354-1370) and ``sample_grids_numba`` (terrain.py:633-694).

TEST INFRASTRUCTURE (see oracle/__init__.py).  States are ``uint64[n, 2]`` = (s0, s1), the
same 16-byte layout as numba's ``xoroshiro128p_dtype``.
"""
import numpy as np

U64 = np.uint64
MASK = (1 << 64) - 1
JUMP = (0xBEAC0467EBA5FACB, 0xD86B048B86AA9922)          # random.py:112


def splitmix64(seed: int) -> int:
    """random.py:60-66 -- one SplitMix64 output; both state words start as it."""
    z = (seed + 0x9E3779B97F4A7C15) & MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


def _rotl(x, k):
    return (x << U64(k)) | (x >> U64(64 - k))


def next_u64(states: np.ndarray, idx=None) -> np.ndarray:
    """random.py:81-99: result = s0 + s1 (before the update); rotations 55/14/36.
    Advances ``states[idx]`` in place (all states if idx is None) and returns uint64 results."""
    sel = slice(None) if idx is None else idx
    s0 = states[sel, 0].copy()
    s1 = states[sel, 1].copy()
    with np.errstate(over="ignore"):
        result = s0 + s1
    s1 ^= s0
    states[sel, 0] = _rotl(s0, 55) ^ s1 ^ (s1 << U64(14))
    states[sel, 1] = _rotl(s1, 36)
    return result


def _next_scalar(s0: int, s1: int):
    r = (s0 + s1) & MASK
    s1 ^= s0
    ns0 = (((s0 << 55) | (s0 >> 9)) & MASK) ^ s1 ^ ((s1 << 14) & MASK)
    ns1 = ((s1 << 36) | (s1 >> 28)) & MASK
    return r, ns0, ns1


def jump_scalar(s0: int, s1: int):
    """random.py:103-126: advance one state by 2**64 steps."""
    a0 = a1 = 0
    for word in JUMP:
        for b in range(64):
            if word & (1 << b):
                a0 ^= s0
                a1 ^= s1
            _, s0, s1 = _next_scalar(s0, s1)
    return a0, a1


def _bits_of(states: np.ndarray) -> np.ndarray:
    """uint64[n,2] -> uint8[128, n] little-endian bit matrix (row b = bit b of s0, 64+b of s1)."""
    n = states.shape[0]
    out = np.empty((128, n), dtype=np.float32)
    for w in range(2):
        col = states[:, w]
        for b in range(64):
            out[64 * w + b] = ((col >> U64(b)) & U64(1)).astype(np.float32)
    return out


def _states_of(bits: np.ndarray) -> np.ndarray:
    n = bits.shape[1]
    st = np.zeros((n, 2), dtype=U64)
    ib = bits.astype(np.uint64)
    for w in range(2):
        for b in range(64):
            st[:, w] |= ib[64 * w + b] << U64(b)
    return st


def _jump_matrix() -> np.ndarray:
    """128x128 GF(2) matrix of the 2**64 jump (it is linear in the state): column j is the
    jump applied to basis state e_j."""
    basis = np.zeros((128, 2), dtype=U64)
    for j in range(128):
        basis[j, j // 64] = U64(1) << U64(j % 64)
    acc = np.zeros_like(basis)
    cur = basis.copy()
    for word in JUMP:
        for b in range(64):
            if word & (1 << b):
                acc ^= cur
            next_u64(cur)
    return _bits_of(acc)            # [128 (out bit), 128 (basis j)]


def create_states(n: int, seed: int, subsequence_start: int = 0) -> np.ndarray:
    """random.py:226-241 ``init_xoroshiro128p_states_cpu``: state 0 = splitmix64(seed) in both
    words (jumped ``subsequence_start`` times), state i = state i-1 jumped 2**64 steps.
    The reference builds this sequentially; here by doubling with the GF(2) jump matrix so
    that a million states take a second (results are identical -- the jump is linear)."""
    z = splitmix64(int(seed) & MASK)
    s0, s1 = z, z
    for _ in range(subsequence_start):
        s0, s1 = jump_scalar(s0, s1)
    states = np.array([[s0, s1]], dtype=U64)
    if n <= 1:
        return states[:n].copy()
    if n <= 64:                                   # small: literal sequential restatement
        out = [(s0, s1)]
        for _ in range(1, n):
            out.append(jump_scalar(*out[-1]))
        return np.array(out, dtype=U64)
    J = _jump_matrix()                            # J^(len(bits)) applied to the first block
    bits = _bits_of(states)
    Jk = J
    while bits.shape[1] < n:
        nxt = np.mod(Jk @ bits, 2.0)
        bits = np.concatenate([bits, nxt], axis=1)
        Jk = np.mod(Jk @ Jk, 2.0)
    return _states_of(bits[:, :n])


def uniform_float32(x: np.ndarray) -> np.ndarray:
    """random.py:130-154: float32( (x >> 11) * 2**-53 computed in float64 )."""
    return ((x >> U64(11)).astype(np.float64) * (1.0 / (1 << 53))).astype(np.float32)


TWO_PI_F32 = np.float32(2 * np.pi)                 # random.py:172


def normal_float32(states: np.ndarray, idx=None, arith=None) -> np.ndarray:
    """random.py:176-197: Box-Muller in float32, two draws per call, the sine branch is
    discarded.  (Compiled for CUDA this uses libdevice's precise logf/cosf and sqrt.approx;
    by default numpy's float32 log/cos/sqrt are the exact-math stand-in -- SURVEY.md 2.3; an exact
    ``arith`` (oracle/arith.py) takes them from its provider and rounds each product once, as
    csrc/common.cuh::xoro_normal does.)"""
    u1 = uniform_float32(next_u64(states, idx))
    u2 = uniform_float32(next_u64(states, idx))
    if arith is not None and arith.exact:
        with np.errstate(divide="ignore", invalid="ignore"):
            r = arith.sqrt32(arith.mul32(np.float32(-2.0), arith.logf32(u1)))
            return arith.mul32(r, arith.cosf32(arith.mul32(TWO_PI_F32, u2)))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.sqrt(np.float32(-2.0) * np.log(u1))
        return (r * np.cos(TWO_PI_F32 * u2)).astype(np.float32)
