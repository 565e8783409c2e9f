"""The windowed (TMA-staged) rollout kernel's real source -- the kernel solve() runs in the stochastic mode -- and
its prepare kernel, executed on the host by tests/emu_rollout_win.py, against the per-(n,m) costs the REFERENCE's
rollout_numba produced for the same inputs (tests/golden/ref_rollout.npz), with the window around the robot, with
the window pushed away so that every lookup takes the global-memory path, and against the generic kernel."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.emu_rollout import build as build_generic
from tests.emu_rollout_win import build
from tests.test_rollout_emulated_cpu import _c, _fparams, _p, _ratios

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F32 = np.float32


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("emu_win"))
    return build(d), build_generic(d)


@pytest.mark.parametrize("gname", ["near", "far"])
def test_windowed_kernel_matches_reference_and_generic_kernel(emu, gname):
    win, gen = emu
    g = np.load(os.path.join(GOLDEN, "ref_rollout.npz"))
    lin, ang = _c(g["lin"], np.int8), _c(g["ang"], np.int8)
    obs, unk = _c(g["obs"], np.int8), _c(g["unk"], np.int8)
    noise, u_cur = _c(g["noise"], F32), _c(g["u_cur"], F32)
    M, R, Cc = lin.shape
    Hp, Wp = obs.shape
    N, T = noise.shape[:2]
    f = _fparams(g["res"], g["xlim"][0], g["ylim"][0], g["dt"], g["x0"], g["xgoal_" + gname], g["goal_tol"], g["v_post"],
                 g["lam"], g["u_std"], g["vrange"], g["wrange"], g["obs_cost"], g["unk_cost"], g["dist_weight"],
                 g["lin_bounds"][0], g["ang_bounds"][0])
    ratios = _ratios(g["lin_bounds"], g["ang_bounds"])
    geo = _c([Hp, Wp, R, Cc, Cc, Wp, T, N, M], np.int32)
    ref = g["sto_cnm_" + gname]

    m01 = int(((obs & ~1) == 0).all() and ((unk & ~1) == 0).all())     # the kernel variant the launcher would pick

    def run_win(sx, sy):
        out = np.zeros((N, M), F32)
        origin = np.zeros(2, np.int32)
        reach = np.zeros(1, F32)
        assert win.emu_rollout_win(_p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), _p(noise), _p(u_cur),
                                   _p(out), sx, sy, _p(origin), _p(reach), 0, 1, 0, 0, m01) == 0
        return out, origin
    inside, origin = run_win(0, 0)
    assert origin[0] % 16 == 0                                    # TMA: 16-byte aligned inner coordinate
    assert (np.abs(inside - ref) / np.maximum(np.abs(ref), 1e-6)).max() < 5e-6
    shifted, origin2 = run_win(4000, -4000)                       # the window is clamped into the map (here: the whole map)
    assert 0 <= origin2[0] <= max(Cc - 240, 0) and 0 <= origin2[1] <= max(R - 232, 0)
    assert (shifted == inside).all()                              # same numbers wherever the window sits
    cnm, costs = np.zeros((N, M), F32), np.zeros(N, F32)
    gen.emu_rollout(0, _p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), None, _p(noise), _p(u_cur), _p(cnm),
                    _p(costs), None, 0)
    # the generic kernel adds the control-cost terms one by one, the windowed one adds their pre-summed total: ~1 ulp
    assert (np.abs(inside - cnm) / np.maximum(np.abs(cnm), 1e-6)).max() < 2e-6


def test_two_sided_floor_criterion_never_disagrees_with_the_reference_floor_division():
    """The windowed kernel takes floor(a/res) from round-down magic-number sums at both ends of the interval
    [a*inv*(1-2.4e-7) - 1e-30, a*inv*(1+2.4e-7) + 1e-30] and trusts it only when both ends give the same integer.
    Whenever they do, the integer must be what the reference's float floor-division yields (oracle floor_div_f32,
    numba real_divmod as compiled): random positions, positions within 1e-5 cells of an edge, exact multiples of the
    resolution, tiny and denormal offsets, ten resolutions."""
    from oracle.mppi_ref import floor_div_f32
    rng = np.random.default_rng(0)
    MAGIC = F32(12582912.0)

    def fadd_rd(a, b):                       # round-down add from the rounded sum and its exact error (TwoSum)
        b = np.full_like(a, b)
        s = (a + b).astype(F32)
        bb = (s - a).astype(F32)
        err = ((a - (s - bb).astype(F32)).astype(F32) + (b - bb).astype(F32)).astype(F32)
        r = s.copy()
        r[err < 0] = np.nextafter(s[err < 0], F32(-np.inf))
        return r

    def fma32(a, b, c):
        return (a.astype(np.longdouble) * np.longdouble(b) + np.longdouble(c)).astype(F32)
    total = trusted = 0
    for res in (0.05, 0.1, 0.2, 0.25, 0.5, 1.0, 2.0, 0.3, 0.07, 3.3):
        r = F32(res)
        inv = F32(1.0) / r
        inv_lo, inv_hi = F32(inv * F32(1.0 - 2.4e-7)), F32(inv * F32(1.0 + 2.4e-7))
        n = 200000
        k = rng.integers(-300, 2500, n)
        # edge-hugging positions: within 1e-5, 1e-6 cells and a few float32 ulps (relative 1e-7 .. 4e-7) of an edge
        near = [(k * np.float64(res) * (1.0 + rng.choice([-1, 1], n) * rng.uniform(0.5e-7, 4e-7, n))).astype(F32),
                (k * np.float64(res) + rng.normal(0, 1e-6, n) * res).astype(F32)]
        near += [np.nextafter(near[0], F32(np.inf)), np.nextafter(near[0], F32(-np.inf))]
        sets = tuple(near) + (rng.uniform(-50, 250, n).astype(F32), (k * np.float64(res) + rng.normal(0, 1e-5, n) * res).astype(F32),
                (k * np.float64(res)).astype(F32), rng.uniform(-1e-6, 1e-6, n).astype(F32),
                (rng.uniform(-1, 1, n) * 10.0 ** rng.uniform(-37, -5, n)).astype(F32),
                np.array([0.0, -0.0, 1.2e-38, -1.2e-38], F32))
        for a in sets:
            kl = fadd_rd(fma32(a, inv_lo, -1e-30), MAGIC)
            kh = fadd_rd(fma32(a, inv_hi, 1e-30), MAGIC)
            same = kl.view(np.int32) == kh.view(np.int32)
            idx = kl.view(np.int32) - np.int32(0x4B400000)
            assert (idx[same] == floor_div_f32(a, r)[same]).all(), res
            total += a.size
            trusted += int(same.sum())
    assert trusted > 0.4 * total             # the criterion is not vacuous (random positions pass it ~99.9 % of the time)


def test_windowed_kernel_on_a_cell_edge_takes_the_exact_sequence(emu):
    """A robot standing exactly on a cell edge (a = k*res, the interval around a/res contains the integer k): the
    two-sided test must refuse and the exact sequence must pick cell k -- an obstacle placed in that cell and
    nowhere else has to show up in every step's cost, in the windowed and in the generic kernel alike."""
    win, gen = emu
    res, T, N, M = F32(0.25), 6, 40, 2
    R = Cc = 32
    lin = np.full((M, R, Cc), 50, np.int8)
    ang = np.full((M, R, Cc), 50, np.int8)
    obs = np.zeros((R, Cc), np.int8)
    unk = np.zeros((R, Cc), np.int8)
    obs[5, 7] = 1
    xlo, ylo = F32(-1.0), F32(2.0)
    x0 = [float(F32(xlo + 7 * res)), float(F32(ylo + 5 * res)), 0.3]          # exactly on the lower edges of cell (5, 7)
    noise, u_cur = np.zeros((N, T, 2), F32), np.zeros((T, 2), F32)             # no motion: every step looks up (5, 7)
    f = _fparams(res, xlo, ylo, 0.1, x0, [30.0, 30.0], 0.5, 0.01, 1.0, [2, 3], [0, 3], [-np.pi, np.pi], 1e5, 1e2, 1.0, 0.0, 0.0)
    ratios = _ratios([0, 1], [0, 1])
    geo = _c([R, Cc, R, Cc, Cc, Cc, T, N, M], np.int32)
    out = np.zeros((N, M), F32)
    assert win.emu_rollout_win(_p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), _p(noise), _p(u_cur), _p(out),
                               0, 0, None, None, 0, 1, 0, 1, 0) == 0
    cnm, costs = np.zeros((N, M), F32), np.zeros(N, F32)
    gen.emu_rollout(0, _p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), None, _p(noise), _p(u_cur), _p(cnm),
                    _p(costs), None, 0)
    assert (out == cnm).all()
    assert (out > T * 1e5).all() and (out < (T + 1) * 1e5).all()          # the obstacle penalty of cell (5, 7), T times


@pytest.mark.parametrize("ctas,blocks,unit,sync", [(0, 1, 0, 0), (1, 1, 0, 0), (3, 1, 0, 1), (7, 3, 0, 0), (5, 7, 0, 1), (3, 1, 32, 0),
                                                   (2, 1, 16, 1), (1, 1, 32, 1), (2, 1, -1, 0), (5, 3, -1, 0), (7, 1, -1, 1),
                                                   (4, 1, 0, 0)])
def test_windowed_kernel_multi_tile_random_scenario_matches_generic_kernel_and_oracle(emu, ctas, blocks, unit, sync):
    """N = 2100 control sequences (66 chunks of 32 per map, the last one ragged) x 2 maps on a persistent grid of
    `ctas` CTAs (0: the launcher's own rule): shares of 132 chunks that start and end inside a map, CTAs that
    stage two windows one after the other, warps pulling chunks from the shared counter; 200 x 200 cells of random
    traction, obstacles and unknown cells, T = 40: windowed kernel == generic kernel (~1 ulp: pre-summed control
    cost) whatever the grid, and both follow the oracle.  blocks > 1: the sharded destination layout -- every cost
    stored into the "receive buffer" of the rank that reduces its control sequence, flags raised once by the last
    CTA (checked inside the harness).  N = 2100 = 3 x 700 = 7 x 300.  unit > 0: share boundaries at multiples of
    `unit` chunks (0 = the launcher's rule; -1 = shares that never cross a map: map m gets ctas/M or one more of the
    CTAs, what the launcher picks for short shares when there are at least as many CTAs as maps); sync = 1: the chunks are dealt pass by pass with a CTA barrier in between
    (what the launcher picks for short shares) instead of pulled from the shared counter.  The masks hold only 0 / 1:
    both penalty variants of the kernel (MASK01 and the general one) run, alternating over the parameter sets;
    ctas = 4: obstacle bytes in -3 .. 3 through the general variant."""
    from tests.scenarios import make_scenario, oracle_rollout_costs   # noqa: F401  (scenario generator only)
    from oracle import mppi_ref as MR
    win, gen = emu
    rng = np.random.default_rng(5)
    N, M, T, R, Cc = 2100, 2, 40, 420, 400                  # larger than the 240 x 232 window
    res = F32(0.1)
    lin = rng.integers(0, 101, (M, R, Cc)).astype(np.int8)
    ang = rng.integers(0, 101, (M, R, Cc)).astype(np.int8)
    obs = (rng.random((R, Cc)) < 0.02).astype(np.int8)
    if ctas == 4:                                            # mask bytes other than 0 / 1 (-3 .. 3): the general penalty variant only
        obs = (obs * rng.integers(-3, 4, (R, Cc))).astype(np.int8)
    unk = (rng.random((R, Cc)) < 0.02).astype(np.int8)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(F32)
    u_cur = np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(F32)
    x0 = [20.03, 19.97, 0.7]
    goal = [23.0, 22.0]                                      # within reach: some rollouts exit early
    f = _fparams(res, 0.0, 0.0, 0.1, x0, goal, 0.5, 0.01, 1.0, [2, 3], [0, 3], [-np.pi, np.pi], 1e5, 1e2, 1.0, 0.0, 0.0)
    ratios = _ratios([0, 1], [0, 1])
    geo = _c([R, Cc, R, Cc, Cc, Cc, T, N, M], np.int32)
    out = np.zeros((N, M), F32)
    reach = np.zeros(1, F32)
    assert win.emu_rollout_win(_p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), _p(noise), _p(u_cur), _p(out),
                               0, 0, None, _p(reach), ctas, blocks, unit, sync, 0 if ctas == 4 else (ctas + blocks) & 1) == 0
    # the reach statistic of the prepare kernel: max_n sum_t |clip(u_v + e_v)|, never below the exact sum
    vsum = np.abs(np.clip(u_cur[None, :, 0] + noise[:, :, 0], 0, 3).astype(np.float64)).sum(1).max()
    assert vsum <= float(reach[0]) <= vsum * (1 + 1e-5)
    cnm, costs = np.zeros((N, M), F32), np.zeros(N, F32)
    gen.emu_rollout(0, _p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), None, _p(noise), _p(u_cur), _p(cnm),
                    _p(costs), None, 0)
    rel = np.abs(out - cnm) / np.maximum(np.abs(cnm), 1e-6)
    assert rel.max() < 2e-6, rel.max()
    want = MR.rollout_costs(MR.MODE_STOCHASTIC, lin, ang, [0, 1], [0, 1], obs, unk, res, [0.0, Cc * 0.1], [0.0, R * 0.1],
                            [0, 3], [-np.pi, np.pi], goal, 0.01, 1e5, 1e2, 0.5, 1.0, [2, 3], x0, 0.1, 1.0, noise, u_cur)
    r2 = np.abs(out - want) / np.maximum(np.abs(want), 1e-6)
    assert (r2 < 1e-4).mean() > 0.995 and np.median(r2) < 2e-6          # libm vs numpy sin/cos: a few cell flips at most
    assert (out < 0.5 * np.median(out)).any()                          # early exits happened
    if ctas == 3:
        # window pushed 110 cells right / 100 up: the robot sits near its edge, many lookups take the global-memory
        # path (the generic kernel's wrap + clamp) -- same numbers whatever the source of the bytes
        out2 = np.zeros((N, M), F32)
        origin = np.zeros(2, np.int32)
        assert win.emu_rollout_win(_p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), _p(noise), _p(u_cur),
                                   _p(out2), 110, 100, _p(origin), None, ctas, 1, 0, sync, 0 if ctas == 4 else 1 - ((ctas + blocks) & 1)) == 0
        assert origin[0] % 16 == 0 and origin[0] > 80 + 16 and origin[1] > 80
        assert (out2 == out).all()


@pytest.mark.parametrize("N,T", [(100, 50), (64, 128), (37, 3), (257, 33)])
def test_fused_noise_and_controls_kernel_equals_the_two_kernels(emu, N, T):
    """noise_prepare_kernel (what solve() launches) against sample_noise + prepare_rollout one after the other:
    generator states, noise, float64 controls, control costs, reach statistic bit for bit (compared inside the
    harness); the noise is the reference stream (oracle/xoroshiro.py)."""
    from oracle import xoroshiro as X
    win, _ = emu
    rng = np.random.default_rng(N + T)
    states = np.ascontiguousarray(X.create_states(N * T, 5))
    u_cur = np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(F32)
    vr, wr = _c([0, 3], F32), _c([-np.pi, np.pi], F32)
    npad = (N + 31) // 32 * 32
    st_out = np.zeros_like(states)
    noise, noiseT = np.zeros((N, T, 2), F32), np.zeros((T, npad, 2), np.float64)
    ctrl, reach = np.zeros(npad, F32), np.zeros(1, F32)
    rc = win.emu_noise_prepare(_p(states), _p(u_cur), N, T, F32(2.0), F32(3.0), F32(1.0), _p(vr), _p(wr), _p(st_out), _p(noise),
                               _p(noiseT), _p(ctrl), _p(reach))
    assert rc == 0, rc
    from oracle import mppi_ref as MR
    want_states = states.copy()
    want = MR.sample_noise(want_states, np.array([2.0, 3.0], F32), N, T)
    np.testing.assert_allclose(noise, want, rtol=3e-6, atol=2e-6)
    assert (st_out == want_states).all()
    assert (noiseT[:, :N, 0] == np.clip(u_cur[:, None, 0] + noise[:, :, 0].T, 0, 3).astype(np.float64)).all()
    assert (noiseT[:, :N, 1] == np.clip(u_cur[:, None, 1] + noise[:, :, 1].T, F32(-np.pi), F32(np.pi)).astype(np.float64)).all()


@pytest.mark.parametrize("case", ["big_then_tiny", "tiny_then_big", "reverse", "reverse_tiny", "random"])
def test_reach_statistic_bounds_the_exact_path_length(emu, case):
    """The reach box rests on the prepare kernel's statistic: it must never fall below the exact float64 sum of the
    float32 |v| each rollout uses, even where a round-to-nearest float32 sum loses terms (T = 1024: one large |v| and
    1023 tiny ones below half its ulp), nor with a negative vrange (reverse driving).  Round-up adds overshoot by at
    most one ulp of the sum per step."""
    win, _ = emu
    N, T = 70, 1024
    rng = np.random.default_rng(len(case))
    vr = _c({"reverse": [-3, -0.5], "reverse_tiny": [-3, 0]}.get(case, [0, 3]), F32)
    wr = _c([-np.pi, np.pi], F32)
    u_cur = np.zeros((T, 2), F32)
    noise = np.zeros((N, T, 2), F32)
    if case == "big_then_tiny":
        u_cur[0, 0] = 2.5
        noise[:, 1:, 0] = rng.uniform(1e-8, 1e-7, (N, T - 1))          # each below half an ulp of 2.5 (1.2e-7)
    elif case == "tiny_then_big":
        noise[:, :-1, 0] = rng.uniform(1e-9, 3e-8, (N, T - 1))
        u_cur[-1, 0] = 2.9
    elif case == "reverse":
        u_cur[:, 0] = -1.7
        noise[..., 0] = rng.standard_normal((N, T)) * 0.8
    elif case == "reverse_tiny":
        u_cur[0, 0] = -2.75
        noise[:, 1:, 0] = -rng.uniform(1e-8, 1e-7, (N, T - 1))
    else:
        u_cur[:, 0] = rng.uniform(0, 2, T)
        noise[..., 0] = rng.standard_normal((N, T)) * 2
    noise[..., 1] = rng.standard_normal((N, T))
    noise = np.ascontiguousarray(noise)
    reach = float(win.emu_prepare_reach(_p(noise), _p(u_cur), N, T, _p(vr), _p(wr)))
    v = np.clip((u_cur[None, :, 0] + noise[..., 0]).astype(F32), vr[0], vr[1]).astype(F32)     # fminf / fmaxf clip
    exact = np.abs(v.astype(np.float64)).sum(1)
    assert reach >= exact.max(), (case, reach, exact.max())
    assert reach <= exact.max() + T * float(np.spacing(F32(reach))), (case, reach, exact.max())
    rn = np.zeros(N, F32)                                    # what a round-to-nearest float32 sum would have given
    for t in range(T):
        rn = (rn + np.abs(v[:, t])).astype(F32)
    if case in ("big_then_tiny", "reverse_tiny"):
        assert float(rn.max()) < exact.max()                 # the case is adversarial: round-to-nearest loses the tail


def test_veltkamp_split_equals_float32_rounding_including_ties():
    """round_to_f32_precision (csrc/rollout_win.cu, WIN_ROUND_FP64): g = RN(a * (2^29 + 1)), hi = RN(g + RN(a - g)) must be
    the float64 value of float32(a) -- round to nearest, ties to EVEN -- for every magnitude the state can take.  numpy
    float64 arithmetic is the same IEEE arithmetic as the kernel's __dmul_rn / __dsub_rn / __dadd_rn.  10^7 values within
    a few float64 ulps of a 24-bit tie (both parities, binade ends included), exact ties, and random mantissas."""
    rng = np.random.default_rng(2)

    def split_hi(a):
        g = a * np.float64(2 ** 29 + 1)
        return g + (a - g)

    for _ in range(20):
        m = rng.integers(2 ** 23, 2 ** 24, 500000).astype(np.float64)
        m[:1000] = 2 ** 24 - 1
        m[1000:2000] = 2 ** 23
        e = rng.integers(-60, 60, 500000)
        off = rng.integers(-3, 4, 500000).astype(np.float64)            # float64 ulps around the tie (2^-29 at this scale)
        a = (m + 0.5 + off * 2.0 ** -29) * 2.0 ** e * rng.choice([-1.0, 1.0], 500000)
        assert (split_hi(a) == a.astype(np.float32).astype(np.float64)).all()
    a = rng.integers(2 ** 52, 2 ** 53, 2000000).astype(np.float64) * 2.0 ** rng.integers(-80, 20, 2000000)
    assert (split_hi(a) == a.astype(np.float32).astype(np.float64)).all()
    assert split_hi(np.float64(0.0)) == 0.0 and split_hi(np.float64(-0.0)) == 0.0


@pytest.mark.parametrize("ctas,M,N,unit", [(3, 3, 200, -1), (7, 3, 500, -1), (11, 5, 333, -1), (16, 5, 1000, -1), (5, 5, 64, -1),
                                           (6, 4, 700, 1), (9, 7, 130, 32)])
def test_share_arithmetic_covers_every_chunk_once(emu, ctas, M, N, unit):
    """The share rules of the persistent grid (contiguous shares in units of 1 / 32 chunks, shares that never cross a map)
    for CTA counts that do not divide the maps or the chunks: every (m, n) cost is written exactly once and equals the
    generic kernel's (the destination starts as -1; an unwritten or doubly-claimed chunk would show)."""
    win, gen = emu
    rng = np.random.default_rng(ctas * 100 + M)
    T, R, Cc = 6, 260, 250
    res = F32(0.1)
    lin = rng.integers(0, 101, (M, R, Cc)).astype(np.int8)
    ang = rng.integers(0, 101, (M, R, Cc)).astype(np.int8)
    obs = (rng.random((R, Cc)) < 0.02).astype(np.int8)
    unk = (rng.random((R, Cc)) < 0.02).astype(np.int8)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(F32)
    u_cur = np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(F32)
    x0, goal = [12.03, 12.97, 0.7], [20.0, 20.0]
    f = _fparams(res, 0.0, 0.0, 0.1, x0, goal, 0.5, 0.01, 1.0, [2, 3], [0, 3], [-np.pi, np.pi], 1e5, 1e2, 1.0, 0.0, 0.0)
    ratios = _ratios([0, 1], [0, 1])
    geo = _c([R, Cc, R, Cc, Cc, Cc, T, N, M], np.int32)
    out = np.full((N, M), -1.0, F32)
    assert win.emu_rollout_win(_p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), _p(noise), _p(u_cur), _p(out),
                               0, 0, None, None, ctas, 1, unit, 0, 1) == 0
    cnm, costs = np.zeros((N, M), F32), np.zeros(N, F32)
    gen.emu_rollout(0, _p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), None, _p(noise), _p(u_cur), _p(cnm),
                    _p(costs), None, 0)
    assert (out > 0).all()
    rel = np.abs(out - cnm) / np.maximum(np.abs(cnm), 1e-6)
    assert rel.max() < 2e-6, rel.max()


@pytest.mark.parametrize("res", [0.1, 0.05, 0.3, 1.0, 0.0625, 0.7])
def test_division_free_cell_decision_equals_reference_sequence(emu, res):
    """cell_from_interval (csrc/rollout_win.cu: floor(a / res) from the magic-number floors of the interval's ends, decided
    by the exact float64 product hi * res when the interval holds an integer) returns what the reference's exact sequence (cell_index_exact: three
    float32 divisions) returns -- on coordinates within a few float32 ulps of every kind of cell edge (both signs, indices
    up to 2^20 and beyond the guarded range), where the decision actually runs, and on random coordinates."""
    win, _ = emu
    rng = np.random.default_rng(int(res * 1e4))
    r32 = F32(res)
    k = np.concatenate([rng.integers(-2000, 20000, 300000), rng.integers(-(1 << 20), 1 << 20, 200000),
                        rng.integers(-(1 << 23), 1 << 23, 20000)])
    edge = (k.astype(np.float64) * np.float64(r32)).astype(F32)                       # the float32 nearest the edge k * res
    a = edge.copy()
    for _ in range(3):                                                                # ... and up to 3 ulps either side
        step = rng.integers(-1, 2, a.size)
        a = np.where(step > 0, np.nextafter(a, F32(np.inf)), np.where(step < 0, np.nextafter(a, F32(-np.inf)), a)).astype(F32)
    a = np.concatenate([a, edge, (rng.standard_normal(200000) * 300).astype(F32), np.zeros(4, F32)])
    a = np.ascontiguousarray(a, F32)
    new, ref, differ = np.zeros(a.size, np.int32), np.zeros(a.size, np.int32), np.zeros(a.size, np.int32)
    win.emu_cell_between(_p(a), a.size, float(r32), _p(new), _p(ref), _p(differ))
    assert differ.sum() > 10000                                                       # the decision ran often
    bad = np.nonzero(new != ref)[0]
    assert bad.size == 0, (a[bad[:5]], new[bad[:5]], ref[bad[:5]])
    # and inside the range where the division-free decision is used (|index| < 2^21) both are the true floor of the exact
    # quotient of the two float32 values (where float64 can tell); beyond 2^22 the reference's float32 sequence itself
    # departs from it, which is why the kernel runs that sequence there
    q = a.astype(np.float64) / np.float64(r32)
    clear = (np.abs(q - np.round(q)) > 1e-6) & (np.abs(q) < 2 ** 21 - 2)
    assert (ref[clear] == np.floor(q[clear])).all()
