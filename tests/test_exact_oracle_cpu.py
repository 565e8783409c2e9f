"""The exact oracle (oracle/arith.py: operations rounded where the kernels round them, approximate operations from a
provider) against the real kernel sources executed on the host (tests/emu_rollout.py, tests/emu_rollout_win.py) with
the libm provider -- what the emulation substitutes for the MUFU operations -- element for element, on the rare paths
a statistical comparison cannot see: traction bounds with a nonzero / negative lower end, starts on cell edges and
within an ulp of them far from the map origin, lookups outside the staged window and outside the map (on both sides), goals reached
at the first and at the last step, T = 1, N = 1, ragged chunks, mask bytes other than 0 / 1.  And the once-rounded FMA
helpers against exact rational arithmetic."""
import zlib
from fractions import Fraction

import numpy as np
import pytest

from oracle import arith as AR
from oracle import mppi_ref as MR
from tests.emu_rollout import build as build_generic
from tests.emu_rollout_win import build as build_win
from tests.test_rollout_emulated_cpu import _c, _fparams, _p, _ratios

F32, F64 = np.float32, np.float64
EXACT = AR.Exact(AR.LibmProvider())


# ----------------------------------------------------------------------------- FMA helpers vs Fraction
def _round_frac(fr, mant_bits, emin):
    """Exact rational -> nearest binary float with ``mant_bits`` significant bits, ties to even, subnormals down to
    2^(emin - mant_bits + 1) (no overflow in these tests)."""
    if fr == 0:
        return 0.0
    sign = -1 if fr < 0 else 1
    fr = abs(fr)
    e = fr.numerator.bit_length() - fr.denominator.bit_length()
    while Fraction(2) ** e > fr:
        e -= 1
    while Fraction(2) ** (e + 1) <= fr:
        e += 1
    q = max(e, emin) - (mant_bits - 1)                  # quantum of the result's binade
    m = round(fr / Fraction(2) ** q)                    # Fraction.__round__: ties to even
    return sign * float(m * Fraction(2) ** q)


def _want32(a, b, c, ftz=False):
    a, b, c = (AR.flush32(v) if ftz else F32(v) for v in (a, b, c))
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if exact == 0:                                      # IEEE: exact zero sum is +0 unless both addends are -0
        prod_neg = (np.signbit(a) != np.signbit(b)) and float(a) * float(b) == 0
        return F32(-0.0) if (prod_neg and np.signbit(c)) else F32(0.0)
    r = F32(_round_frac(exact, 24, -126))
    return AR.flush32(r)[()] if ftz else r


def _want64(a, b, c):
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if exact == 0:
        return 0.0
    return _round_frac(exact, 53, -1022)


def _same(x, y):
    return np.asarray(x).view(np.uint32 if np.asarray(x).dtype == F32 else np.uint64) == \
        np.asarray(y).view(np.uint32 if np.asarray(y).dtype == F32 else np.uint64)


def test_fma_helpers_round_once_like_exact_arithmetic():
    rng = np.random.default_rng(0)
    n = 3000
    a = (rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6, n)).astype(F32)
    b = (rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6, n)).astype(F32)
    c = (-(a.astype(F64) * b.astype(F64)) * (1 + rng.uniform(-1e-6, 1e-6, n))).astype(F32)   # heavy cancellation
    c[::3] = rng.standard_normal(n)[::3].astype(F32)
    got = AR.fma32_once(a, b, c)
    want = np.array([_want32(*t) for t in zip(a, b, c)], F32)
    assert _same(got, want).all()
    a64 = rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)
    b64 = rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)
    c64 = -(a64 * b64) * (1 + rng.uniform(-1e-12, 1e-12, n))
    got64 = AR.fma64_once(a64, b64, c64)
    assert _same(got64, np.array([_want64(*t) for t in zip(a64, b64, c64)])).all()


def test_fma_helpers_on_double_rounding_ties_zeros_and_ftz():
    """Constructed cases: a float32 product that is an exact float32 midpoint plus an addend below half a float64 ulp
    (rounding to float64 first lands on the tie and then rounds to even: wrong), an exact tie (to even), a float64
    product that needs 55 bits, signed zeros, and the .ftz flushes of inputs and results.  The default arithmetic
    (two roundings) fails some of them -- the cases are not vacuous."""
    k = F32(2 ** 12 + 1)                                  # k*k = 2^24 + 2^13 + 1: halfway between two float32
    cases32 = [(k, k, F32(2.0 ** -40)), (k, k, F32(-2.0 ** -40)), (k, k, F32(0)),
               (F32(-0.0), F32(1), F32(-0.0)), (F32(1), F32(-0.0), F32(0)), (F32(1), F32(1), F32(-1)),
               (F32(-0.0), F32(0), F32(-0.0)), (F32(3), F32(1e-45), F32(0)), (F32(1e-20), F32(1e-20), F32(0)),
               (F32(1e-40), F32(1e30), F32(0)), (F32(1.5), F32(-1e-39), F32(1e-39))]
    for ftz in (False, True):
        A = AR.Exact(AR.LibmProvider(), ftz=ftz)
        for t in cases32:
            got = A.fma32(np.array([t[0]]), np.array([t[1]]), np.array([t[2]]))[0]
            want = _want32(*t, ftz=ftz)
            assert _same(got, want), (t, ftz, got, want)
    assert AR.Exact(AR.LibmProvider(), ftz=True).fma32(F32(1e-40), F32(1e30), F32(0)) == 0          # input flushed
    assert AR.Exact(AR.LibmProvider(), ftz=False).fma32(F32(1e-40), F32(1e30), F32(0)) > 0
    assert AR.Exact(AR.LibmProvider(), ftz=True).fma32(F32(1e-20), F32(1e-20), F32(0)) == 0         # result flushed
    assert np.signbit(AR.Exact(AR.LibmProvider(), ftz=True).fma32(F32(-1e-20), F32(1e-20), F32(0)))
    kk = F64(2 ** 27 + 1)                                 # kk*kk = 2^54 + 2^28 + 1: 55 bits
    for t in [(kk, kk, F64(2)), (kk, kk, F64(1)), (kk, kk, -F64(1)), (F64(-0.0), F64(5), F64(-0.0))]:
        assert _same(AR.fma64_once(*t), F64(_want64(*t)) if _want64(*t) != 0 or not
                     (np.signbit(t[0]) and np.signbit(t[2])) else F64(-0.0)), t
    # the default arithmetic rounds twice: wrong on the first float32 case and the first float64 case
    assert not _same(MR._fma32(np.array([k]), np.array([k]), np.array([F32(2.0 ** -40)]))[0], _want32(k, k, F32(2.0 ** -40)))
    assert not _same(AR.NUMPY.fma64(kk, kk, F64(2)), F64(_want64(kk, kk, F64(2))))
    assert _same(AR.fma64_once(kk, kk, F64(2)), F64(_want64(kk, kk, F64(2))))


def test_ftz_conversions():
    A = AR.Exact(AR.LibmProvider(), ftz=True)
    sub = np.array([1e-40, -1e-40, 1.2e-38, 0.0], F32)
    assert (A.f2d(sub) == [0, 0, F64(F32(1.2e-38)), 0]).all() and np.signbit(A.f2d(sub)[1])
    assert A.d2f(np.array([1e-40]))[0] == 0 and A.d2f(np.array([2e-38]))[0] == F32(2e-38)
    B = AR.Exact(AR.LibmProvider(), ftz=False)
    assert B.f2d(sub)[0] == F64(F32(1e-40)) and B.d2f(np.array([1e-40]))[0] != 0


# ----------------------------------------------------------------------------- emulated kernels vs the exact oracle
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("emu_exact"))
    return build_win(d), build_generic(d)


def _scenario(name):
    """Inputs of one edge scenario (dict): maps, masks, noise, controls, geometry, bounds, goal."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    s = dict(N=300, M=2, T=30, R=300, Cc=280, res=F32(0.1), xlo=F32(0.0), ylo=F32(0.0), lb=[0, 1], ab=[0, 1],
             x0=[14.03, 15.07, 0.7], goal=[17.0, 18.0], tol=0.5, dt=0.1, shift=(0, 0), mask_lo=0, mask_hi=2)
    if name == "lo_pos":
        s.update(lb=[0.2, 0.9], ab=[0.15, 1.3])
    elif name == "lo_neg":
        s.update(lb=[-0.4, 1.0], ab=[-0.5, 0.8])
    elif name == "edge_start":                            # exactly on the lower edges of cell (151, 140)
        s.update(x0=[float(F32(140 * F32(0.1))), float(F32(151 * F32(0.1))), 0.0])
    elif name == "far_origin":                            # 4096 m origin, the robot within an ulp of a cell edge
        xlo = F32(4096.0)
        e = F32(xlo + F32(140 * 0.1))
        s.update(xlo=xlo, ylo=xlo, x0=[float(np.nextafter(e, F32(np.inf))), float(np.nextafter(F32(xlo + F32(15.0)), F32(0))), 1.1],
                 goal=[float(xlo) + 17.0, float(xlo) + 18.0])
    elif name == "outside":                               # window pushed off the robot, rollouts leaving the map
        s.update(R=260, Cc=250, x0=[23.4, 24.1, 0.8], goal=[60.0, 60.0], shift=(100, 90), T=40)
    elif name == "outside_neg":                           # leaving the map below its origin: negative cell indices
        s.update(R=260, Cc=250, x0=[2.3, 1.9, 3.9], goal=[-30.0, -30.0], T=40)
    elif name in ("goal_first", "goal_last"):
        s.update(T=25, tol=0.05)
    elif name == "t1_n1":
        s.update(N=1, T=1, M=3)
    elif name == "ragged":
        s.update(N=33, M=3)
    elif name == "mask_bytes":
        s.update(mask_lo=-128, mask_hi=128)
    N, M, T, R, Cc = s["N"], s["M"], s["T"], s["R"], s["Cc"]
    s["lin"] = rng.integers(0, 101, (M, R, Cc)).astype(np.int8)
    s["ang"] = rng.integers(0, 101, (M, R, Cc)).astype(np.int8)
    s["obs"] = (rng.random((R, Cc)) < 0.03).astype(np.int8) * rng.integers(s["mask_lo"], s["mask_hi"], (R, Cc)).astype(np.int8)
    s["unk"] = (rng.random((R, Cc)) < 0.03).astype(np.int8) * rng.integers(s["mask_lo"], s["mask_hi"], (R, Cc)).astype(np.int8)
    s["risk"] = rng.integers(0, 101, (R, Cc)).astype(np.int8)
    s["noise"] = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(F32)
    s["u_cur"] = np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(F32)
    if name == "edge_start":
        s["noise"][: N // 2] = 0                          # half the rollouts stand still on the edge
        s["u_cur"][:] = 0
        s["lin"][:, :, :] = np.maximum(s["lin"], 1)
    if name in ("outside", "outside_neg"):
        s["u_cur"][:, 0] = 3.0
        s["noise"][..., 0] = np.abs(s["noise"][..., 0]) + 5.0   # clipped to vmax: straight out of the 25 m map
    if name in ("goal_first", "goal_last"):
        # rollout 0 without noise on uniform maps: the goal sits where its step 0 / step T-1 ends (oracle states), so it
        # is reached exactly then, on every map
        s["noise"][:1] = 0
        s["u_cur"][:, 0] = 2.0
        s["lin"][:] = 100
        s["ang"][:] = 100
        _, st = MR.rollout_costs(MR.MODE_STOCHASTIC, s["lin"], s["ang"], s["lb"], s["ab"], s["obs"], s["unk"], s["res"],
                                 [s["xlo"], 0], [s["ylo"], 0], [0, 3], [-np.pi, np.pi], [1e9, 1e9], 0.01, 1e5, 1e2,
                                 0.0, 1.0, [2, 3], s["x0"], 0.1, 1.0, s["noise"][:1], s["u_cur"], return_states=True,
                                 arith=EXACT, wrap_clamp=True)
        k = 1 if name == "goal_first" else T
        s["goal"] = [float(st[0, 0, k, 0]), float(st[0, 0, k, 1])]
    return s


def _run_all(emu, s, masks01=None):
    win, gen = emu
    N, M, T, R, Cc = s["N"], s["M"], s["T"], s["R"], s["Cc"]
    f = _fparams(s["res"], s["xlo"], s["ylo"], s["dt"], s["x0"], s["goal"], s["tol"], 0.01, 1.0, [2, 3], [0, 3],
                 [-np.pi, np.pi], 1e5, 1e2, 1.0, s["lb"][0], s["ab"][0])
    ratios = _ratios(s["lb"], s["ab"])
    geo = _c([R, Cc, R, Cc, Cc, Cc, T, N, M], np.int32)
    args = [_c(s[k], np.int8) for k in ("lin", "ang", "obs", "unk")]
    noise, u_cur = _c(s["noise"], F32), _c(s["u_cur"], F32)
    m01 = int(((s["obs"] & ~1) == 0).all() and ((s["unk"] & ~1) == 0).all()) if masks01 is None else masks01
    out = np.zeros((N, M), F32)
    assert win.emu_rollout_win(_p(f), _p(geo), _p(ratios), *[_p(a) for a in args], _p(noise), _p(u_cur), _p(out),
                               s["shift"][0], s["shift"][1], None, None, 0, 1, 0, 0, m01) == 0
    gens = {}
    for mode in (0, 1, 2):
        cnm, costs = np.zeros((N, M if mode == 0 else 1), F32), np.zeros(N, F32)
        gen.emu_rollout(mode, _p(f), _p(_c([R, Cc, R, Cc, Cc, Cc, T, N, M if mode == 0 else 1], np.int32)), _p(ratios),
                        *[_p(a) for a in args], _p(_c(s["risk"], np.int8)), _p(noise), _p(u_cur), _p(cnm), _p(costs), None, 0)
        gens[mode] = cnm if mode == 0 else costs[:, None]
    return out, gens


def _oracle(s, mode, order="sequential"):
    return MR.rollout_costs(mode, s["lin"], s["ang"], s["lb"], s["ab"], s["obs"], s["unk"], s["res"],
                            [s["xlo"], 0], [s["ylo"], 0], [0, 3], [-np.pi, np.pi], s["goal"], 0.01, 1e5, 1e2, s["tol"],
                            1.0, [2, 3], s["x0"], s["dt"], 1.0, s["noise"], s["u_cur"], risk_map=s["risk"][None],
                            wrap_clamp=True, arith=EXACT, ctrl_order=order)


def assert_equal(got, want, what):
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, "%s: %d of %d differ; first (n, m, got, want): %s" % (
        what, len(bad), got.size, [(int(n), int(m), float(got[n, m]), float(want[n, m])) for n, m in bad[:5]])


SCENARIOS = ["lo_pos", "lo_neg", "edge_start", "far_origin", "outside", "outside_neg", "goal_first", "goal_last", "t1_n1", "ragged",
             "mask_bytes"]


@pytest.mark.parametrize("name", SCENARIOS)
def test_emulated_kernels_equal_exact_oracle_on_edge_scenarios(emu, name):
    s = _scenario(name)
    out, gens = _run_all(emu, s)
    assert_equal(out, _oracle(s, MR.MODE_STOCHASTIC, "presummed"), "windowed kernel")
    assert_equal(gens[0], _oracle(s, MR.MODE_STOCHASTIC), "generic kernel, mode 0")
    assert_equal(gens[1], _oracle(s, MR.MODE_DET_DYN), "generic kernel, mode 1")
    assert_equal(gens[2], _oracle(s, MR.MODE_SPEED_MAP), "generic kernel, mode 2")
    if name == "mask_bytes":
        assert (s["obs"] < 0).any() and (s["obs"] > 1).any()
    if name in ("goal_first", "goal_last"):
        # rollout 0 reaches the goal exactly at its first / last step (the stage cost of that step, no terminal cost)
        _, st = MR.rollout_costs(MR.MODE_STOCHASTIC, s["lin"], s["ang"], s["lb"], s["ab"], s["obs"], s["unk"], s["res"],
                                 [s["xlo"], 0], [s["ylo"], 0], [0, 3], [-np.pi, np.pi], s["goal"], 0.01, 1e5, 1e2,
                                 s["tol"], 1.0, [2, 3], s["x0"], 0.1, 1.0, s["noise"][:1], s["u_cur"],
                                 return_states=True, arith=EXACT, wrap_clamp=True)
        d = np.hypot(st[0, :, 1:, 0] - s["goal"][0], st[0, :, 1:, 1] - s["goal"][1])
        k = 0 if name == "goal_first" else s["T"] - 1
        assert (d[:, k] == 0).all() and (d[:, :k] > s["tol"]).all()
    if name in ("outside", "outside_neg"):
        _, st = MR.rollout_costs(MR.MODE_STOCHASTIC, s["lin"], s["ang"], s["lb"], s["ab"], s["obs"], s["unk"], s["res"],
                                 [s["xlo"], 0], [s["ylo"], 0], [0, 3], [-np.pi, np.pi], s["goal"], 0.01, 1e5, 1e2,
                                 s["tol"], 1.0, [2, 3], s["x0"], 0.1, 1.0, s["noise"], s["u_cur"], return_states=True,
                                 arith=EXACT, wrap_clamp=True)
        if name == "outside":
            assert (st[..., 0] > s["Cc"] * 0.1).any() and (st[..., 1] > s["R"] * 0.1).any()     # left the map
        else:
            assert (st[..., 0] < 0).any() and (st[..., 1] < 0).any()


@pytest.mark.parametrize("name", ["lo_pos", "lo_neg", "far_origin"])
def test_state_rollout_and_barebone_kernels_equal_exact_oracle(emu, name):
    _, gen = emu
    s = _scenario(name)
    T, R, Cc = s["T"], s["R"], s["Cc"]
    V = 5
    f = _fparams(s["res"], s["xlo"], s["ylo"], 0.1, s["x0"], [0, 0], 0.0, 1.0, 1.0, [1, 1], [0, 3], [-np.pi, np.pi],
                 0.0, 0.0, 1.0, s["lb"][0], s["ab"][0])
    u_prev = _c(s["u_cur"][::-1], F32)
    for mode in (0, 1):
        out = np.zeros((V, T + 1, 3), F32)
        gen.emu_state_rollout(mode, V, _p(f), _p(_c([R, Cc, R, Cc, Cc, Cc, T, s["N"], s["M"]], np.int32)),
                              _p(_ratios(s["lb"], s["ab"])), _p(_c(s["lin"], np.int8)), _p(_c(s["ang"], np.int8)),
                              _p(_c(s["noise"], F32)), _p(_c(s["u_cur"], F32)), _p(u_prev), _p(out))
        want = MR.state_rollouts(MR.MODE_STOCHASTIC if mode == 0 else MR.MODE_DET_DYN, V if mode else min(V, s["M"]),
                                 s["lin"], s["ang"], s["lb"], s["ab"], s["res"], [s["xlo"], 0], [s["ylo"], 0], s["x0"],
                                 0.1, s["u_cur"], u_prev, s["noise"], [0, 3], [-np.pi, np.pi], arith=EXACT)
        k = want.shape[0]
        assert (out[:k].view(np.uint32) == want.view(np.uint32)).all(), (mode, int((out[:k] != want).sum()))
    # barebone: obstacles around the path, one of them containing the start
    obs_pos = np.array([[s["x0"][0], s["x0"][1]], [s["x0"][0] + 1.0, s["x0"][1] + 0.5], [s["goal"][0], s["goal"][1]]], F32)
    obs_r = np.array([0.3, 0.7, 0.4], F32)
    fb = _fparams(1.0, 0.0, 0.0, 0.1, s["x0"], s["goal"], 0.5, 0.0, 1.0, [2, 3], [0, 3], [-np.pi, np.pi], 1e3, 0.0, 1.0,
                  0.0, 0.0)
    ob = _c(np.concatenate([obs_pos, obs_r[:, None]], axis=1), F32)
    costs = np.zeros(s["N"], F32)
    gen.emu_rollout(3, _p(fb), _p(_c([1, 1, 1, 1, 1, 1, T, s["N"], 1], np.int32)), _p(_c([0.01, 0.01], np.float64)),
                    None, None, None, None, None, _p(_c(s["noise"], F32)), _p(_c(s["u_cur"], F32)), None, _p(costs),
                    _p(ob), 3)
    want = MR.rollout_costs_barebone(obs_pos, obs_r, [0, 3], [-np.pi, np.pi], s["goal"], 1e3, 0.5, 1.0, [2, 3], s["x0"],
                                     0.1, 1.0, s["noise"], s["u_cur"], arith=EXACT)
    assert_equal(costs[:, None], want[:, None], "barebone kernel")


# ----------------------------------------------------------------------------- directed: the float64 contractions
@pytest.mark.parametrize("kind", ["state", "traction", "speed"])
def test_float64_contractions_on_a_float32_rounding_boundary(emu, kind):
    """The traction value fma(ratio, q, lo) and the state update fma(dv, cos, x), each rounded once: on inputs where
    rounding the product first moves the first step's float32 x by one ulp and flips the goal flag, every kernel
    equals the exact oracle -- so a kernel (or an oracle) that split either contraction would differ here.  Kind
    "speed": the speed map's eff = fma(ratio, risk, lo), on inputs where splitting it moves the time step dt / (eff +
    1e-6), the whole cost of a one-step rollout that starts on its goal, by one float32 ulp."""
    from tests.directed_cases import boundary_case, directed_scenario
    case = boundary_case(EXACT, kind)
    s = directed_scenario(case)
    _, st = MR.rollout_costs(MR.MODE_STOCHASTIC, s["lin"], s["ang"], s["lb"], s["ab"], s["obs"], s["unk"], s["res"],
                             [s["xlo"], 0], [s["ylo"], 0], [0, 3], [-np.pi, np.pi], s["goal"], 0.01, 1e5, 1e2, s["tol"],
                             1.0, [2, 3], s["x0"], s["dt"], 1.0, s["noise"], s["u_cur"], return_states=True, arith=EXACT)
    assert (st[:, :, 1, 0] == case["x1_exact"]).all()
    if kind == "speed":
        assert s["T"] == 1 and case["risk"] != case["q"] and case["cost_exact"] != case["cost_other"]
        assert (_oracle(s, MR.MODE_SPEED_MAP) == case["cost_exact"]).all()
    else:
        assert case["x1_exact"] != case["x1_other"]
        assert (st[:, :, 2, 0] == 0).all() == case["exact_reaches"]      # reached at the first step: no second step ran
    out, gens = _run_all(emu, s)
    assert_equal(out, _oracle(s, MR.MODE_STOCHASTIC, "presummed"), "windowed kernel")
    for mode in (0, 1, 2):
        assert_equal(gens[mode], _oracle(s, mode), "generic kernel, mode %d" % mode)
    if kind == "speed":
        assert (gens[2] == case["cost_exact"]).all()
    _, gen = emu
    f = _fparams(s["res"], s["xlo"], s["ylo"], s["dt"], s["x0"], [0, 0], 0.0, 1.0, 1.0, [1, 1], [0, 3],
                 [-np.pi, np.pi], 0.0, 0.0, 1.0, s["lb"][0], s["ab"][0])
    vis = np.zeros((1, s["T"] + 1, 3), F32)
    gen.emu_state_rollout(1, 1, _p(f), _p(_c([100, 100, 100, 100, 100, 100, s["T"], s["N"], 1], np.int32)),
                          _p(_ratios(s["lb"], s["ab"])), _p(_c(s["lin"], np.int8)), _p(_c(s["ang"], np.int8)),
                          _p(s["noise"]), _p(s["u_cur"]), _p(s["u_cur"]), _p(vis))
    assert vis[0, 1, 0] == case["x1_exact"]
