"""High-precision references of the CVaR and control-update reductions, and per-element error bounds for the
kernels that compute them (TEST INFRASTRUCTURE).

The references do not restate any kernel's summation order: a kernel's result is accepted when it lies within a
bound derived from the SHAPE of its reduction (chain lengths and tree depths), so a kernel that selects the wrong
elements, drops or repeats a term, or mis-scales a partial fails, whatever order it sums in.

Notation: u = 2^-24 (float32 unit roundoff), TINY = 2^-126 (the smallest normal float32), and
gamma(d) = d*u / (1 - d*u).  A float32 sum whose every term passes through at most d roundings (round to nearest)
differs from the exact sum by at most gamma(d) * sum|terms| (Higham, Accuracy and Stability of Numerical Algorithms,
Lemma 3.1 / eq. 4.4).  The kernels are built with -ftz: a result below TINY is flushed to zero, so each operation may
also add an absolute error of TINY; the bounds carry that term.

CVaR (cvar_kernel / cvar_batch_kernel, cvar_large_kernel, csrc/rollout.cu)
---------------------------------------------------------------------------
numel = ceil(float64(M) * float64(float32(alpha))), clamped to [1, M] -- the reference passes alpha as np.float32
and Numba multiplies the int block width by it in float64.  mu = the exact mean of the numel largest values of the
row (ties resolved by value: which of several equal values is chosen does not change mu).  The kernels sum the
values strictly above the numel-th largest, then add (numel - greater) * threshold:
  * warp kernel: each lane adds its <= PER values (PER = the template parameter, the power of two >= ceil(M/32)),
    then 5 butterfly levels; the threshold product is rounded once and added once:  d = PER + 5 + 2;
  * CTA kernel: each thread adds its <= ceil(M/256) values, 5 butterfly levels, then thread 0 adds the 8 warp sums
    in sequence, then the product and its add:  d = ceil(M/256) + 5 + 8 + 2;
  * a pairwise tree (the numpy oracle's cvar_reduce and the reference's own kernel): d = ceil(log2(numel)).
The mean is (float)((double)sum / numel): the float64 quotient is within 2^-53 relative of sum / numel, its float32
rounding within half an ulp, so
    |y - mu| <= gamma(d) * sum_top|v| / numel + d * TINY / numel + (1/2 + 2^-28) * ulp32(|mu| + E_sum),
where E_sum is the first two terms (the ulp is taken at the largest value the quotient can have).  A top set that
contains +inf has mu = +inf and the kernel must return +inf exactly.

Update (update_partial_kernel / update_apply_kernel / merge_partials, csrc/reduce.cu, and the host combine)
------------------------------------------------------------------------------------------------------------
Reference: beta = min(c); d_n = f32(c_n - beta) (the reference's own float32 subtraction); a_n = exp(-d_n / lambda),
A = fsum(a); w_n = a_n / A; u_j = clip(u0_j + fsum_n(w_n * eps_nj)) in float64 (clipping is exact).  A rollout of
cost +inf has a_n = 0.

The kernels split the exponent: a rollout's weight is w_raw_n = f32(exp(-f32(c_n - beta_c)/lambda)) against its
CTA's minimum beta_c, multiplied (through the partials) by the merge scale f32(exp(-f32(beta_c - beta')/lambda)) of
each further level (CTA -> rank partial -> merged ranks: L = 2 scale roundings on one rank, 3 when rank partials are
merged as well).  Per rollout:
  * exponent: the float32 differences along the split sum to c_n - beta and each errs by at most u times itself
    (or TINY when flushed); with the reference's own f32(c_n - beta) the exponent differs by at most
    Delta_n = (2u * d_n / (1 - u) + (L + 1) * TINY) / lambda, plus 2^-48 * (x_n + 1) for the float64 exp and
    products (x_n = d_n / lambda);
  * the L float32 roundings of w_raw and the scales: relative (1 +- u)^L, absolute (L + 1) * TINY (each factor is
    <= 1, a flushed or subnormal factor errs by less than TINY).
So the product p_n of the rounded factors lies in [p_lo_n, p_hi_n] with
    p_hi_n = exp(-(x_n - Delta_n)) * (1 + u)^L + (L + 1) * TINY,  p_lo_n = max(0, exp(-(x_n + Delta_n)) * (1 - u)^L - (L + 1) * TINY),
and D_n = max(p_hi_n - a_n, a_n - p_lo_n).  A +inf cost gives w_raw = 0 exactly (exp(-inf) = 0, and a slab whose
every cost is +inf is given w_raw = 0, S = 0, V = 0), so D_n = 0 there.

W: S per CTA adds rows_per_cta non-negative terms in sequence; each merge level adds <= 2 strided FMAs per thread
(count <= 512 partials over 256 threads), 5 butterfly levels and 8 sequential adds: chain 15.  All terms are
non-negative, so W_hat lies in [sum(p_lo) (1 - gW) - opsW * TINY, sum(p_hi) (1 + gW) + opsW * TINY] with
1 + gW = (1 + gamma(rows_per_cta)) * prod over merge levels (1 + gamma(15)).

V_j: rows_per_cta FMAs per CTA, then num_ctas FMAs in the CTA merge, then `count` FMAs per further merge:
    |V_hat_j - sum_n a_n eps_nj| <= gV * sum_n p_hi_n |eps_nj| + sum_n D_n |eps_nj| + opsV * TINY,
with 1 + gV = prod over the chains (1 + gamma(len)).  Then q = f32(V_hat / W_hat) and u = f32(u0 + q):
    |q_tilde - V/A| <= E_V / W_lo + A * S1_j * max|1/W_hat - 1/A|,   S1_j = sum_n w_n |eps_nj|,
    |u_kernel - u_ref| <= that + u * |q| + TINY + u * (|u0| + |q|) + 2^-48 * (S1_j + |u0_j|)   (the last term covers
the reference's own float64 roundings).  Clipping does not increase the difference.  The bound scales with
S1_j = sum w_n |eps_nj|, not with |sum w_n eps_nj|, so noise whose weighted sum cancels is covered.

Weights: weight_n = f32(w_raw_n * f32(scale / W_hat)) with the CTA's scale relative to the global minimum
(L = 2 roundings of factors in every path), so
    weight_n in [p_lo_n / W_hi * (1 - u)^2 - 2 TINY, p_hi_n / W_lo * (1 + u)^2 + 2 TINY],
a relative bound around w_n plus the absolute subnormal term.

Every cost +inf: the reference has no weights to normalise (A = 0, its own result is NaN).  The kernels take a zero
step: u = clip(u0) exactly and every weight exactly 0.
"""
import math
from fractions import Fraction

import numpy as np

F32, F64 = np.float32, np.float64
U = 2.0 ** -24
TINY = 2.0 ** -126
# a computed float64 bound is inflated by this factor before it is compared: it is itself rounded
SLACK = 1.0 + 2.0 ** -40


def gamma(d):
    return d * U / (1.0 - d * U)


def ulp32(x):
    """ulp of a float32 of magnitude x (x >= 0, finite): 2^(e-23) for x in [2^e, 2^(e+1)), 2^-149 below TINY."""
    if x < TINY:
        return 2.0 ** -149
    m, e = math.frexp(x)             # x = m * 2^e, m in [0.5, 1)
    return 2.0 ** (e - 24)


# ----------------------------------------------------------------------------- CVaR
def cvar_numel(M, alpha):
    """numel as the reference computes it (mppi.py:744): ceil(int * float32 alpha) in float64, clamped to [1, M]."""
    n = int(math.ceil(float(M) * float(F32(alpha))))
    return min(max(n, 1), M)


def cvar_per(M):
    """PER template of the warp kernel (launch_cvar): the power of two >= ceil(M / 32)."""
    per = (M + 31) // 32
    p = 1
    while p < per:
        p *= 2
    return p


def cvar_depth(M, numel, kind):
    if kind == "warp":
        return cvar_per(M) + 5 + 2
    if kind == "cta":
        return -(-M // 256) + 5 + 8 + 2
    if kind == "tree":
        return max(0, math.ceil(math.log2(numel))) if numel > 1 else 0
    raise ValueError(kind)


def kernel_kind(M):
    return "warp" if M <= 1024 else "cta"


def _exact_sum(vals):
    """Exact sum of finite float32 values as a Fraction (every float32 is an integer multiple of 2^-149)."""
    scaled = np.asarray(vals, dtype=F64) * 2.0 ** 149          # exact: a float32 significand fits a float64
    return Fraction(sum(int(x) for x in scaled), 1 << 149)


def cvar_exact(costs_nm, alpha):
    """Per row: (mu, sum_top|v|, numel), mu the exact mean of the numel largest values (a Fraction, or +inf)."""
    c = np.asarray(costs_nm, dtype=F32)
    numel = cvar_numel(c.shape[1], alpha)
    out = []
    for row in c:
        top = np.sort(row)[::-1][:numel]
        if np.isposinf(top).any():
            out.append((math.inf, math.inf, numel))
            continue
        mu = _exact_sum(top) / numel
        out.append((mu, math.fsum(np.abs(top.astype(F64))) * SLACK, numel))
    return out


def cvar_bound(M, numel, abs_sum, mu, kind):
    d = cvar_depth(M, numel, kind)
    e_sum = (gamma(d) * abs_sum + d * TINY) / numel
    return (e_sum + (0.5 + 2.0 ** -28) * ulp32(abs(float(mu)) + e_sum)) * SLACK


def check_cvar(got, costs_nm, alpha, kind=None, extra_kind=None, label=""):
    """Assert every got[n] is within the bound of the exact CVaR of row n; `kind` the kernel's reduction ("warp",
    "cta", "tree"; default: the one launch_cvar picks for M); `extra_kind`: add a second reduction's bound (two
    computed results compared with each other).  Returns the largest |error| / bound."""
    c = np.asarray(costs_nm, dtype=F32)
    M = c.shape[1]
    kind = kind or kernel_kind(M)
    got = np.asarray(got, dtype=F32)
    worst = 0.0
    for n, (mu, abs_sum, numel) in enumerate(cvar_exact(c, alpha)):
        y = got[n]
        if mu == math.inf:
            assert y == np.inf, "%s row %d: CVaR of a top set with +inf is %r, want +inf" % (label, n, y)
            continue
        assert np.isfinite(y), "%s row %d: CVaR %r, want %r" % (label, n, y, float(mu))
        b = cvar_bound(M, numel, abs_sum, mu, kind)
        if extra_kind:
            b += cvar_bound(M, numel, abs_sum, mu, extra_kind)
        err = abs(Fraction(float(y)) - mu)
        assert err <= Fraction(b), "%s row %d (M %d numel %d): CVaR %r, exact %r, |error| %.3e > bound %.3e" % (
            label, n, M, numel, float(y), float(mu), float(err), b)
        if b > 0:
            worst = max(worst, float(err) / b)
    return worst


# ----------------------------------------------------------------------------- update
def num_ctas_rows(N):
    """The planner's CTA partition of N rollouts (update_num_ctas + api.cu): (num_ctas, rows_per_cta)."""
    ctas = min(max((N + 31) // 32, 1), 296)
    rpc = (N + ctas - 1) // ctas
    return (N + rpc - 1) // rpc, rpc


def update_reference(costs, noise, u0, lam, vrange, wrange):
    """(u (T, 2) float64, weights (N,) float64, ctx): the update in float64 with math.fsum sums."""
    c = np.asarray(costs, dtype=F32)
    eps = np.asarray(noise, dtype=F32).reshape(c.shape[0], -1).astype(F64)        # (N, 2T), column j = (t, k)
    beta = c.min()
    with np.errstate(invalid="ignore"):
        d = (c - beta).astype(F32).astype(F64)
    x = d / float(F32(lam))
    a = np.exp(-x)
    A = math.fsum(a)
    w = a / A
    prod = w[:, None] * eps
    V = np.array([math.fsum(prod[:, j]) for j in range(eps.shape[1])])
    u0f = np.asarray(u0, dtype=F32).reshape(-1).astype(F64)
    un = u0f + V
    lo = np.tile([float(F32(vrange[0])), float(F32(wrange[0]))], eps.shape[1] // 2)
    hi = np.tile([float(F32(vrange[1])), float(F32(wrange[1]))], eps.shape[1] // 2)
    u = np.minimum(hi, np.maximum(lo, un))
    ctx = dict(d=d, x=x, a=a, A=A, w=w, eps=eps, u0=u0f, inf=np.isposinf(c), lam=float(F32(lam)))
    return u.reshape(-1, 2), w, ctx


def _p_range(ctx, L):
    d, x, a, inf = ctx["d"], ctx["x"], ctx["a"], ctx["inf"]
    lam = ctx["lam"]
    fin = ~inf
    delta = np.zeros_like(x)
    delta[fin] = (2 * U * d[fin] / (1 - U) + (L + 1) * TINY) / lam + 2.0 ** -48 * (x[fin] + 1)
    p_hi = np.zeros_like(x)
    p_lo = np.zeros_like(x)
    p_hi[fin] = np.exp(-(x[fin] - delta[fin])) * (1 + U) ** L + (L + 1) * TINY
    p_lo[fin] = np.maximum(0.0, np.exp(-(x[fin] + delta[fin])) * (1 - U) ** L - (L + 1) * TINY)
    D = np.maximum(p_hi - a, a - p_lo)
    D[inf] = 0.0
    return p_lo, p_hi, D


def update_bounds(ctx, N, merges=1):
    """Per-element bounds (on u (T, 2), on weights (N,)) for the kernels' update of N rollouts on one rank
    (merges=1: CTA partials -> one partial, merged once more with itself by the apply step), or over `merges`
    gathered rank partials with N the rollouts of each rank (the sharded path: a third scale rounding)."""
    num_ctas, rpc = num_ctas_rows(N)
    L = 2 if merges == 1 else 3
    p_lo, p_hi, D = _p_range(ctx, L)
    A, eps, w, u0 = ctx["A"], ctx["eps"], ctx["w"], ctx["u0"]
    levels = 2                                          # CTA merge, then the apply step's merge of the partial(s)
    gW = (1 + gamma(rpc)) * (1 + gamma(15)) ** levels - 1
    opsW = len(D) + levels * 16 * 512
    W_hi = (math.fsum(p_hi) * (1 + gW) + opsW * TINY) * SLACK
    W_lo = max((math.fsum(p_lo) * (1 - gW) - opsW * TINY) / SLACK, 0.0)
    assert W_lo > 0, "the bound needs W > 0"
    inv_dev = max(abs(1 / W_lo - 1 / A), abs(1 / W_hi - 1 / A))
    gV = (1 + gamma(rpc)) * (1 + gamma(num_ctas * merges)) * (1 + gamma(merges)) - 1
    opsV = len(D) + num_ctas * merges + merges + 2
    ae = np.abs(eps)
    S_hi = (p_hi @ ae) * SLACK
    E_V = gV * S_hi + (D @ ae) * SLACK + opsV * TINY
    S1 = (w @ ae) * SLACK
    e_q = E_V / W_lo + A * S1 * inv_dev
    q_max = S1 + e_q
    e_u = e_q + U * q_max + TINY + U * (np.abs(u0) + q_max) + TINY + 2.0 ** -48 * (S1 + np.abs(u0))
    # weights: two factor roundings (w_raw, the CTA's scale against the global minimum), the division and the product
    q_lo, q_hi, _ = _p_range(ctx, 2)
    wt_hi = q_hi / W_lo * (1 + U) ** 2 + 2 * TINY
    wt_lo = np.maximum(q_lo / W_hi * (1 - U) ** 2 - 2 * TINY, 0.0)
    e_w = np.maximum(wt_hi - w, w - wt_lo) * SLACK + 2.0 ** -48 * w
    e_w[ctx["inf"]] = 0.0
    return (e_u * SLACK).reshape(-1, 2), e_w


def check_update(u, weights, costs, noise, u0, lam, vrange, wrange, N=None, merges=1, label=""):
    """Assert the kernels' u (T, 2) and weights (N,) lie within the bounds of the float64 reference; a +inf cost must
    get weight exactly 0 and no weight may be NaN.  N: rollouts per rank (default: all).  Returns the largest
    |error| / bound of u and of the weights.  When every cost is +inf: u == clip(u0) and every weight 0, exactly."""
    if np.isposinf(np.asarray(costs, dtype=F32)).all():
        want = np.asarray(u0, dtype=F32).copy()
        want[:, 0] = np.maximum(F32(vrange[0]), np.minimum(F32(vrange[1]), want[:, 0]))
        want[:, 1] = np.maximum(F32(wrange[0]), np.minimum(F32(wrange[1]), want[:, 1]))
        u = np.asarray(u, dtype=F32)
        bad = np.argwhere(u != want)
        assert bad.size == 0, "%s: every cost +inf, u%s = %r, want clip(u0) = %r (%d elements differ)" % (
            label, tuple(bad[0]), u[tuple(bad[0])], want[tuple(bad[0])], len(bad))
        if weights is not None:
            wt = np.asarray(weights, dtype=F32)
            assert (wt == 0).all(), "%s: every cost +inf, %d weights are not 0 (first %r)" % (
                label, int((wt != 0).sum()), wt[wt != 0][:3].tolist())
        return 0.0, 0.0
    want_u, want_w, ctx = update_reference(costs, noise, u0, lam, vrange, wrange)
    eu, ew = update_bounds(ctx, len(want_w) if N is None else N, merges)
    u = np.asarray(u, dtype=F32).astype(F64)
    assert np.isfinite(u).all(), "%s: u has non-finite values at %s" % (label, np.argwhere(~np.isfinite(u))[:4].tolist())
    err_u = np.abs(u - want_u)
    bad = np.argwhere(err_u > eu)
    assert bad.size == 0, "%s: u%s = %r, reference %r, |error| %.3e > bound %.3e (%d elements out)" % (
        label, tuple(bad[0]), u[tuple(bad[0])], want_u[tuple(bad[0])], err_u[tuple(bad[0])], eu[tuple(bad[0])], len(bad))
    ratio_u = float((err_u / np.maximum(eu, 1e-300)).max())
    ratio_w = 0.0
    if weights is not None:
        wt = np.asarray(weights, dtype=F32).astype(F64)
        assert not np.isnan(wt).any(), "%s: %d weights are NaN" % (label, int(np.isnan(wt).sum()))
        assert (wt[ctx["inf"]] == 0).all(), "%s: a rollout of cost +inf has a nonzero weight" % label
        err_w = np.abs(wt - want_w)
        bad = np.argwhere(err_w > ew)
        assert bad.size == 0, "%s: weight %d = %r, reference %r, |error| %.3e > bound %.3e (%d out)" % (
            label, bad[0][0], wt[bad[0][0]], want_w[bad[0][0]], err_w[bad[0][0]], ew[bad[0][0]], len(bad))
        ratio_w = float((err_w / np.maximum(ew, 1e-300)).max())
    return ratio_u, ratio_w


def update_inputs(kind, N, T, seed, lam=1.0):
    """(costs, noise, u0) for the value cases of the update tests, vrange [0, 3], wrange [-pi, pi]."""
    rng = np.random.default_rng(seed)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(F32)
    u0 = np.stack([rng.uniform(0, 2.9, T), rng.uniform(-3, 3, T)], 1).astype(F32)
    if kind == "mild":
        costs = rng.uniform(900, 930, N)
    elif kind == "underflow":
        # slab minima 0, 40, 95 and 130 lambda above the global one: merge scales exp(-95) (subnormal in float32) and
        # exp(-130) (0); within a slab a 105-lambda spread gives subnormal w_raw (exp(-87.3) .. exp(-103.3))
        _, rpc = num_ctas_rows(N)
        base = np.array([0.0, 95.0, 130.0, 40.0])[(np.arange(N) // rpc) % 4]
        costs = (base + rng.uniform(0, 105, N)) * lam
        costs[0] = 0.0
    elif kind == "far":
        # costs near 1e6 with a small global minimum: beta_c - beta is not exact in float32
        costs = 1e6 + rng.uniform(-30 * lam, 30 * lam, N)
        costs[N // 3] = 0.125
    elif kind == "signed":
        costs = rng.uniform(-5 * lam, 5 * lam, N)                                   # negative and zero-crossing
        costs[::7] = 0.0
    elif kind == "inf":
        costs = rng.uniform(900, 900 + 20 * lam, N)
        costs[rng.choice(N, max(1, N // 9), replace=False)] = np.inf                 # scattered +inf
        costs[N // 2] = 900.0
    elif kind == "clip":
        costs = rng.uniform(100, 100 + 3 * lam, N)
        u0[:, 0] = np.where(np.arange(T) % 2, 3.0, np.nextafter(F32(3.0), F32(0)))   # on / just inside the bounds
        u0[:, 1] = np.where(np.arange(T) % 2, -np.pi, np.nextafter(F32(np.pi), F32(0))).astype(F32)
    elif kind == "cancel":
        # noise whose weighted sum cancels: rollouts come in +eps / -eps pairs of (nearly) equal weight
        costs = np.repeat(rng.uniform(50, 50 + 2 * lam, (N + 1) // 2), 2)[:N]
        half = noise[: (N + 1) // 2]
        noise = np.repeat(half, 2, axis=0)[:N].copy()
        noise[1::2] *= -1
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(costs, dtype=F32), np.ascontiguousarray(noise), np.ascontiguousarray(u0)


def inf_slab_costs(N, seed=5):
    """Costs uniform in [900, 930] with the whole slab of CTA 2 (rows 2 * rows_per_cta .. 3 * rows_per_cta - 1) at +inf."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(900, 930, N).astype(F32)
    _, rpc = num_ctas_rows(N)
    c[2 * rpc: 3 * rpc] = np.inf
    return c


# ----------------------------------------------------------------------------- CVaR inputs
def cvar_rows(M, numel, seed):
    """A (rows, M) float32 matrix of the CVaR value cases for one (M, numel)."""
    rng = np.random.default_rng(seed)
    rows = []
    # the numel-th and (numel+1)-th values far apart: one element too many or too few moves the mean by >> bound
    base = rng.uniform(1.0, 2.0, M)
    order = rng.permutation(M)
    r = np.empty(M)
    r[order[:numel]] = base[:numel] + 1000.0
    r[order[numel:]] = base[numel:] - 1000.0
    rows.append(r)
    # ties at the threshold with multiplicity 2 .. M
    for mult in sorted({2, 3, max(2, M // 2), M}):
        if mult > M:
            continue
        r = rng.normal(0, 100, M)
        pos = rng.permutation(M)
        thr = 7.25
        above = max(0, numel - 1 - (mult - 1) // 2)               # the tie straddles the numel-th position
        above = min(above, M - mult)
        r[pos[:above]] = thr + rng.uniform(1, 50, above)
        r[pos[above:above + mult]] = thr
        r[pos[above + mult:]] = thr - rng.uniform(1, 50, M - above - mult)
        rows.append(r)
    # -0.0 and +0.0 at the threshold: numel - 2 positive values, then the zeros, then negative ones
    r = -rng.uniform(1, 9, M)
    pos = rng.permutation(M)
    k = max(0, numel - 2)
    r[pos[:k]] = rng.uniform(1, 9, k)
    nz = min(4, M - k)
    r[pos[k:k + nz]] = np.array([-0.0, 0.0, -0.0, 0.0])[:nz]
    rows.append(r)
    # +inf inside the top set
    r = rng.normal(0, 10, M)
    r[rng.integers(M)] = np.inf
    rows.append(r)
    # -inf below the top set: numel finite values, the rest -inf (what the warp kernel pads its lanes with)
    r = np.full(M, -np.inf)
    r[rng.permutation(M)[:numel]] = rng.normal(0, 10, numel)
    rows.append(r)
    # all negative
    rows.append(-np.abs(rng.normal(0, 100, M)) - 1)
    # magnitudes 1e-30 .. 1e30, both signs
    rows.append(np.where(rng.random(M) < 0.5, -1.0, 1.0) * 10.0 ** rng.uniform(-30, 30, M))
    # 1e30-sized values of one sign (the sum stays below float32's 3.4e38 for M <= 16384)
    rows.append(rng.uniform(1e30, 2e30, M))
    return np.ascontiguousarray(np.array(rows), dtype=F32)
