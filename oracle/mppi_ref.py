"""CPU restatement of the planner side of the hot path (TEST INFRASTRUCTURE, see oracle/__init__.py).

Follows mppi_numba/mppi.py of the reference, typed as the COMPILED kernels type it (PTX census in
SURVEY.md 2.3; re-derived from ``numba.cuda.compile_ptx`` of the reference kernels):
  * sample_noise_numba            mppi.py:1354-1370
  * rollout_numba                 mppi.py:613-755   (stochastic, "CVaR-cost"; per-(n,m) costs + CVaR)
  * rollout_det_dyn_numba         mppi.py:916-1009  (deterministic, "CVaR-dynamics"/nominal)
  * rollout_det_dyn_w_speed_map   mppi.py:1013-1111 (nominal dynamics + worst-case speed map)
  * update_useq_numba             mppi.py:1113-1191
  * shift_optimal_control_sequence mppi.py:539-542
Every floating-point operation of the rollouts and of the noise goes through an arithmetic object
(oracle/arith.py, argument ``arith``):

* default (``arith=None``, ``oracle.arith.NUMPY``) -- exact-math stand-ins: numpy float32 sin/cos/sqrt and IEEE
  division replace sin.approx/cos.approx/sqrt.approx/div.approx/div.full of the GPU build (~1e-7 relative per op), and
  a float32 FMA is a float64 multiply-add rounded twice, a float64 FMA a product and a sum.  What the reference's
  golden vectors are checked against (<= 2e-6), and what bench.py's cpu_baseline leg times.
* ``oracle.arith.Exact(provider, ftz)`` -- the exact oracle: each operation placed and rounded where the kernels
  (csrc/rollout.cu, csrc/rollout_win.cu) place it -- the FMA contractions the compiled code has, each rounded once,
  float32 add / sub / mul rounded once, optionally the .ftz flushes -- and the approximate operations from a provider:
  ``LibmProvider`` (what the host emulation of the kernels uses) or ``DeviceProvider`` (the GPU's own results).  With
  the provider of the machine that runs the kernel, costs, states and noise are predicted bit for bit.

``ctrl_order`` chooses the control-cost summation of the stochastic mode: "sequential" (each term added to the running
cost, as the reference and the generic kernel do) or "presummed" (the windowed kernel: the terms summed from 0 by
an FMA chain, the total added after the stage costs).
"""
import math
import numpy as np

from . import arith as AR
from . import xoroshiro as X

F32 = np.float32
F64 = np.float64

MODE_STOCHASTIC = 0      # use_tdm
MODE_DET_DYN = 1         # use_det_dynamics
MODE_SPEED_MAP = 2       # use_nom_dynamics_with_speed_map
MODE_BAREBONE = 3        # the map-free notebook planner (rollout_costs_barebone, state_rollouts_barebone)

DEFAULT_UNKNOWN_COST = 1e2   # mppi.py:32
DEFAULT_OBS_COST = 1e5       # mppi.py:33
DEFAULT_DIST_WEIGHT = 1.0    # mppi.py:36


def _fma32(a, b, c):
    """fma.rn.f32: the float64 product of two float32 is exact; one extra rounding in the sum is
    below 2**-29 relative -- negligible against the exact-math stand-ins above."""
    return (a.astype(F64) * F64(b) + c.astype(F64)).astype(F32) if np.ndim(b) == 0 else \
           (a.astype(F64) * b.astype(F64) + c.astype(F64)).astype(F32)


# ----------------------------------------------------------------------------- noise
def sample_noise(states, u_std, N, T, arith=None):
    """mppi.py:1365-1370: generator n*T+t produces BOTH components (two Box-Muller calls = 4 draws)."""
    A = arith or AR.NUMPY
    us = np.asarray(u_std, dtype=F32)
    z0 = X.normal_float32(states, arith=arith)            # all N*T generators advance together
    z1 = X.normal_float32(states, arith=arith)
    noise = np.empty((N, T, 2), dtype=F32)
    noise[..., 0] = A.mul32(us[0], z0).reshape(N, T)
    noise[..., 1] = A.mul32(us[1], z1).reshape(N, T)
    return noise


# ----------------------------------------------------------------------------- cell index
def floor_div_f32(a, r, arith=None):
    """Python ``//`` on float32 as Numba lowers it (numba/cpython/numbers.py real_divmod; PTX of
    rollout_det_dyn_numba): remainder via abs/div.rn/floor/mul/sub, quotient (a-mod)/r, sign fix,
    floor, snap-to-nearest.  ptxas contracts the remainder's mul+sub into ONE FMA (SASS of the
    reference kernel: FFMA.FTZ m = -floor(t)*|r| + |a|), i.e. the remainder is exact -- the same
    result CPython's fmod-based float_divmod gives in the simulator.
    ``a`` float32 array, ``r`` float32 scalar != 0.

    With an exact ``arith`` the sequence is csrc/common.cuh::cell_index_exact operation by operation (div.rn,
    cvt.rmi, the contracted FMA, div.full from the provider, the q == 0 / NaN branch, cvt.rzi)."""
    if arith is not None and arith.exact:
        return _floor_div_exact(a, r, arith)
    a = a.astype(F32)
    r = F32(r)
    aa = np.abs(a)
    rr = np.abs(r)
    t = (aa / rr).astype(F32)
    m = (aa.astype(F64) - np.floor(t).astype(F64) * F64(rr)).astype(F32)      # one rounding (FMA)
    m = np.where(a < 0, -m, m).astype(F32)
    q = ((a - m).astype(F32) / r).astype(F32)
    fix = (m != 0) & ((r < 0) != (m < 0))
    q = np.where(fix, (q - F32(1)).astype(F32), q)
    fl = np.floor(q)
    fl = np.where((q - fl).astype(F32) > F32(0.5), fl + F32(1), fl)
    res = np.where(q == 0, F32(0), fl)
    return res.astype(np.int32)                      # cvt.rzi


def _floor_div_exact(a, r, A):
    a = np.asarray(a, dtype=F32)
    r = F32(r)
    aa, rr = np.abs(A.f2d(a).astype(F32)), np.abs(r)              # fabsf of the (flushed) operand
    t = A.div_rn32(aa, rr)
    m = A.fma32(-A.floor32(t), rr, aa)
    m = np.where(a < 0, -m, m).astype(F32)
    q = A.div_full32(A.sub32(a, m), r)
    fix = (m != 0) & ((r < 0) != (m < 0))
    q = np.where(fix, A.add32(q, F32(-1)), q).astype(F32)
    fl = A.floor32(q)
    res = np.where(A.sub32(q, fl) > F32(0.5), A.add32(fl, F32(1)), fl).astype(F32)
    odd = (q == 0) | np.isnan(q)
    if odd.any():
        res = np.where(odd, A.div_full32(A.mul32(a, A.mul32(q, q)), r), res).astype(F32)
    res = np.where(np.isnan(res), F32(0), res)        # cvt.rzi of NaN is 0
    return np.trunc(res).astype(np.int32)


# ----------------------------------------------------------------------------- rollouts
def rollout_costs(mode, lin_grid, ang_grid, lin_bounds, ang_bounds, obstacle_map, unknown_map,
                  res, xlimits, ylimits, vrange, wrange, xgoal, v_post_rollout, obs_cost, unknown_cost,
                  goal_tolerance, lambda_weight, u_std, x0, dt, dist_weight, noise, u_cur,
                  risk_map=None, return_states=False, arith=None, ctrl_order="sequential", wrap_clamp=False):
    """Per-(n, m) rollout cost, float32 (N, Mg).  Mg = lin_grid.shape[0] maps are used in
    MODE_STOCHASTIC, map 0 only otherwise (tid == 0 in the one-thread blocks, mppi.py:334,978).

    Loop body mppi.py:677-706 / 969-1001 / 1069-1103; epilogue order: stochastic adds the control
    cost then the terminal cost (:708-713), the deterministic kernels add terminal then control
    (:1004-1009, :1106-1111).  ``arith`` / ``ctrl_order``: see the module docstring.  ``wrap_clamp``: the engine's rule
    for cells outside the map (negative indices wrapped like Numba's indexing, then clamped into the array; the
    reference reads outside its allocation there -- DESIGN.md 2); otherwise such a lookup is an IndexError."""
    A = arith or AR.NUMPY
    if ctrl_order not in ("sequential", "presummed"):
        raise ValueError("ctrl_order: 'sequential' or 'presummed'")
    noise = np.asarray(noise, dtype=F32)
    u_cur = np.asarray(u_cur, dtype=F32)
    N, T, _ = noise.shape
    Mg = lin_grid.shape[0] if mode == MODE_STOCHASTIC else 1
    lb = np.asarray(lin_bounds, dtype=F32)
    ab = np.asarray(ang_bounds, dtype=F32)
    xl = np.asarray(xlimits, dtype=F32)
    yl = np.asarray(ylimits, dtype=F32)
    vr = np.asarray(vrange, dtype=F32)
    wr = np.asarray(wrange, dtype=F32)
    xg = np.asarray(xgoal, dtype=F32)
    us = np.asarray(u_std, dtype=F32)
    x0 = np.asarray(x0, dtype=F32)
    res, dt = F32(res), F32(dt)
    v_post, obs_c, unk_c = F32(v_post_rollout), F32(obs_cost), F32(unknown_cost)
    tol2 = F32(F32(goal_tolerance) * F32(goal_tolerance))
    lam = F32(lambda_weight)
    w_dist = F32(dist_weight)                        # stage_cost signature casts to float32 (mppi.py:20)

    lin_ratio = 0.01 * F64(F32(lb[1] - lb[0]))       # float64 (mppi.py:674)
    ang_ratio = 0.01 * F64(F32(ab[1] - ab[0]))
    dt64 = A.f2d(dt)
    lin_lo, ang_lo = A.f2d(lb[0]), A.f2d(ab[0])

    x = np.full((N, Mg), x0[0], dtype=F32)
    y = np.full((N, Mg), x0[1], dtype=F32)
    th = np.full((N, Mg), x0[2], dtype=F32)
    cost = np.zeros((N, Mg), dtype=F32)
    d2 = np.full((N, Mg), 1e9, dtype=F32)            # dist_to_goal2 = 1e9 (values stay f32-exact)
    active = np.ones((N, Mg), dtype=bool)
    reached = np.zeros((N, Mg), dtype=bool)
    m_idx = np.broadcast_to(np.arange(Mg)[None, :], (N, Mg))
    states = np.zeros((N, Mg, T + 1, 3), dtype=F32) if return_states else None
    if return_states:
        states[:, :, 0, :] = x0

    for t in range(T):
        if not active.any():
            break
        xi = floor_div_f32(A.sub32(x, xl[0]), res, A)
        yi = floor_div_f32(A.sub32(y, yl[0]), res, A)
        gy, gx, my, mx = yi, xi, yi, xi
        if wrap_clamp:
            gy, gx = _wrap_clamp(yi, lin_grid.shape[1]), _wrap_clamp(xi, lin_grid.shape[2])
            my, mx = _wrap_clamp(yi, obstacle_map.shape[0]), _wrap_clamp(xi, obstacle_map.shape[1])
        ql = lin_grid[m_idx, gy, gx].astype(F64)
        qa = ang_grid[m_idx, gy, gx].astype(F64)
        vtr = A.fma64(lin_ratio, ql, lin_lo)          # fma(ratio, q, lo): the traction value, one rounding
        wtr = A.fma64(ang_ratio, qa, ang_lo)
        v_nom = A.add32(u_cur[t, 0], noise[:, t, 0])
        w_nom = A.add32(u_cur[t, 1], noise[:, t, 1])
        v = np.maximum(vr[0], np.minimum(vr[1], v_nom)).astype(F32)[:, None]
        w = np.maximum(wr[0], np.minimum(wr[1], w_nom)).astype(F32)[:, None]
        dv = (vtr * dt64) * A.f2d(v)
        c32 = A.cos32(th)
        s32 = A.sin32(th)
        xn = A.d2f(A.fma64(dv, A.f2d(c32), A.f2d(x)))  # float64 FMA rounded once to float32
        yn = A.d2f(A.fma64(dv, A.f2d(s32), A.f2d(y)))
        thn = A.d2f(A.fma64(wtr * dt64, A.f2d(w), A.f2d(th)))
        dx = A.sub32(xg[0], xn)
        dy = A.sub32(xg[1], yn)
        d2n = A.fma32(dx, dx, A.mul32(dy, dy))
        sq = A.sqrt32(d2n)
        if mode == MODE_SPEED_MAP:
            eff = A.fma64(lin_ratio, risk_map[0, my, mx].astype(F64), lin_lo)
            dt_eff = A.d2f(dt64 / (eff + 1e-6))
            stage = A.fma32(sq, w_dist, dt_eff)
        else:
            stage = A.fma32(sq, w_dist, np.full_like(sq, dt))
        cn = A.add32(cost, stage)
        cn = A.fma32(obstacle_map[my, mx].astype(F32), obs_c, cn)
        cn = A.fma32(unknown_map[my, mx].astype(F32), unk_c, cn)
        x = np.where(active, xn, x)
        y = np.where(active, yn, y)
        th = np.where(active, thn, th)
        cost = np.where(active, cn, cost)
        d2 = np.where(active, d2n, d2)
        hit = active & (d2n <= tol2)
        reached |= hit
        active &= ~hit
        if return_states:
            states[:, :, t + 1, 0] = x
            states[:, :, t + 1, 1] = y
            states[:, :, t + 1, 2] = th

    def add_terminal(c):
        term = ((1.0 - reached.astype(F64)) * A.f2d(A.sqrt32(d2))) / (A.f2d(v_post) + 1e-6)
        return A.add32(c, A.d2f(term))

    def add_control(c):
        terms = _control_terms(A, us, u_cur, noise)
        if ctrl_order == "presummed":                 # rollout_win.cu: FMA chain from 0, total added once
            acc = np.zeros(N, dtype=F32)
            for s in terms:
                acc = A.fma32(s, lam, acc)
            return A.add32(c, acc[:, None])
        for s in terms:
            c = A.fma32(np.broadcast_to(s[:, None], c.shape).astype(F32), lam, c)
        return c

    if mode == MODE_STOCHASTIC:
        cost = add_terminal(add_control(cost))
    else:
        cost = add_control(add_terminal(cost))
    if return_states:
        return cost, states
    return cost


def _wrap_clamp(i, n):
    """csrc/rollout.cu wrap_clamp: i < 0 -> i + n, then clamped to [0, n - 1]."""
    return np.clip(np.where(i < 0, i + n, i), 0, n - 1)


def _control_terms(A, us, u_cur, noise):
    """The per-step control-cost terms u_v/s_v^2 * e_v + u_w/s_w^2 * e_w (mppi.py:708-710; rollout.cu ctrl_term),
    float32 (N,) each."""
    N, T, _ = noise.shape
    sv2 = A.mul32(us[0], us[0])
    sw2 = A.mul32(us[1], us[1])
    for t in range(T):
        a = A.div_approx32(u_cur[t, 0], sv2)
        b = A.div_approx32(u_cur[t, 1], sw2)
        p = A.mul32(b, noise[:, t, 1])
        yield A.fma32(np.full(N, a, dtype=F32), noise[:, t, 0], p)


def state_rollouts(mode, V, lin_grid, ang_grid, lin_bounds, ang_bounds, res, xlimits, ylimits, x0, dt,
                   u_cur, u_prev=None, noise=None, vrange=None, wrange=None, arith=None, wrap_clamp=False):
    """get_state_rollout's kernels (mppi.py:1194-1351): float32 (V, T+1, 3), no goal test, no costs.

    MODE_STOCHASTIC -- get_state_rollout_across_envs_numba (:1303-1351): u_cur, unclipped and without
      noise, rolled out on sampled maps 0..V-1.
    other modes -- get_state_rollout_across_control_noise (:1194-1300) on map 0 (tid == 0 in its one-thread
      blocks): block 0 rolls out u_cur unclipped, block b > 0 rolls out clip(u_prev + noise[b])."""
    u_cur = np.asarray(u_cur, dtype=F32)
    T = u_cur.shape[0]
    Hg, Wg = lin_grid.shape[1:]
    zeros = np.zeros((Hg, Wg), dtype=np.int8)
    far = np.array([1e18, 1e18], dtype=F32)              # never within the (zero) goal tolerance
    wide = np.array([-np.inf, np.inf], dtype=F32)

    def run(grid_mode, lg, ag, noise_, u_, vr, wr):
        _, st = rollout_costs(grid_mode, lg, ag, lin_bounds, ang_bounds, zeros, zeros, res, xlimits, ylimits,
                              vr, wr, far, 1.0, 0.0, 0.0, 0.0, 1.0, [1.0, 1.0], x0, dt, 1.0, noise_, u_,
                              return_states=True, arith=arith, wrap_clamp=wrap_clamp)
        return st
    if mode == MODE_STOCHASTIC:
        st = run(MODE_STOCHASTIC, lin_grid[:V], ang_grid[:V], np.zeros((1, T, 2), dtype=F32), u_cur, wide, wide)
        return st[0]                                     # (V, T+1, 3)
    out = np.zeros((V, T + 1, 3), dtype=F32)
    out[0] = run(MODE_DET_DYN, lin_grid[:1], ang_grid[:1], np.zeros((1, T, 2), dtype=F32), u_cur, wide, wide)[0, 0]
    if V > 1:
        st = run(MODE_DET_DYN, lin_grid[:1], ang_grid[:1], np.asarray(noise, dtype=F32)[1:V],
                 np.asarray(u_prev, dtype=F32), vrange, wrange)
        out[1:] = st[:, 0]
    return out


def rollout_costs_barebone(obs_pos, obs_r, vrange, wrange, xgoal, obs_cost, goal_tolerance, lambda_weight, u_std,
                           x0, dt, dist_weight, noise, u_cur, return_states=False, arith=None):
    """The map-free variant of the reference's barebone_mppi_numba.ipynb (cell 3, rollout_numba): nominal
    unicycle in float32 (dv = dt*v; x = fma(dv, cos, x); theta = fma(w, dt, theta)), stage cost w*d^2,
    circular obstacles (indicator of d^2 - r^2 <= 0, float64 FMA into the float32 cost), terminal cost
    (1-reached)*d^2, then the control cost.  Contractions as in the SASS of the compiled kernel.  ``arith``: see the
    module docstring."""
    A = arith or AR.NUMPY
    noise = np.asarray(noise, dtype=F32)
    u_cur = np.asarray(u_cur, dtype=F32)
    N, T, _ = noise.shape
    vr, wr = np.asarray(vrange, dtype=F32), np.asarray(wrange, dtype=F32)
    xg, us = np.asarray(xgoal, dtype=F32), np.asarray(u_std, dtype=F32)
    x0 = np.asarray(x0, dtype=F32)
    dt, lam, w_dist, obs_c = F32(dt), F32(lambda_weight), F32(dist_weight), F32(obs_cost)
    tol2 = F32(F32(goal_tolerance) * F32(goal_tolerance))
    op = np.asarray(obs_pos, dtype=F32).reshape(-1, 2)
    orad = np.asarray(obs_r, dtype=F32).reshape(-1)
    x = np.full(N, x0[0], dtype=F32)
    y = np.full(N, x0[1], dtype=F32)
    th = np.full(N, x0[2], dtype=F32)
    cost = np.zeros(N, dtype=F32)
    d2 = np.full(N, 1e9, dtype=F32)
    active = np.ones(N, dtype=bool)
    reached = np.zeros(N, dtype=bool)
    states = np.zeros((N, T + 1, 3), dtype=F32) if return_states else None
    if return_states:
        states[:, 0, :] = x0
    for t in range(T):
        if not active.any():
            break
        v = np.maximum(vr[0], np.minimum(vr[1], A.add32(u_cur[t, 0], noise[:, t, 0]))).astype(F32)
        w = np.maximum(wr[0], np.minimum(wr[1], A.add32(u_cur[t, 1], noise[:, t, 1]))).astype(F32)
        dv = A.mul32(v, dt)
        xn = A.fma32(dv, A.cos32(th), x)
        yn = A.fma32(dv, A.sin32(th), y)
        thn = A.fma32(w, dt, th)
        dx, dy = A.sub32(xg[0], xn), A.sub32(xg[1], yn)
        d2n = A.fma32(dx, dx, A.mul32(dy, dy))
        cn = A.fma32(d2n, w_dist, cost)
        if len(orad):                                   # the indicators of every obstacle at once (N, K) ...
            ddx, ddy = A.sub32(xn[:, None], op[None, :, 0]), A.sub32(yn[:, None], op[None, :, 1])
            q = A.fma32(ddx, ddx, A.mul32(ddy, ddy))
            diff = A.fma32(-orad[None, :], orad[None, :], q)                              # FFMA(-r, r, q)
            inside = 1.0 - (diff > 0).astype(F64)
        for k in range(len(orad)):                      # ... and their penalties added in the kernel's order
            cn = A.d2f(A.fma64(inside[:, k], A.f2d(obs_c), A.f2d(cn)))
        x, y, th = np.where(active, xn, x), np.where(active, yn, y), np.where(active, thn, th)
        cost, d2 = np.where(active, cn, cost), np.where(active, d2n, d2)
        hit = active & (d2n <= tol2)
        reached |= hit
        active &= ~hit
        if return_states:
            states[:, t + 1, 0], states[:, t + 1, 1], states[:, t + 1, 2] = x, y, th
    cost = A.add32(cost, A.d2f(np.where(reached, 0.0, 1.0) * A.f2d(d2)))
    for sterm in _control_terms(A, us, u_cur, noise):
        cost = A.fma32(sterm, lam, cost)
    if return_states:
        return cost, states
    return cost


def state_rollouts_barebone(V, x0, dt, u_cur, u_prev=None, noise=None, vrange=None, wrange=None, arith=None):
    """get_state_rollout of the barebone notebook (cell 3, get_state_rollout_across_control_noise): float32 (V, T+1, 3),
    the nominal unicycle of rollout_costs_barebone (dv = v*dt; x = fma(dv, cos, x); theta = fma(w, dt, theta)) with no
    goal test and no early exit.  Row 0 rolls out u_cur unclipped and without noise, row b > 0 rolls out
    clip(u_prev + noise[b])."""
    A = arith or AR.NUMPY
    u_cur = np.asarray(u_cur, dtype=F32)
    T = u_cur.shape[0]
    x0 = np.asarray(x0, dtype=F32)
    dt = F32(dt)
    v = np.empty((V, T), dtype=F32)
    w = np.empty((V, T), dtype=F32)
    v[0], w[0] = u_cur[:, 0], u_cur[:, 1]
    if V > 1:
        e = np.asarray(noise, dtype=F32)[1:V]
        u_prev = np.asarray(u_prev, dtype=F32)
        vr, wr = np.asarray(vrange, dtype=F32), np.asarray(wrange, dtype=F32)
        v[1:] = np.maximum(vr[0], np.minimum(vr[1], A.add32(u_prev[None, :, 0], e[..., 0])))
        w[1:] = np.maximum(wr[0], np.minimum(wr[1], A.add32(u_prev[None, :, 1], e[..., 1])))
    out = np.zeros((V, T + 1, 3), dtype=F32)
    out[:, 0, :] = x0
    x = np.full(V, x0[0], dtype=F32)
    y = np.full(V, x0[1], dtype=F32)
    th = np.full(V, x0[2], dtype=F32)
    for t in range(T):
        dv = A.mul32(v[:, t], dt)
        cs, sn = A.cos32(th), A.sin32(th)
        x, y, th = A.fma32(dv, cs, x), A.fma32(dv, sn, y), A.fma32(w[:, t], dt, th)
        out[:, t + 1, 0], out[:, t + 1, 1], out[:, t + 1, 2] = x, y, th
    return out


def cvar_count(M, cvar_alpha):
    """mppi.py:744: ceil(int32 * float32) evaluated in float64 (SURVEY.md 9-N3)."""
    return int(math.ceil(float(M) * float(F32(cvar_alpha))))


def cvar_reduce(costs_nm, cvar_alpha):
    """mppi.py:718-755: descending sort when alpha < 1, pairwise tree sum (float32) over the first
    ``numel`` entries in the reference's stride order, divided by numel."""
    c = np.array(costs_nm, dtype=F32, copy=True)
    N, M = c.shape
    a32 = F32(cvar_alpha)
    if a32 < 1:
        c = -np.sort(-c, axis=1)
    numel = cvar_count(M, a32)
    s = 1
    while s < numel:
        tid = np.arange(0, M, 2 * s)
        tid = tid[tid + s < numel]
        c[:, tid] = (c[:, tid] + c[:, tid + s]).astype(F32)
        s *= 2
    return (c[:, 0].astype(F64) / F64(numel)).astype(F32)


# ----------------------------------------------------------------------------- update
def update_useq(lambda_weight, costs, noise, vrange, wrange, u_cur):
    """mppi.py:1128-1191 with the single-warp data race (SURVEY.md 9-R1) resolved the way the
    hardware resolves it (beta = the true minimum).  Returns (u_new (T,2) f32, weights (N,) f32).
    w_n = float32(exp(float64(-1/lambda) * float64(c_n - beta))); normalised by their float32 sum;
    u[t] += sum_n w_n * eps[n,t] (atomic order is unspecified in the reference: summed here in
    float64); clipped to vrange / wrange."""
    costs = np.asarray(costs, dtype=F32)
    noise = np.asarray(noise, dtype=F32)
    lam = F32(lambda_weight)
    beta = costs.min()
    w = np.exp((-1.0 / F64(lam)) * (costs - beta).astype(F32).astype(F64)).astype(F32)
    total = F32(np.sum(w.astype(F64)))
    wn = (w / total).astype(F32)
    du = np.einsum("n,ntk->tk", wn.astype(F64), noise.astype(F64))
    u = (np.asarray(u_cur, dtype=F32).astype(F64) + du).astype(F32)
    vr = np.asarray(vrange, dtype=F32)
    wr = np.asarray(wrange, dtype=F32)
    u[:, 0] = np.maximum(vr[0], np.minimum(vr[1], u[:, 0]))
    u[:, 1] = np.maximum(wr[0], np.minimum(wr[1], u[:, 1]))
    return u, wn


def shift_useq(u_cur, num_shifts=1):
    """mppi.py:539-542: u[:-s] = u[s:]; the tail keeps its old values (SURVEY.md 9-Q4)."""
    u = np.array(u_cur, dtype=F32, copy=True)
    u[:-num_shifts] = u[num_shifts:]
    return u


# ----------------------------------------------------------------------------- whole solve
def solve_iteration(mode, rng_states, grids, maps, p, u_cur, N, T):
    """One ``num_opt`` iteration of solve_det_dyn / solve_stochastic (mppi.py:329-364, 402-440)
    given already-sampled grids.  ``p`` is the params dict.  Returns (u_new, costs_n, costs_nm, noise, weights)."""
    noise = sample_noise(rng_states, p["u_std"], N, T)
    cnm = rollout_costs(mode, grids["lin"], grids["ang"], maps["lin_bounds"], maps["ang_bounds"],
                        maps["obstacle"], maps["unknown"], maps["res"], maps["xlimits"], maps["ylimits"],
                        p["vrange"], p["wrange"], p["xgoal"], p["v_post_rollout"],
                        p.get("obs_penalty", DEFAULT_OBS_COST), p.get("unknown_penalty", DEFAULT_UNKNOWN_COST),
                        p["goal_tolerance"], p["lambda_weight"], p["u_std"], p["x0"], p["dt"],
                        p.get("dist_weight", DEFAULT_DIST_WEIGHT), noise, u_cur, risk_map=maps.get("risk"))
    cn = cvar_reduce(cnm, p["cvar_alpha"]) if mode == MODE_STOCHASTIC else cnm[:, 0].copy()
    u_new, w = update_useq(p["lambda_weight"], cn, noise, p["vrange"], p["wrange"], u_cur)
    return u_new, cn, cnm, noise, w
