"""Directed one-step scenarios for the float64 contractions of the unicycle step and of the speed map's time cost (TEST
INFRASTRUCTURE).

Random scenarios cannot tell a float64 FMA from a product and a sum: the two differ by at most one float64 ulp, which
moves the float32 state only when the value lies within ~1e-16 of a float32 rounding boundary.  These cases are built
to lie there.  ``fma_boundary_case(A, kind)`` searches, with the arithmetic ``A`` of the kernel under test (its cos
provider decides the heading's cosine), for a forward speed v and a start x0 such that the first step's float32 x
differs between

* kind "state":    x = RN32(fma(dv, cos, x0))                 and  RN32(RN64(RN64(dv * cos) + x0))
* kind "traction": the traction value fma(ratio, q, lo)        and  RN64(RN64(ratio * q) + lo)   (lo != 0)

and then a goal and a tolerance that the exact x reaches and the other does not (or the reverse): a kernel that
contracts differently reports a different goal flag, hence a different cost.  The start x0 is tiny (|x0| << one
float32 ulp of dv * cos), which lets it place dv * cos + x0 between float64 grid points next to a float32 midpoint.

``speed_map_boundary_case(A)`` (kind "speed") searches for traction bounds, a risk byte r and a float32 dt for which the
speed map's time step RN32(dt / (eff + 1e-6)) differs between eff = fma(ratio, r, lo) and RN64(RN64(ratio * r) + lo).
Its scenario stands still at the goal (v = 0), so the one step reaches it with d2 = 0 and the cost is that time step
alone: a kernel that splits the contraction reports a cost one float32 ulp off.
"""
import numpy as np

from oracle import arith as AR

F32, F64 = np.float32, np.float64


def fma_boundary_case(A, kind, lb=(0.2, 1.3), th0=0.6, y0=0.3, dt=0.1):
    assert kind in ("state", "traction")
    dt64 = F64(F32(dt))
    lo, hi = F32(lb[0]), F32(lb[1])
    ratio, lo64 = 0.01 * F64(F32(hi - lo)), F64(lo)
    qs = np.arange(0, 101, dtype=F64)
    fused = AR.fma64_once(ratio, qs, lo64)
    if kind == "traction":
        differ = np.nonzero(fused != ratio * qs + lo64)[0]
        assert differ.size, "no traction byte where the two roundings differ for bounds %s" % (lb,)
        q = int(differ[0])
        vtr_e, vtr_m = fused[q], ratio * qs[q] + lo64
    else:
        q = 77
        vtr_e = vtr_m = fused[q]
    th = F32(th0)
    cs64 = F64(A.cos32(np.array([th], F32))[0])
    sn64 = F64(A.sin32(np.array([th], F32))[0])
    v = (F32(0.5) + np.arange(1 << 18, dtype=F32) * F32(2.0 ** -20)).astype(F32)
    dv_e = (vtr_e * dt64) * v.astype(F64)
    dv_m = (vtr_m * dt64) * v.astype(F64)
    p = dv_e * cs64
    ulp = np.spacing(p.astype(F32)).astype(F64)
    mid = (np.floor(p / ulp) + 0.5) * ulp                      # the float32 midpoint above p
    t = mid - p
    idx = np.nonzero((np.abs(t) < ulp * 2.0 ** -8) & (t != 0))[0]
    x0s = np.stack([t[idx].astype(F32)] * 7, 1)
    for k, j in enumerate((1, 2, 3)):                           # neighbours of the rounded offset
        x0s[:, 1 + 2 * k] = x0s[:, 0]
        x0s[:, 2 + 2 * k] = x0s[:, 0]
        for _ in range(j):
            x0s[:, 1 + 2 * k] = np.nextafter(x0s[:, 1 + 2 * k], F32(np.inf))
            x0s[:, 2 + 2 * k] = np.nextafter(x0s[:, 2 + 2 * k], F32(-np.inf))
    de, dm = np.repeat(dv_e[idx], 7), np.repeat(dv_m[idx], 7)
    x0 = x0s.reshape(-1)
    xe = AR.fma64_once(de, cs64, x0.astype(F64)).astype(F32)
    xm = (dm * cs64 + x0.astype(F64)).astype(F32) if kind == "state" else \
        AR.fma64_once(dm, cs64, x0.astype(F64)).astype(F32)
    for i in np.nonzero(xe != xm)[0]:
        ye = AR.fma64_once(de[i], sn64, F64(F32(y0))).astype(F32)
        ym = F32(dm[i] * sn64 + F64(F32(y0))) if kind == "state" else AR.fma64_once(dm[i], sn64, F64(F32(y0))).astype(F32)
        goal = (F32(0.0), ye)

        def d2(x, y):
            dx, dy = A.sub32(goal[0], x), A.sub32(goal[1], y)
            return F32(A.fma32(np.array([dx]), np.array([dx]), A.mul32(np.array([dy]), np.array([dy])))[0])
        d2e, d2m = d2(xe[i], ye), d2(xm[i], ym)
        if d2e == d2m:
            continue
        lo2, hi2 = min(d2e, d2m), max(d2e, d2m)
        tol = F32(np.sqrt(F64(lo2)))
        for _ in range(8):                                      # tol2 = RN32(tol * tol) in [lo2, hi2)
            tol2 = F32(tol * tol)
            if tol2 < lo2:
                tol = np.nextafter(tol, F32(np.inf))
            elif tol2 >= hi2:
                tol = np.nextafter(tol, F32(-np.inf))
            else:
                break
        if not (lo2 <= F32(tol * tol) < hi2):
            continue
        return dict(kind=kind, lb=[float(lo), float(hi)], q=q, v=F32(v[idx[i // 7]]), x0=[float(x0[i]), float(F32(y0)), float(th)],
                    goal=[float(goal[0]), float(goal[1])], tol=float(tol), x1_exact=xe[i], x1_other=xm[i],
                    exact_reaches=bool(d2e <= F32(tol * tol)), dt=float(dt64))
    raise AssertionError("no %s boundary case found" % kind)


def speed_map_boundary_case(A, seed=0, x0=(0.3, 0.3, 0.6), q=100):
    """Bounds (lo, hi) drawn from ``seed``, risk byte r and dt: the first float32 dt in [1/16, 1/8) and the first byte of
    the first bounds where the fused and the split eff give different float32 time steps.  Traction byte ``q``."""
    dts = (F32(1 / 16) + np.arange(1 << 23, dtype=F64) * 2.0 ** -27).astype(F32)     # every float32 in [1/16, 1/8)
    dt64 = dts.astype(F64)
    qs = np.arange(0, 101, dtype=F64)
    rng = np.random.default_rng(seed)
    for _ in range(64):
        lo, hi = F32(rng.uniform(0.05, 0.5)), F32(rng.uniform(0.8, 1.5))
        ratio, lo64 = 0.01 * F64(F32(hi - lo)), F64(lo)
        fused = A.fma64(np.full(101, ratio), qs, np.full(101, lo64))
        split = ratio * qs + lo64
        for r in np.nonzero(fused != split)[0]:
            k = np.nonzero((dt64 / (fused[r] + 1e-6)).astype(F32) != (dt64 / (split[r] + 1e-6)).astype(F32))[0]
            if not k.size:
                continue
            dt = dt64[k[0]]

            def cost(eff):                       # one step at the goal: d2 = 0, cost = 0 + (sqrt(0) * w + dt_eff)
                dt_eff = A.d2f(np.array([dt / (eff + 1e-6)]))
                return F32(A.add32(F32(0), A.fma32(A.sqrt32(np.zeros(1, F32)), F32(1), dt_eff))[0])
            ce, cm = cost(fused[r]), cost(split[r])
            assert ce != cm, "speed case: the fused and the split time step give the same cost"
            x = F32(x0[0])
            return dict(kind="speed", lb=[float(lo), float(hi)], q=q, risk=int(r), v=F32(0), dt=float(dt),
                        x0=[float(x), float(F32(x0[1])), float(F32(x0[2]))], goal=[float(x), float(F32(x0[1]))],
                        tol=0.5, T=1, x1_exact=x, x1_other=x, exact_reaches=True, cost_exact=ce, cost_other=cm)
    raise AssertionError("no speed boundary case found")


def boundary_case(A, kind):
    """The directed case of a kind: "state" and "traction" (fma_boundary_case) or "speed" (speed_map_boundary_case)."""
    return speed_map_boundary_case(A) if kind == "speed" else fma_boundary_case(A, kind)


def directed_scenario(case, N=33, M=2, T=None):
    """Inputs of a directed case: uniform maps (traction byte ``case['q']``, risk byte ``case['risk']`` or the traction
    byte), no masks, no noise, speed v, its start, goal, tolerance and dt -- the first step decides the goal flag by one
    float32 ulp of x (or, kind "speed", the cost by one float32 ulp of the time step).  T: the case's, else 2."""
    R = Cc = 100
    T = case.get("T", 2) if T is None else T
    s = dict(N=N, M=M, T=T, R=R, Cc=Cc, res=F32(0.1), xlo=F32(-5.0), ylo=F32(-5.0), lb=case["lb"], ab=[0.0, 1.0],
             x0=case["x0"], goal=case["goal"], tol=case["tol"], dt=case["dt"], shift=(0, 0))
    s["lin"] = np.full((M, R, Cc), case["q"], np.int8)
    s["ang"] = np.full((M, R, Cc), 50, np.int8)
    s["obs"] = np.zeros((R, Cc), np.int8)
    s["unk"] = np.zeros((R, Cc), np.int8)
    s["risk"] = np.full((R, Cc), case.get("risk", case["q"]), np.int8)
    s["noise"] = np.zeros((N, T, 2), F32)
    s["u_cur"] = np.zeros((T, 2), F32)
    s["u_cur"][:, 0] = case["v"]
    return s
