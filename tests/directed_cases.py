"""Directed one-step scenarios for the two float64 contractions of the unicycle step (TEST INFRASTRUCTURE).

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
                    exact_reaches=bool(d2e <= F32(tol * tol)))
    raise AssertionError("no %s boundary case found" % kind)


def directed_scenario(case, N=33, M=2, T=2):
    """Inputs of a case of fma_boundary_case: uniform maps (traction byte ``case['q']``), no masks, no noise, speed v, its
    start, goal and tolerance -- the first step decides the goal flag by one float32 ulp of x."""
    R = Cc = 100
    s = dict(N=N, M=M, T=T, R=R, Cc=Cc, res=F32(0.1), xlo=F32(-5.0), ylo=F32(-5.0), lb=case["lb"], ab=[0.0, 1.0],
             x0=case["x0"], goal=case["goal"], tol=case["tol"], shift=(0, 0))
    s["lin"] = np.full((M, R, Cc), case["q"], np.int8)
    s["ang"] = np.full((M, R, Cc), 50, np.int8)
    s["obs"] = np.zeros((R, Cc), np.int8)
    s["unk"] = np.zeros((R, Cc), np.int8)
    s["risk"] = np.full((R, Cc), case["q"], np.int8)
    s["noise"] = np.zeros((N, T, 2), F32)
    s["u_cur"] = np.zeros((T, 2), F32)
    s["u_cur"][:, 0] = case["v"]
    return s
