"""Soundness of the reach box (reach_box_decide, csrc/kernels.h, compiled from the header's text for the host): every
cell a rollout reads at steps 0 .. T-1 lies in the region the sampler is obliged to write for the decided box -- box rows
x box columns, intersected with the reach disc (the `need` region of test_sampler_kernel_source_boxed_launch, which
proves the sampler writes every such cell).  Together: every cell a boxed solve reads was sampled this solve.

The rollouts are adversarial: straight lines (w = 0) at the speed limit or just below it, per-step displacements just
above half an ulp of the coordinate (each step then rounds up to a whole ulp, twice the exact motion), map origins far
from 0 (georeferenced maps), reverse driving, negative traction, cos / sin off by 2e-6 (the approximate MUFU functions).
Their float32 states follow the oracle's arithmetic (oracle/mppi_ref.py rollout_costs: dv = (traction * dt) * v in
float64, x = f32(dv * cos + x), cell = floor_div_f32(f32(x - xlo), res)).  Boxed decisions must also stay tight."""
import ctypes as C

import numpy as np
import pytest

from oracle import mppi_ref as MR
from tests.emu_core import build, region

F32, F64 = np.float32, np.float64
U = 2.0 ** -24

HARNESS = r'''
extern "C" int emu_decide(const int* ci, const float* cf, float x, float y, const float* reach, int* out, float* outf) {
  using namespace b200;
  ReachBoxConst c{};
  c.mode = ci[0]; c.disc = ci[1]; c.T = ci[2]; c.rows = ci[3]; c.cols = ci[4];
  c.nt = ci[5]; c.tx = ci[6]; c.ty = ci[7]; c.num_maps = ci[8]; c.bpad0 = ci[9]; c.bpad1 = ci[10];
  c.vr0 = cf[0]; c.vr1 = cf[1]; c.dt = cf[2]; c.tr_abs_max = cf[3]; c.res = cf[4]; c.pxl = cf[5]; c.pyl = cf[6];
  ReachBox b;
  const int how = reach_box_decide(c, x, y, reach, &b);
  out[0] = how; out[1] = b.row_lo; out[2] = b.row_hi; out[3] = b.col_lo; out[4] = b.col_hi;
  outf[0] = b.cx; outf[1] = b.cy; outf[2] = b.r;
  return how;
}
'''


@pytest.fixture(scope="module")
def decide(tmp_path_factory):
    lib = build(str(tmp_path_factory.mktemp("reachbox")), "reachbox", [region("kernels.h", "sampler_args")], HARNESS)

    def run(mode, T, rows, cols, vr, dt, trm, res, pxl, pyl, x, y, reach=None):
        # one TDM, 16 x 256 generator tiles, 64 maps: a staged launch that fits any box of these maps
        ci = (C.c_int * 11)(mode, 1, T, rows, cols, 1, 16, 256, 64, 4, 4)
        cf = (C.c_float * 7)(vr[0], vr[1], dt, trm, res, pxl, pyl)
        o, of = (C.c_int * 5)(), (C.c_float * 3)()
        r = None if reach is None else C.byref(C.c_float(reach))
        lib.emu_decide(ci, cf, float(x), float(y), r, o, of)
        return list(o), [float(v) for v in of]
    return run


def straight_paths(x0, y0, th, v, tr, dt, T, scale):
    """Float32 states at steps 0 .. T-1 of rollouts that keep their heading (w = 0): per rollout a heading th[i], a speed
    sequence v[i] (float32, (N, T)), cos / sin scaled by scale[i] (1 +- 2e-6: the approximate MUFU functions)."""
    c32 = (np.cos(th.astype(F32)).astype(F32).astype(F64) * scale).astype(F32).astype(F64)
    s32 = (np.sin(th.astype(F32)).astype(F32).astype(F64) * scale).astype(F32).astype(F64)
    dv = (F64(tr) * F64(F32(dt))) * v.astype(F64)                # (vtr * dt64) * v, as the rollout kernels
    N = len(th)
    xs, ys = np.empty((T, N), F32), np.empty((T, N), F32)
    x, y = np.full(N, F32(x0)), np.full(N, F32(y0))
    for t in range(T):
        xs[t], ys[t] = x, y
        x = (dv[:, t] * c32 + x.astype(F64)).astype(F32)
        y = (dv[:, t] * s32 + y.astype(F64)).astype(F32)
    return xs, ys


def reach_ru(v):
    """The prepare kernel's reach statistic of speed sequences (N, T): sum_t |v| with round-up float32 adds, max over n."""
    s = np.zeros(v.shape[0], F32)
    for t in range(v.shape[1]):
        a = np.abs(v[:, t]).astype(F32)
        r = (s + a).astype(F32)
        bb = (r - s).astype(F32)
        err = ((s - (r - bb).astype(F32)).astype(F32) + (a - bb).astype(F32)).astype(F32)      # TwoSum: exact error
        s = np.where(err > 0, np.nextafter(r, F32(np.inf)), r).astype(F32)
    return float(s.max())


def check_reads(out, outf, xs, ys, res, pxl, pyl, tag):
    """Every cell read lies in box rows x box columns and within the disc (sampler's `need` region)."""
    how, r0, r1, c0, c1 = out
    if how == 0:
        return 0
    ci = MR.floor_div_f32((xs - F32(pxl)).astype(F32), F32(res)).astype(np.int64)
    ri = MR.floor_div_f32((ys - F32(pyl)).astype(F32), F32(res)).astype(np.int64)
    cx, cy, rad = outf
    dxc = np.maximum(np.maximum(ci - cx, cx - (ci + 1)), 0.0)
    dyc = np.maximum(np.maximum(ri - cy, cy - (ri + 1)), 0.0)
    ok = (ri >= r0) & (ri < r1) & (ci >= c0) & (ci < c1) & (dxc ** 2 + dyc ** 2 <= rad ** 2)
    if not ok.all():
        t, n = np.argwhere(~ok)[0]
        raise AssertionError("%s: %d of %d reads outside the sampled region; first: step %d rollout %d cell (row %d, "
                             "col %d), box rows [%d, %d) cols [%d, %d), disc (%.2f, %.2f) r %.2f"
                             % (tag, int((~ok).sum()), ok.size, t, n, ri[t, n], ci[t, n], r0, r1, c0, c1, cx, cy, rad))
    return 1


def drift_allowance(T, R, x, y, pxl, pyl):
    """First-order float32 rounding term of the reach: T state roundings of at most 2^-24 |x| and one of x - xlo."""
    return U * (T * (abs(x) + abs(y) + 2 * R) + abs(x - pxl) + abs(y - pyl) + 2 * R) * 1.001


def check_tight(out, T, R, x, y, pxl, pyl, res, tag):
    side = 2 * (R + drift_allowance(T, R, x, y, pxl, pyl)) / res + 8
    assert out[2] - out[1] <= side and out[4] - out[3] <= side, (tag, out, side)


HEADINGS = [0.0, np.pi / 2, np.pi, -np.pi / 2, np.pi / 4, 3 * np.pi / 4]
TS = (1, 16, 64, 512, 1024)
RESS = (0.01, 0.05, 0.1, 1.0)
ORIGINS = [0.0, 100.0, -100.0, 4096.0, 65536.0, 4.0e5, -65536.0, -4.0e5]
STEPS = [0.51, 0.61, 1.01, 1.49, 1.51, "ordinary"]


def run_family(decide, origin, step, sign, tr=1.0, trm=None, dt=0.1):
    """One family: map corner at `origin` (both axes), start `off` metres inside, per-step displacement `step` ulps of the
    start coordinate (or 1 cm), driving forward (sign 1) or in reverse (-1), for every heading, MUFU scale, resolution and
    horizon.  Mode 1 (static bound) over all rollouts, mode 2 (reach statistic) over those below the speed limit."""
    trm = abs(tr) if trm is None else trm
    Tm = max(TS)
    off = 6.0
    for _ in range(3):                                       # the start's ulp sets the speed, the speed the room needed
        x0 = F32(origin + off)
        ulp = float(np.spacing(abs(x0)))
        d = 0.01 if step == "ordinary" else step * ulp      # metres per step along the heading
        need = 1.2 * Tm * (d + 2 * ulp) + 5.0
        if off >= need:
            break
        off = need
    vmax = F32(d / (dt * abs(tr)))
    vr = (F32(-vmax), F32(-0.5 * vmax)) if sign < 0 else (F32(0.5 * vmax), vmax)
    heads = list(HEADINGS)
    if step != "ordinary" and step > 0.55:                  # a heading whose cosine puts the x displacement just above
        heads.append(float(np.arccos(0.51 / step)))          # half an ulp (the y one at sin = sqrt(1 - cos^2) ulp)
    th, scale = [], []
    for h in heads:
        for s in (1.0, 1 + 2e-6, 1 - 2e-6):
            th.append(h)
            scale.append(s)
    th, scale = np.array(th), np.array(scale)
    N = len(th)
    rng = np.random.default_rng(int(abs(origin)) % 1000 + (7 if sign < 0 else 0))
    v_lim = np.full((N, Tm), F32(sign * vmax), F32)                                     # at the clip limit
    v_in = (sign * vmax * rng.uniform(0.9, 0.99, (N, Tm))).astype(F32)                  # just below it
    paths = [straight_paths(x0, x0, th, v, tr, dt, Tm, scale) for v in (v_lim, v_in)]
    stats = dict(boxed=0, checked=0)
    for res in RESS:
        pxl = F32(origin)
        cols = int(np.ceil(2 * off / res)) + 8
        for T in TS:
            S = T * float(vmax)
            R = dt * trm * S * 1.0002
            for mode, which in ((1, (0, 1)), (2, (1,))):
                for k in which:
                    xs, ys = paths[k][0][:T], paths[k][1][:T]
                    reach = reach_ru(v_in[:, :T]) if mode == 2 else None
                    out, outf = decide(mode, T, cols, cols, vr, dt, trm, res, pxl, pxl, x0, x0, reach)
                    tag = "origin %g step %s sign %d res %g T %d mode %d %s" % (origin, step, sign, res, T, mode,
                                                                              ("limit", "inside")[k])
                    assert out[0] == mode, tag + ": not boxed"     # the map holds the reach with room to spare
                    stats["checked"] += check_reads(out, outf, xs, ys, res, pxl, pxl, tag)
                    check_tight(out, T, R, float(x0), float(x0), float(pxl), float(pxl), res, tag)
                    stats["boxed"] += 1
    return stats


@pytest.mark.parametrize("step", STEPS)
@pytest.mark.parametrize("origin", ORIGINS)
def test_straight_rollouts_read_only_sampled_cells(decide, origin, step):
    st = run_family(decide, origin, step, 1)
    assert st["checked"] == st["boxed"] == len(RESS) * len(TS) * 3


@pytest.mark.parametrize("origin", [0.0, 4096.0, 4.0e5, -65536.0])
def test_reverse_driving_and_negative_traction(decide, origin):
    """Negative vrange (reverse), and a traction of -0.9 from bounds [-1, 1] (|traction| up to 1): the rollouts move
    backwards along their heading."""
    run_family(decide, origin, 1.51, -1)
    tr = -1.0 + 0.01 * F64(F32(2.0)) * 5                    # byte 5 of bounds [-1, 1], as the rollout kernels decode it
    run_family(decide, origin, 0.61, 1, tr=tr, trm=1.0)
    run_family(decide, origin, 1.01, -1, tr=tr, trm=1.0)


@pytest.mark.parametrize("case", ["4096-north", "4096-east", "utm-north"])
def test_far_origin_cases(decide, case):
    """The georeferenced cases: a map at 4096 m at 1 cm (x0 1.2 m inside, 0.61 ulp per step, T 512) heading north and
    east, and one at 4e5 m at 10 cm (T 64, 0.54 ulp per step).  Exact motion 0.154 m / 1.09 m, float32 motion up to twice
    that."""
    if case.startswith("4096"):
        origin, res, T, vr, pad, cells, inside = 4096.0, 0.01, 512, (F32(0.0025), F32(0.003)), 50, 256, 1.2
    else:                                                    # the rounding drift (3 m) needs a larger map for a box
        origin, res, T, vr, pad, cells, inside = 4.0e5, 0.1, 64, (F32(0.16), F32(0.17)), 5, 128, 5.0
    th = np.pi / 2 if case.endswith("north") else 0.0
    dt = 0.1
    pxl = F32(origin - pad * res)
    cols = cells + 2 * pad
    x0 = F32(origin + inside)
    heads, scale = np.array([th, th]), np.array([1.0, 1 + 2e-6])
    for mode, v in ((1, vr[1]), (2, F32(0.97 * vr[1]))):       # mode 2: just below the limit (the statistic stays under it)
        vs = np.full((2, T), v, F32)
        xs, ys = straight_paths(x0, x0, heads, vs, 1.0, dt, T, scale)
        moved = float(np.abs((ys if th else xs)[-1] - x0).max())
        assert moved > 1.4 * dt * T * float(v)               # float32 rounding: the robot outruns its exact path
        out, outf = decide(mode, T, cols, cols, vr, dt, 1.0, res, pxl, pxl, x0, x0, reach_ru(vs) if mode == 2 else None)
        assert out[0] == mode, (case, out)
        check_reads(out, outf, xs, ys, res, pxl, pxl, "%s mode %d" % (case, mode))
        check_tight(out, T, dt * T * float(vr[1]) * 1.0002, float(x0), float(x0), float(pxl), float(pxl), res, case)


def test_whole_maps_pass_trivially(decide):
    """A box that would leave the map is not used: whole maps (how 0), nothing to check."""
    out, _ = decide(1, 64, 40, 40, (0.0, 3.0), 0.1, 1.0, 0.1, 0.0, 0.0, 2.0, 2.0)
    assert out == [0, 0, 40, 0, 40]
