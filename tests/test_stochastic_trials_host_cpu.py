"""Closed-loop trials of stochastic batches without a GPU: the C-ABI entry point (export, prototype as the header declares
it, argument errors before any device work), MPPI_StochasticBatch.run_stochastic_trials on a fake backend (marshalling,
logs and NaN conventions, refusals issuing nothing, run_trials still refused), and the shared host / device helpers
compiled from the header's text for the host: the reach-box decision against a host restatement of it (the decision
solve() made before it was shared, with the float32 rounding terms of reach_radius), and the window origin against
fill_win_args' former code."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import emu_core, emu_trial
from tests.fake_backend import disarm
from tests.test_stochastic_batch_host_cpu import StochasticFake, planner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "b200mppi_batch_run_stochastic_trials"


def test_entry_point_exported_with_header_prototype(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    assert hasattr(C.CDLL(_lib.LIB_PATH), NAME) and NAME in _lib.EXPORTS
    src = tmp_path / "proto.c"
    src.write_text('#include "b200mppi.h"\n'
                   "int (*f)(b200mppi_batch*, const b200mppi_trial_desc*, int32_t, double*, float*, "
                   "b200mppi_trial_result*, int32_t*) = %s;\n" % NAME)
    r = subprocess.run(["gcc", "-c", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                        str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    fn = getattr(_lib.lib, NAME)
    assert fn.restype is C.c_int and len(fn.argtypes) == 7
    res = (_lib.TrialResult * 1)()
    assert fn(None, None, 5, None, None, res, None) == -1
    assert "null batch" in _lib.lib.b200mppi_last_error().decode()


class TrialFake(StochasticFake):
    """Plays the entry point: planner k runs k + 1 steps (xhist row t = (t, k, 0.5 t), u = (t, -k)) and ends with status
    (goal, max_steps, left_map)[k % 3]."""

    def b200mppi_batch_run_stochastic_trials(self, h, descs, max_steps, xh, uh, res, issued):
        K = len(self.members)
        self.trials = [{f: (list(getattr(descs[i], f)) if hasattr(getattr(descs[i], f), "__len__") else
                            getattr(descs[i], f)) for f, _ in descs[i]._fields_} for i in range(K)]
        self.calls.append(("batch_run_stochastic_trials", (K, max_steps)))
        xa = np.ctypeslib.as_array(C.cast(xh, C.POINTER(C.c_double)), (K, max_steps + 1, 3))
        ua = np.ctypeslib.as_array(C.cast(uh, C.POINTER(C.c_float)), (K, max_steps, 2))
        for k in range(K):
            n = k + 1
            xa[k] = np.nan
            ua[k] = np.nan
            xa[k, :n + 1] = [[t, k, 0.5 * t] for t in range(n + 1)]
            ua[k, :n] = [[t, -k] for t in range(n)]
            r = res[k]
            r.cum_obj, r.cum_dist_to_goal, r.dist_to_goal = 10.0 + k, 2.0 * k, (-0.1 if k % 3 == 0 else 1.5 + k)
            r.steps, r.status = n, (1, 2, 3)[k % 3]
        C.cast(issued, C.POINTER(C.c_int32))[0] = K
        return 0


@pytest.fixture()
def host(monkeypatch):
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    import mppi_numba_b200.barebone as B
    import mppi_numba_b200.batch as BT
    import mppi_numba_b200.mppi as M
    import mppi_numba_b200.terrain as T
    fake = TrialFake()
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    made = []
    real = BT.MPPI_StochasticBatch.__init__

    def init(self, planners):
        made.append(self)
        real(self, planners)
    monkeypatch.setattr(BT.MPPI_StochasticBatch, "__init__", init)
    yield E, fake
    for b in made:                                   # fake handles must never reach the real destroy function
        b._handle = None
    disarm(fake)


def test_marshalling_logs_and_nan_padding(host):
    E, fake = host
    pls = [planner(E, k) for k in range(3)]
    prev = [p.u_prev_d for p in pls]
    batch = E.MPPI_StochasticBatch(pls)
    rng = np.random.default_rng(0)
    grids = [E.TractionGrid(rng.uniform(0, 1, (5, 7)), rng.uniform(0, 1, (5, 7)), res=0.5, xlimits=(-1.0, 2.5)),
             E.TractionGrid(rng.uniform(0, 1, (5, 7)), rng.uniform(0, 1, (5, 7)), use_int8=True),
             E.TractionGrid(rng.uniform(0, 1, (4, 4)), rng.uniform(0, 1, (4, 4)), res=0.25)]
    x0s = [p.params["x0"].copy() for p in pls]
    out = batch.run_stochastic_trials(grids, 6, dt=0.05)
    t = fake.trials
    assert [tr["x0"] for tr in t] == [[float(v) for v in x] for x in x0s]
    assert t[0]["xlo"] == -1.0 and t[0]["res"] == 0.5 and (t[0]["height"], t[0]["width"]) == (5, 7)
    for k, p in enumerate(pls):
        assert t[k]["dt"] == 0.05 and t[k]["pylim"] == [float(v) for v in p.lin_tdm.padded_ylimits]
        assert p.u_prev_d is prev[k]                  # a stochastic solve leaves u_prev_d alone
        assert np.array_equal(p.params["x0"], [k + 1, k, 0.5 * (k + 1)])
    assert out["steps"].tolist() == [1, 2, 3] and out["status"] == ["goal", "max_steps", "left_map"]
    assert np.isnan(out["xhist"][0, 2:]).all() and np.isnan(out["uhist"][1, 2:]).all()
    L = out["logs"]
    assert L[0]["success"] is True and np.isnan(L[0]["dist_to_goal"]) and L[0]["time_to_goal"] == 0.05
    assert L[2]["success"] is False and L[2]["cum_obj"] == 12.0 + 3.5 / pls[2].params["v_post_rollout"]
    names = fake.names()
    assert names.index("batch_run_stochastic_trials") > max(i for i, n in enumerate(names) if n == "planner_set_params")
    assert batch.steps_issued == 3


def test_refusals_issue_nothing(host, capsys):
    E, fake = host
    pls = [planner(E, k) for k in range(3)]
    batch = E.MPPI_StochasticBatch(pls)
    g = E.TractionGrid(np.ones((4, 4)), np.ones((4, 4)))
    with pytest.raises(ValueError, match="MPPI_StochasticBatch.run_trials: closed-loop trials run det-dynamics or "
                                         "speed-map.*run_stochastic_trials"):
        batch.run_trials([g] * 3, 5)
    with pytest.raises(ValueError, match="run_stochastic_trials: 2 traction grids for 3 planners"):
        batch.run_stochastic_trials([g, g], 5)
    with pytest.raises(ValueError, match="max_steps 0 < 1"):
        batch.run_stochastic_trials([g] * 3, 0)
    pls[1].params["num_opt"] = 0
    with pytest.raises(ValueError, match="planner 1 has num_opt 0 < 1"):
        batch.run_stochastic_trials([g] * 3, 5)
    pls[1].params["num_opt"] = 1
    pls[2].params["x0"] = np.array([-50.0, 0.0, 0.0])
    with pytest.raises(ValueError, match="planner 2 cannot solve"):
        batch.run_stochastic_trials([g] * 3, 5)
    pls[2].params["x0"] = pls[0].params["x0"].copy()
    g32 = E.TractionGrid(np.ones((4, 4), np.float32), np.ones((4, 4), np.float32))
    with pytest.raises(ValueError, match="planner 1: traction grid of dtype float32"):
        batch.run_stochastic_trials([g, g32, g], 5)
    assert "batch_run_stochastic_trials" not in fake.names()


# ------------------------------------------------------------------------------------------- shared helpers, emulated
HARNESS = r'''
extern "C" int emu_decide(const int* ci, const float* cf, float x, float y, const float* reach, int* out, float* outf) {
  using namespace b200;
  ReachBoxConst c{};
  c.mode = ci[0]; c.disc = ci[1]; c.T = ci[2]; c.rows = ci[3]; c.cols = ci[4];
  c.nt = ci[5]; c.tx = ci[6]; c.ty = ci[7]; c.num_maps = ci[8]; c.bpad0 = ci[9]; c.bpad1 = ci[10];
  c.vr0 = cf[0]; c.vr1 = cf[1]; c.dt = cf[2]; c.tr_abs_max = cf[3]; c.res = cf[4]; c.pxl = cf[5]; c.pyl = cf[6];
  ReachBox b;
  const int how = reach_box_decide(c, x, y, reach, &b);
  const int v[11] = {how, b.geo, b.how, b.row_lo, b.row_hi, b.col_lo, b.col_hi, b.tiy_lo, b.nact, b.gm, 0};
  for (int i = 0; i < 11; ++i) out[i] = v[i];
  outf[0] = b.cx; outf[1] = b.cy; outf[2] = b.r;
  return how;
}
extern "C" void emu_win(float x, float y, float pxl, float pyl, float res, int cols, int rows, int* f) {
  b200::win_origin(x, y, pxl, pyl, res, cols, rows, f);
}
'''


@pytest.fixture(scope="module")
def helpers(tmp_path_factory):
    return emu_core.build(str(tmp_path_factory.mktemp("helpers")), "helpers",
                          [emu_core.region("kernels.h", "sampler_args"), emu_core.region("kernels.h", "trial_args")],
                          HARNESS)


def host_decision(ci, cf, x, y, reach):
    """planner_reach_box, apply_box and sample_grids_v2_fits as sample_finish combined them before the decision was
    shared with the device, R widened by the float32 rounding of the state and of the cell index (reach_radius):
    (last_box 5-tuple, disc) -- Python floats are IEEE doubles, float32 via numpy."""
    mode, disc, T, rows, cols, nt, tx, ty, M, bp0, bp1 = ci
    vr0, vr1, dt, trm, res, pxl, pyl = [float(np.float32(v)) for v in cf]
    whole = ((0, 0, rows, 0, cols), None)
    if mode == 0:
        return whole
    S = float(T) * max(abs(vr0), abs(vr1))
    how = 1
    if reach is not None:
        if not float(np.float32(reach)) <= S:
            return whole
        S, how = float(np.float32(reach)), 2
    # plus the float32 rounding of the state (T steps, at most 2^-24 |x| each) and of the cell index (reach_radius)
    u = 5.9605e-8
    Tu = T * u
    R0 = dt * trm * S * 1.0002
    if not Tu < 0.5 or not R0 >= 0.0:
        return whole
    D = (R0 + Tu * (abs(x) + abs(y))) / (1.0 - Tu)
    R = D + u * ((abs(x - pxl) + abs(y - pyl)) + 2.0 * D)
    if not (R >= 0.0) or not np.isfinite(R):
        return whole
    fx0, fx1 = (x - R - pxl) / res, (x + R - pxl) / res
    fy0, fy1 = (y - R - pyl) / res, (y + R - pyl) / res
    if not (fx0 > 2.0 and fy0 > 2.0 and fx1 < cols - 3.0 and fy1 < rows - 3.0):
        return whole
    box = (int(np.floor(fy0)) - 1, int(np.floor(fy1)) + 3, int(np.floor(fx0)) - 1, int(np.floor(fx1)) + 3)
    dsc = (np.float32((x - pxl) / res), np.float32((y - pyl) / res),
           np.float32(np.float32(R / res + 3.0) * np.float32(1.0001)) if disc else np.float32(0))
    ncol = (cols + ty - 1) // ty
    tiy_lo = box[2] // ncol
    nact = (box[3] - 1) // ncol - tiy_lo + 1
    gm = max(1, min(128 // nact, 32, M))
    cfirst = min(tiy_lo * ncol, cols)
    wcols = min((tiy_lo + nact) * ncol, cols) - (cfirst & ~15)
    smem = nt * ((wcols * bp0 + 15) & ~15) + max(nt * gm * ((wcols + 15) & ~15), 4096) + 2048 + nt * 128
    fits = (nt > 0 and 1 <= gm <= 32 and nact >= 1 and tiy_lo >= 0 and tiy_lo + nact <= ty and
            (nact * gm + 31) // 32 * 32 <= 256 and bp0 <= 32 and smem <= 200 * 1024 and (nt == 1 or bp0 == bp1))
    return ((how,) + box, dsc) if fits else whole


def test_box_decision_matches_host_restatement(helpers):
    rng = np.random.default_rng(7)
    cases, far_boxed = 0, 0
    for mode in (0, 1, 2):
        for disc in (0, 1):
            for (rows, cols, res, pxl, pyl, ty, M, nt, bp) in [(512, 512, 0.1, -0.8, -0.8, 16, 64, 2, 12),
                                                               (100, 130, 0.25, -1.0, 0.5, 8, 24, 1, 32),
                                                               (13, 13, 1.0, -2.0, -2.0, 4, 1024, 2, 12),
                                                               (300, 40, 0.2, 0.0, 0.0, 2, 8, 0, 12),
                                                               # georeferenced: the rounding terms are metres here
                                                               (2000, 2000, 0.1, 4.0e5, -4.0e5, 64, 64, 1, 12)]:
                T, vr, dt, trm = 64, (-1.0, 2.5), 0.1, 1.27
                ci = [mode, disc, T, rows, cols, nt, 8, ty, M, bp, bp]
                cf = [vr[0], vr[1], dt, trm, res, pxl, pyl]
                S = T * 2.5
                xs = np.concatenate([[pxl - 3 * res, pxl, pxl + 2.5 * res, pxl + cols * res - res / 2,
                                      pxl + cols * res, pxl + cols * res * 0.5],
                                     pxl + rng.uniform(-0.1, 1.1, 10) * cols * res]).astype(np.float32)
                ys = np.concatenate([[pyl - res, pyl + rows * res - 0.3 * res, pyl + rows * res * 0.5],
                                     pyl + rng.uniform(-0.1, 1.1, 6) * rows * res]).astype(np.float32)
                for reach in (None, 0.0, 3.7, S * 0.4, S, S * 1.001, float("nan")):
                    for x in xs:
                        for y in ys:
                            out, outf = (C.c_int * 11)(), (C.c_float * 3)()
                            r = None if reach is None else C.c_float(reach)
                            helpers.emu_decide((C.c_int * 11)(*ci), (C.c_float * 7)(*cf), float(x), float(y),
                                               None if r is None else C.byref(r), out, outf)
                            last, dsc = host_decision(ci, cf, float(x), float(y), reach)
                            got = (out[0],) + tuple(out[3:7]) if out[0] else (0, 0, rows, 0, cols)
                            assert got == last, (ci, cf, x, y, reach, got, last)
                            if out[0]:
                                assert (np.float32(outf[0]), np.float32(outf[1]), np.float32(outf[2])) == dsc
                                far_boxed += abs(pxl) > 1000
                            cases += 1
    assert cases > 10000 and far_boxed > 100, (cases, far_boxed)


def test_window_origin_matches_fill_win_args(helpers):
    rng = np.random.default_rng(3)
    for (rows, cols, res, pxl) in [(512, 512, 0.1, -0.8), (13, 13, 1.0, -2.0), (200, 90, 0.25, 1.5), (300, 700, 0.2, 0)]:
        for WW, WH in ((256, 232), (256, 224)):
            for x, y in rng.uniform(-0.2, 1.2, (40, 2)) * np.array([cols, rows]) * res + pxl:
                x, y = np.float32(x), np.float32(y)
                f = (C.c_int * 6)(WW, WH, 0, 0, 0, 0)
                helpers.emu_win(float(x), float(y), pxl, pxl, res, cols, rows, f)
                xi0 = int(np.floor((float(x) - float(np.float32(pxl))) / float(np.float32(res))))
                yi0 = int(np.floor((float(y) - float(np.float32(pxl))) / float(np.float32(res))))
                cx = max(0, min(xi0 - WW // 2, cols - WW))
                cy = max(0, min(yi0 - WH // 2, rows - WH))
                wx0 = cx & ~15
                assert list(f) == [WW, WH, wx0, cy, min(WW, cols - wx0), min(WH, rows - cy)]


PLANT_HARNESS = r'''
// one plant step of one planner on a uniform grid (traction lt, at) from pose x; win = {WW, WH, wx0, wy0, ww, wh} of its
// RolloutWinArgs, recomputed by the kernel over a map of rows x cols cells at res from (pxl, pyl)
extern "C" void emu_plant_win(const double* x, float v, float w, double lt, double at, double dt, float pxl, float pyl,
                              float res, int rows, int cols, int* win, float* x0_out) {
  using namespace b200;
  const double lin[1] = {lt}, ang[1] = {at};
  float u[4] = {v, w, 0.0f, 0.0f};
  TrialDev d{};
  d.lin = lin; d.ang = ang; d.H = 1; d.W = 1; d.xlo = -1e6; d.ylo = -1e6; d.res = 2e6; d.dt = dt;
  d.xgoal[0] = 1e9; d.xgoal[1] = 1e9; d.tol = 0.0; d.pxlim[0] = d.pylim[0] = -1e9; d.pxlim[1] = d.pylim[1] = 1e9;
  d.u_cur = u; d.x0_out = x0_out;
  d.win = win; d.win_pxl = pxl; d.win_pyl = pyl; d.win_res = res; d.win_rows = rows; d.win_cols = cols;
  TrialState st{};
  for (int c = 0; c < 3; ++c) st.x[c] = x[c];
  int active = 1, count = 1;
  double xh[6];
  float uh[2];
  PlantArgs a{&d, &st, &active, &count, xh, uh, 1, 2, 1, 0};
  emu::launch({1, 1, 1}, 32, [&] { plant_step_body(a, 0, (int)threadIdx.x); });
}
'''


def test_plant_step_window_matches_fill_win_args(tmp_path):
    """The window fields the plant step writes into a stochastic planner's RolloutWinArgs (TrialDev::win) against
    fill_win_args' former computation from the float32 x0 it wrote, including maps smaller than one window."""
    lib = emu_trial.build(str(tmp_path), extra=PLANT_HARNESS)
    rng = np.random.default_rng(5)
    for (rows, cols, res, pxl, pyl) in [(512, 512, 0.1, -0.8, -0.8), (9, 9, 1.0, -2.0, -2.0), (200, 90, 0.25, 1.5, 0.0),
                                         (300, 700, 0.2, 0.0, -3.0)]:
        for WW, WH in ((256, 232), (256, 224)):
            for _ in range(30):
                x = np.array([pxl + rng.uniform(-0.2, 1.2) * cols * res, pyl + rng.uniform(-0.2, 1.2) * rows * res,
                              rng.uniform(-3, 3)])
                win = np.array([WW, WH, -1, -1, -1, -1], dtype=np.int32)
                x0 = np.zeros(3, dtype=np.float32)
                lib.emu_plant_win(x.ctypes.data, 1.5, -0.3, 0.8, 0.9, 0.1, pxl, pyl, res, rows, cols, win.ctypes.data,
                                  x0.ctypes.data)
                f32 = lambda v: float(np.float32(v))                                   # noqa: E731
                xi0 = int(np.floor((float(x0[0]) - f32(pxl)) / f32(res)))
                yi0 = int(np.floor((float(x0[1]) - f32(pyl)) / f32(res)))
                cx = max(0, min(xi0 - WW // 2, cols - WW))
                cy = max(0, min(yi0 - WH // 2, rows - WH))
                wx0 = cx & ~15
                assert list(win) == [WW, WH, wx0, cy, min(WW, cols - wx0), min(WH, rows - cy)]
