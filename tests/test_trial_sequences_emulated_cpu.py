"""The sequence variant of the plant-step kernel (csrc/reduce.cu, ``plant_step_body<true>``) emulated on the host against
a numpy model of the trial-sequence loop, step by step and bit for bit: episode boundaries on goal, max_steps and
left_map with and without reset_x0, ragged episode counts (1, 2, 5), one-step episodes, the not_run tail, per-slot
history offsets, x0_out and the rollout window after a boundary, the running count and stopped planners."""
import ctypes as C

import numpy as np
import pytest

from mppi_numba_b200.terrain import TractionGrid
from tests import emu_trial
from tests.trial_loop import plant_step

GOAL, MAX_STEPS, LEFT_MAP, NOT_RUN = 1, 2, 3, 4
WIN = dict(pxl=-0.8, pyl=-0.6, res=0.2, rows=40, cols=48, WW=16, WH=12)

SEQ_HARNESS = r'''
// slots: descriptors g[11 j ..] as emu_plant's, grids lin[j] / ang[j]; planner i: u_cur[i], x0_out[i], win[i] (may be
// null; window map wf = pxl, pyl, res and wi = rows, cols)
extern "C" void emu_plant_seq(int K, int T, int max_steps, int slots, const double** lin, const double** ang,
                              const int* H, const int* W, const double* g, float** u_cur, float** x0_out, int** win,
                              const float* wf, const int* wi, void* state, int* active, int* count, double* xhist,
                              float* uhist, const int* first, int* episode, const double* start, void* results,
                              int reset_x0) {
  std::vector<TrialDev> d(slots);
  for (int i = 0; i < K; ++i)
    for (int j = first[i]; j < first[i + 1]; ++j) {
      const double* q = g + 11 * j;
      d[j] = TrialDev{lin[j], ang[j], H[j], W[j], q[0], q[1], q[2], q[3], {q[4], q[5]}, q[6], {q[7], q[8]},
                      {q[9], q[10]}, u_cur[i], x0_out[i], win[i], wf[0], wf[1], wf[2], wi[0], wi[1]};
    }
  PlantArgs a{d.data(), reinterpret_cast<TrialState*>(state), active, count, xhist, uhist, K, T, max_steps, -1};
  SeqArgs q{first, episode, start, reinterpret_cast<TrialState*>(results), reset_x0};
  emu::launch({(unsigned)K, 1, 1}, 32, [&] { plant_step_body<true>(a, (int)blockIdx.x, (int)threadIdx.x, q); });
}
'''


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_trial.build(str(tmp_path_factory.mktemp("trial_seq_emu")), extra=SEQ_HARNESS)


def f32(v):
    return float(np.float32(v))


def window(x0):
    """win_origin of the float32 pose x0 (kernels.h): {WW, WH, wx0, wy0, ww, wh}."""
    w = WIN
    xi0 = int(np.floor((float(x0[0]) - f32(w["pxl"])) / f32(w["res"])))
    yi0 = int(np.floor((float(x0[1]) - f32(w["pyl"])) / f32(w["res"])))
    cx = max(0, min(xi0 - w["WW"] // 2, w["cols"] - w["WW"]))
    cy = max(0, min(yi0 - w["WH"] // 2, w["rows"] - w["WH"]))
    wx0 = cx & ~15
    return [w["WW"], w["WH"], wx0, cy, min(w["WW"], w["cols"] - wx0), min(w["WH"], w["rows"] - cy)]


def grid(seed, n=12, res=0.5):
    rng = np.random.default_rng(seed)
    return TractionGrid(rng.uniform(0.2, 1.0, (n, n)), rng.uniform(0.2, 1.0, (n, n)), res=res)


def episode(seed, start, kind):
    """One episode's descriptor: 'goal' within a step (large tolerance), 'max' goal out of reach, 'left' padded limits
    the first step leaves."""
    start = np.asarray(start, dtype=np.float64)
    d = dict(grid=grid(seed), start=start, dt=0.1 + 0.01 * (seed % 3), xgoal=start[:2] + 40.0, tol=0.25,
             pxlim=(-5.0, 10.0), pylim=(-5.0, 10.0))
    if kind == "goal":
        d.update(xgoal=start[:2] + 0.05, tol=0.5)
    elif kind == "left":
        d.update(pxlim=(start[0] - 1e-3, start[0] + 1e-3))
    return d


# ragged sequences: E = 1, 2, 5, 2 (planner 3 is stopped before the call and must be left alone)
def sequences():
    s0, s1, s2, s3 = [1.0, 2.0, 0.3], [2.5, 1.5, -0.7], [3.0, 3.0, 1.1], [1.5, 1.0, 0.0]
    return [[episode(1, s0, "goal")],
            [episode(2, s1, "max"), episode(3, s1, "goal")],
            [episode(4, s2, "goal"), episode(5, s2, "left"), episode(6, s2, "max"), episode(7, s2, "goal"),
             episode(8, s2, "left")],
            [episode(9, s3, "max"), episode(10, s3, "goal")]]


class Model(object):
    """numpy restatement of the sequence loop of one planner."""

    def __init__(self, eps, u, reset_x0, max_steps):
        self.eps, self.u, self.reset, self.S = eps, u.copy(), reset_x0, max_steps
        self.e, self.x, self.cum, self.steps, self.active, self.status = 0, eps[0]["start"].copy(), [0.0, 0.0], 0, 1, 0
        self.dist = 0.0
        self.results = [None] * len(eps)
        self.xh = np.full((len(eps), max_steps + 1, 3), -7.0)
        self.uh = np.full((len(eps), max_steps, 2), -7.0, dtype=np.float32)
        self.x0 = None

    def step(self):
        d, t = self.eps[self.e], self.steps
        u0 = self.u[0].copy()
        self.u[:-1] = self.u[1:].copy()
        xn = plant_step(d["grid"], self.x, u0, d["dt"])
        self.uh[self.e, t] = u0
        self.xh[self.e, t + 1] = xn
        self.x0 = xn.astype(np.float32)
        dx, dy = xn[0] - d["xgoal"][0], xn[1] - d["xgoal"][1]
        dist = np.sqrt(dx * dx + dy * dy) - d["tol"]
        self.cum = [self.cum[0] + (d["dt"] + dist), self.cum[1] + dist]
        self.x, self.dist, self.steps = xn, dist, t + 1
        if dist <= 0:
            status = GOAL
        elif not (d["pxlim"][0] <= xn[0] <= d["pxlim"][1] and d["pylim"][0] <= xn[1] <= d["pylim"][1]):
            status = LEFT_MAP
        elif t + 1 >= self.S:
            status = MAX_STEPS
        else:
            return
        self.results[self.e] = (self.cum[0], self.cum[1], dist, self.steps, status)
        if self.e + 1 < len(self.eps) and (self.reset or status != LEFT_MAP):
            self.e += 1
            self.x, self.cum, self.dist, self.steps = self.eps[self.e]["start"].copy(), [0.0, 0.0], 0.0, 0
            if self.reset:
                self.x0 = self.x.astype(np.float32)
            return
        self.active, self.status = 0, status


def run(emu, seqs, reset_x0, max_steps, stopped=(3,)):
    K, T = len(seqs), 6
    eps = [e for s in seqs for e in s]
    first = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int32)
    slots = int(first[-1])
    lin = [np.ascontiguousarray(e["grid"].lin_traction, dtype=np.float64) for e in eps]
    ang = [np.ascontiguousarray(e["grid"].ang_traction, dtype=np.float64) for e in eps]
    g = np.array([[e["grid"].xlimits[0], e["grid"].ylimits[0], e["grid"].res, e["dt"], e["xgoal"][0], e["xgoal"][1],
                   e["tol"], e["pxlim"][0], e["pxlim"][1], e["pylim"][0], e["pylim"][1]] for e in eps])
    start = np.array([e["start"] for e in eps], dtype=np.float64)
    rng = np.random.default_rng(3)
    us = [rng.uniform(-1.5, 1.5, (T, 2)).astype(np.float32) for _ in range(K)]
    models = [Model(s, u, reset_x0, max_steps) for s, u in zip(seqs, us)]
    u = [x.copy() for x in us]
    x0 = [np.full(3, -9.0, np.float32) for _ in range(K)]
    win = [np.array([WIN["WW"], WIN["WH"], -1, -1, -1, -1], np.int32) if k % 2 == 0 else None for k in range(K)]
    wf = np.array([WIN["pxl"], WIN["pyl"], WIN["res"]], np.float32)
    wi = np.array([WIN["rows"], WIN["cols"]], np.int32)
    state = np.zeros((K, 7))
    state[:, :3] = [s[0]["start"] for s in seqs]
    results = np.zeros((slots, 7))
    results[:, 6] = np.array([[0, NOT_RUN]], np.int32).view(np.float64)[0, 0]
    active = np.ones(K, np.int32)
    for k in stopped:
        active[k] = 0
        models[k].active = 0
    count = np.array([K - len(stopped)], np.int32)
    episode_ = np.zeros(K, np.int32)
    xh = np.full((slots, max_steps + 1, 3), -7.0)
    uh = np.full((slots, max_steps, 2), -7.0, np.float32)
    P = lambda arrs: (C.c_void_p * len(arrs))(*[a.ctypes.data if a is not None else None for a in arrs])  # noqa: E731
    Hs = np.array([a.shape[0] for a in lin], np.int32)
    Ws = np.array([a.shape[1] for a in lin], np.int32)
    trace = []
    for s in range(max_steps * max(len(q) for q in seqs)):
        if count[0] == 0:
            break
        emu.emu_plant_seq(K, T, max_steps, slots, P(lin), P(ang), Hs.ctypes.data, Ws.ctypes.data, g.ctypes.data, P(u),
                          P(x0), P(win), wf.ctypes.data, wi.ctypes.data, state.ctypes.data, active.ctypes.data,
                          count.ctypes.data, xh.ctypes.data, uh.ctypes.data, first.ctypes.data, episode_.ctypes.data,
                          start.ctypes.data, results.ctypes.data, int(reset_x0))
        for k, m in enumerate(models):
            if m.active:
                m.step()
        for k, m in enumerate(models):                # after every step: the planner's whole state
            assert active[k] == m.active and episode_[k] == m.e, (s, k)
            assert np.array_equal(u[k], m.u), (s, k)
            if k in stopped:
                assert np.array_equal(x0[k], np.full(3, -9.0, np.float32)) and np.array_equal(state[k, :3], m.x)
                continue
            assert np.array_equal(state[k, :3], m.x) and list(state[k, 3:6]) == [m.cum[0], m.cum[1], m.dist], (s, k)
            ints = state[k, 6:7].view(np.int32)
            assert ints[0] == m.steps and ints[1] == m.status, (s, k, ints, m.steps)
            assert np.array_equal(x0[k], m.x0), (s, k, x0[k], m.x0)
            if win[k] is not None:
                assert list(win[k]) == window(x0[k]), (s, k)
        assert count[0] == sum(m.active for m in models)
        trace.append(int(count[0]))
    return dict(models=models, xh=xh, uh=uh, first=first, results=results, count=trace)


@pytest.mark.parametrize("reset_x0", [False, True])
def test_sequence_boundaries_match_model(emu, reset_x0):
    S = 4
    out = run(emu, sequences(), reset_x0, S)
    first, res = out["first"], out["results"]
    for k, m in enumerate(out["models"]):
        for e in range(len(m.eps)):
            j = first[k] + e
            ints = res[j, 6:7].view(np.int32)
            if m.results[e] is None:                  # never ran: NOT_RUN and untouched rows
                assert ints[1] == NOT_RUN and ints[0] == 0 and (out["xh"][j] == -7.0).all()
                assert (out["uh"][j] == -7.0).all()
                continue
            co, cd, d, n, st = m.results[e]
            assert list(res[j, :6][3:]) == [co, cd, d] and (ints[0], ints[1]) == (n, st), (k, e)
            # histories at the slot's own offset, rows past the episode's steps untouched
            assert np.array_equal(out["xh"][j, 1:n + 1], m.xh[e, 1:n + 1]) and (out["xh"][j, n + 1:] == -7.0).all()
            assert np.array_equal(out["uh"][j, :n], m.uh[e, :n]) and (out["uh"][j, n:] == -7.0).all()
            assert (out["xh"][j, 0] == -7.0).all()   # row 0 (the start) is the host's
    st = [[None if r is None else r[4] for r in m.results] for m in out["models"]]
    print(reset_x0, st)
    assert st[0] == [GOAL] and out["models"][0].results[0][3] == 1           # a one-step episode
    assert st[1] == [MAX_STEPS, GOAL]
    if reset_x0:                                      # left_map does not end the sequence
        assert st[2] == [GOAL, LEFT_MAP, MAX_STEPS, GOAL, LEFT_MAP]
    else:                                             # it does: the not_run tail
        assert st[2] == [GOAL, LEFT_MAP, None, None, None]
    assert st[3] == [None, None]                      # stopped before the call: left alone
    # the running count falls only when a sequence ends: planner 0 after step 1, planner 1 after its 2 episodes
    c = out["count"]
    assert c[0] == 2 and all(a >= b for a, b in zip(c, c[1:])) and c[-1] == 0
    ends = sorted(sum(r[3] for r in m.results if r is not None) for m in out["models"][:3])
    assert [c[n - 1] for n in ends] == [2, 1, 0]
