"""What the sequence plant step (csrc/reduce.cu, ``plant_step_body<true>``) adds for recorded and barebone trial
sequences, emulated on the host against a numpy restatement after every step: each planner's record flag (it runs, and
its next episode step is a multiple of n), the record pointer it writes into its visualisation descriptor (slot
first[k] + episode, record step / n) across episode boundaries and after its sequence ends, flags and pointers of
planners stopped before the call left alone, and barebone contact counts per slot."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_trial
from tests.barebone_trial_loop import in_contact
from tests.test_trial_sequences_emulated_cpu import NOT_RUN, Model, episode, sequences

REC_HARNESS = r'''
// as emu_plant_seq (tests/test_trial_sequences_emulated_cpu.py) without windows; lin[j] null: a barebone slot with
// obstacles obst[j] (nobs[j] rows); vis: K descriptors of rec_stride pointer slots, slot 0 the record pointer
extern "C" void emu_plant_seq_rec(int K, int T, int max_steps, int slots, const double** lin, const double** ang,
                                  const int* H, const int* W, const double* g, float** u_cur, float** x0_out,
                                  const float** obst, const int* nobs, void* state, int* active, int* count,
                                  double* xhist, float* uhist, const int* first, int* episode, const double* start,
                                  void* results, int reset_x0, int* contacts, int* rec_flag, void* vis, int rec_stride,
                                  float* rec, long long rec_per, int rec_every, int rec_R) {
  std::vector<TrialDev> d(slots);
  for (int i = 0; i < K; ++i)
    for (int j = first[i]; j < first[i + 1]; ++j) {
      const double* q = g + 11 * j;
      d[j] = TrialDev{lin[j], ang[j], H[j], W[j], q[0], q[1], q[2], q[3], {q[4], q[5]}, q[6], {q[7], q[8]},
                      {q[9], q[10]}, u_cur[i], x0_out[i]};
      d[j].obstacles = obst[j]; d[j].num_obstacles = nobs[j];
    }
  PlantArgs a{d.data(), reinterpret_cast<TrialState*>(state), active, count, xhist, uhist, K, T, max_steps, -1,
              contacts};
  SeqArgs q{first, episode, start, reinterpret_cast<TrialState*>(results), reset_x0};
  if (rec_flag) {
    q.rec_flag = rec_flag; q.rec_out = reinterpret_cast<float**>(vis); q.rec = rec; q.rec_per = rec_per;
    q.rec_every = rec_every; q.rec_R = rec_R; q.rec_stride = rec_stride;
  }
  emu::launch({(unsigned)K, 1, 1}, 32, [&] { plant_step_body<true>(a, (int)blockIdx.x, (int)threadIdx.x, q); });
}
'''

STRIDE = 8                                            # sizeof(VisBatchDesc) / sizeof(float*) on the device
PER = 5                                               # floats of one record (any size: only pointers are written)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_trial.build(str(tmp_path_factory.mktemp("trial_rec_emu")), extra=REC_HARNESS)


class Unit(object):
    """The barebone plant's traction: 1 everywhere (dt * 1.0 == dt), so tests/trial_loop.plant_step is its step."""
    xlimits, ylimits, res = (0.0, 1.0), (0.0, 1.0), 1.0

    def get(self, x, y):
        return 1.0, 1.0


def barebone_sequences():
    """Per planner its episodes on the unit plant, no padded limits; planner 1 drives through an obstacle."""
    out = []
    for k, (n, start) in enumerate([(3, [0.0, 0.0, 0.2]), (4, [1.0, -0.5, 0.0]), (1, [2.0, 2.0, 1.0]), (2, [0, 0, 0])]):
        eps = []
        for e in range(n):
            d = episode(20 + 5 * k + e, start, ["max", "goal"][(k + e) % 2])
            d.update(grid=Unit(), pxlim=(-np.inf, np.inf), pylim=(-np.inf, np.inf))
            eps.append(d)
        out.append(eps)
    return out


OBST = np.array([[1.0, -0.5, 0.6], [5.0, 5.0, 0.1]], np.float32)


def run(emu, seqs, reset_x0, max_steps, every, barebone=False, stopped=(3,)):
    K, T = len(seqs), 6
    eps = [e for s in seqs for e in s]
    first = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int32)
    slots = int(first[-1])
    R = -(-max_steps // every)
    if barebone:
        lin = ang = [None] * slots
        Hs = Ws = np.zeros(slots, np.int32)
    else:
        lin = [np.ascontiguousarray(e["grid"].lin_traction, dtype=np.float64) for e in eps]
        ang = [np.ascontiguousarray(e["grid"].ang_traction, dtype=np.float64) for e in eps]
        Hs = np.array([a.shape[0] for a in lin], np.int32)
        Ws = np.array([a.shape[1] for a in lin], np.int32)
    g = np.array([[e["grid"].xlimits[0], e["grid"].ylimits[0], e["grid"].res, e["dt"], e["xgoal"][0], e["xgoal"][1],
                   e["tol"], e["pxlim"][0], e["pxlim"][1], e["pylim"][0], e["pylim"][1]] for e in eps])
    obst = [OBST if barebone else None] * slots
    nobs = np.array([len(OBST) if barebone else 0] * slots, np.int32)
    start = np.array([e["start"] for e in eps], dtype=np.float64)
    rng = np.random.default_rng(5)
    us = [rng.uniform(-1.5, 1.5, (T, 2)).astype(np.float32) for _ in range(K)]
    models = [Model(s, u, reset_x0, max_steps) for s, u in zip(seqs, us)]
    u = [x.copy() for x in us]
    x0 = [np.zeros(3, np.float32) for _ in range(K)]
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
    xh = np.zeros((slots, max_steps + 1, 3))
    uh = np.zeros((slots, max_steps, 2), np.float32)
    contacts = np.zeros(slots, np.int32)
    rec = np.zeros(slots * R * PER, np.float32)
    base = rec.ctypes.data

    def at(slot, r):                                  # address of record r of a slot
        return base + ((slot * R + r) * PER) * 4
    # before step 0, as the driver sets them: every flag 1, every pointer at record 0 of the planner's first slot
    flag = np.ones(K, np.int32)
    vis = np.zeros((K, STRIDE), np.uint64)
    vis[:, 0] = [at(int(first[k]), 0) for k in range(K)]
    vis[:, 1:] = 0xabcdef
    want_flag, want_ptr = flag.copy(), vis[:, 0].copy()
    P = lambda arrs: (C.c_void_p * len(arrs))(*[a.ctypes.data if a is not None else None for a in arrs])  # noqa: E731
    for s in range(max_steps * max(len(q) for q in seqs)):
        if count[0] == 0:
            break
        emu.emu_plant_seq_rec(K, T, max_steps, slots, P(lin), P(ang), Hs.ctypes.data, Ws.ctypes.data, g.ctypes.data,
                              P(u), P(x0), P(obst), nobs.ctypes.data, state.ctypes.data, active.ctypes.data,
                              count.ctypes.data, xh.ctypes.data, uh.ctypes.data, first.ctypes.data,
                              episode_.ctypes.data, start.ctypes.data, results.ctypes.data, int(reset_x0),
                              contacts.ctypes.data, flag.ctypes.data, vis.ctypes.data, STRIDE, rec.ctypes.data, PER,
                              every, R)
        for k, m in enumerate(models):
            if not m.active:
                continue
            m.step()
            if m.active:                              # its next step: m.steps of episode m.e (0 after a boundary)
                want_flag[k] = m.steps % every == 0
                if want_flag[k]:
                    want_ptr[k] = at(int(first[k]) + m.e, m.steps // every)
            else:
                want_flag[k] = 0
        assert flag.tolist() == want_flag.tolist(), (s, flag, want_flag)
        assert vis[:, 0].tolist() == want_ptr.tolist(), s
        assert (vis[:, 1:] == 0xabcdef).all()
        assert count[0] == sum(m.active for m in models)
    return dict(models=models, xh=xh, first=first, contacts=contacts, results=results)


@pytest.mark.parametrize("every", [1, 2, 3, 50])
@pytest.mark.parametrize("reset_x0", [False, True])
def test_record_flags_and_pointers(emu, reset_x0, every):
    out = run(emu, sequences(), reset_x0, 4, every)
    m = out["models"]
    assert [r is None for r in m[2].results] == ([False] * 5 if reset_x0 else [False, False, True, True, True])


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("reset_x0", [False, True])
def test_barebone_contacts_per_slot(emu, reset_x0, every):
    S = 5
    seqs = barebone_sequences()
    out = run(emu, seqs, reset_x0, S, every, barebone=True)
    first, xh = out["first"], out["xh"]
    hit = 0
    for k, mod in enumerate(out["models"]):
        for e in range(len(seqs[k])):
            j = first[k] + e
            n = out["results"][j, 6:7].view(np.int32)[0]
            if k == 3:                                # stopped before the call: no episode ran
                assert n == 0 and out["contacts"][j] == 0
                continue
            assert mod.results[e] is not None and mod.results[e][3] == n   # every barebone episode runs
            want = sum(in_contact(xh[j, t + 1], OBST) for t in range(n))
            assert out["contacts"][j] == want, (k, e)
            hit += want
    assert hit > 0
