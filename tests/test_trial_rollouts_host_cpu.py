"""Visualisation rollouts of batches and recording trials without a GPU: the C-ABI of b200mppi_batch_get_state_rollout
and b200mppi_batch_run_trials_recorded (prototypes as the header declares them, the ctypes bindings, arguments refused
without a device), and the Python layer on a fake backend -- MPPI_Batch.get_state_rollout and record_every of every
trial call: the arguments passed, the shapes returned, the NaN records kept, record_every=None making today's call with
today's keys, and every refusal naming its planner and issuing nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.fake_backend import disarm
from tests.test_batch_host_cpu import BatchFake, barebone_planner, det_planner
from tests.test_stochastic_batch_host_cpu import planner as tdm_planner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLAIN_KEYS = {"logs", "xhist", "uhist", "steps", "status"}
ISSUED = ("planner_set_params", "batch_run", "batch_get")     # what a refused call must not have made


def test_abi(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    src = tmp_path / "proto.c"
    src.write_text('#include "b200mppi.h"\n'
                   "int (*f)(b200mppi_batch*, float*, size_t) = b200mppi_batch_get_state_rollout;\n"
                   "int (*g)(b200mppi_batch*, int32_t, const b200mppi_trial_desc*, int32_t, double*, float*, "
                   "b200mppi_trial_result*, int32_t*, int32_t, float*, size_t, int32_t*) = "
                   "b200mppi_batch_run_trials_recorded;\n"
                   "int kinds[3] = {B200MPPI_TRIALS_MAP, B200MPPI_TRIALS_STOCHASTIC, B200MPPI_TRIALS_BAREBONE};\n")
    r = subprocess.run(["gcc", "-c", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                        str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert (_lib.TRIALS_MAP, _lib.TRIALS_STOCHASTIC, _lib.TRIALS_BAREBONE) == (0, 1, 2)
    L = _lib.lib
    assert len(L.b200mppi_batch_get_state_rollout.argtypes) == 3
    assert len(L.b200mppi_batch_run_trials_recorded.argtypes) == 12
    assert L.b200mppi_batch_get_state_rollout(None, None, 0) == -1
    assert "null batch" in L.b200mppi_last_error().decode()
    res = (_lib.TrialResult * 1)()
    assert L.b200mppi_batch_run_trials_recorded(None, 0, None, 5, None, None, res, None, 1, None, 0, None) == -1
    assert "null batch" in L.b200mppi_last_error().decode()


class RecFake(BatchFake):
    """Plays both batch constructors, the three plain trial calls (planner k runs k + 1 steps), the recorded call (the
    same, plus record r of planner k filled with 100 k + r, NaN from step k + 1 on) and the batched get_state_rollout
    (out[k] filled with k)."""

    def b200mppi_batch_create_stochastic(self, arr, n, out):
        return self.b200mppi_batch_create(arr, n, out)

    def _play(self, name, descs, max_steps, xh, uh, res, issued):
        K = len(self.members)
        self.calls.append((name, (K, max_steps)))
        xa = np.ctypeslib.as_array(C.cast(xh, C.POINTER(C.c_double)), (K, max_steps + 1, 3))
        ua = np.ctypeslib.as_array(C.cast(uh, C.POINTER(C.c_float)), (K, max_steps, 2))
        for k in range(K):
            n = k + 1
            xa[k], ua[k] = np.nan, np.nan
            xa[k, :n + 1] = [[t, k, 0.5 * t] for t in range(n + 1)]
            ua[k, :n] = [[t, -k] for t in range(n)]
            res[k].cum_obj, res[k].cum_dist_to_goal, res[k].dist_to_goal = 10.0 + k, 2.0 * k, 1.5 + k
            res[k].steps, res[k].status = n, 2
        C.cast(issued, C.POINTER(C.c_int32))[0] = K
        return 0

    def b200mppi_batch_run_trials(self, h, descs, max_steps, xh, uh, res, issued):
        return self._play("batch_run_trials", descs, max_steps, xh, uh, res, issued)

    def b200mppi_batch_run_stochastic_trials(self, h, descs, max_steps, xh, uh, res, issued):
        return self._play("batch_run_stochastic_trials", descs, max_steps, xh, uh, res, issued)

    def b200mppi_batch_run_barebone_trials(self, h, descs, max_steps, xh, uh, res, contacts, issued):
        return self._play("batch_run_barebone_trials", descs, max_steps, xh, uh, res, issued)

    def b200mppi_batch_run_trials_recorded(self, h, kind, descs, max_steps, xh, uh, res, contacts, every, ro, nbytes,
                                           issued):
        K = len(self.members)
        self.recorded = dict(kind=kind, every=every, nbytes=nbytes, contacts=contacts is not None)
        self._play("batch_run_trials_recorded", descs, max_steps, xh, uh, res, issued)
        R = -(-max_steps // every)
        V = nbytes // (4 * K * R * (self.T + 1) * 3)
        ra = np.ctypeslib.as_array(C.cast(ro, C.POINTER(C.c_float)), (K, R, V, self.T + 1, 3))
        for k in range(K):
            for r in range(R):
                ra[k, r] = 100 * k + r if r * every < k + 1 else np.nan
        return 0

    def b200mppi_batch_get_state_rollout(self, h, out, nbytes):
        K = len(self.members)
        self.calls.append(("batch_get_state_rollout", (K, nbytes)))
        a = np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_float)), (nbytes // 4,)).reshape(K, -1)
        a[:] = np.arange(K, dtype=np.float32)[:, None]
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
    fake = RecFake()
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    made = []
    for cls in (BT.MPPI_Batch, BT.MPPI_StochasticBatch):
        def init(self, planners, real=cls.__init__):
            made.append(self)
            real(self, planners)
        monkeypatch.setattr(cls, "__init__", init)
    yield E, fake
    for b in made:                                   # fake handles must never reach the real destroy function
        b._handle = None
    disarm(fake)


class Grid:
    """A ground-truth grid as run_trials reads it."""
    lin_traction = np.ones((20, 20))
    ang_traction = np.ones((20, 20))
    xlimits, ylimits, res = (0.0, 5.0), (0.0, 5.0), 0.25


def make(E, kind, k, **cfg):
    if kind == "barebone":
        return barebone_planner(k)
    return tdm_planner(E, k, **cfg) if kind == "tdm" else det_planner(E, k, mode=kind, **cfg)


def call(E, kind, pls, max_steps, **kw):
    if kind == "tdm":
        return E.MPPI_StochasticBatch(pls).run_stochastic_trials([Grid()] * len(pls), max_steps, **kw)
    batch = E.MPPI_Batch(pls)
    if kind == "barebone":
        return batch.run_barebone_trials(max_steps, **kw)
    return batch.run_trials([Grid()] * len(pls), max_steps, **kw)


@pytest.mark.parametrize("kind, code", [("det", 0), ("spd", 0), ("tdm", 1), ("barebone", 2)])
def test_record_marshalling_and_shapes(host, kind, code):
    E, fake = host
    pls = [make(E, kind, k) for k in range(3)]
    K, V, T = 3, pls[0].num_vis_state_rollouts, pls[0].num_steps
    fake.T = T
    fake.pods.clear()
    out = call(E, kind, pls, 7, record_every=3)
    assert fake.recorded == dict(kind=code, every=3, nbytes=K * 3 * V * (T + 1) * 3 * 4, contacts=(kind == "barebone"))
    names = fake.names()
    assert "batch_run_trials_recorded" in names and len(fake.pods) == K        # every planner's params uploaded first
    assert names.index("batch_run_trials_recorded") > max(i for i, n in enumerate(names) if n == "planner_set_params")
    assert set(out) == PLAIN_KEYS | {"state_rollouts", "rollout_steps"} | ({"contact_steps"} if kind == "barebone" else set())
    rec = out["state_rollouts"]
    assert rec.dtype == np.float32 and rec.shape == (K, 3, V, T + 1, 3)
    assert out["rollout_steps"].tolist() == [0, 3, 6]
    for k in range(K):                               # planner k ran k + 1 steps: records r with 3 r <= k
        for r in range(3):
            assert (rec[k, r] == 100 * k + r).all() if 3 * r <= k else np.isnan(rec[k, r]).all()
    assert out["steps"].tolist() == [1, 2, 3]


@pytest.mark.parametrize("kind", ["det", "tdm", "barebone"])
def test_no_recording_makes_todays_call(host, kind):
    E, fake = host
    pls = [make(E, kind, k) for k in range(2)]
    out = call(E, kind, pls, 4)
    assert set(out) == PLAIN_KEYS | ({"contact_steps"} if kind == "barebone" else set())
    names = fake.names()
    assert "batch_run_trials_recorded" not in names
    assert names[-1] == {"det": "batch_run_trials", "tdm": "batch_run_stochastic_trials",
                         "barebone": "batch_run_barebone_trials"}[kind]


def test_refusals_issue_nothing(host, capsys):
    E, fake = host
    for kind in ("det", "tdm", "barebone"):
        pls = [make(E, kind, k) for k in range(3)]
        for bad in (0, -2):
            n = len(fake.calls)
            with pytest.raises(ValueError, match="record_every %d < 1" % bad):
                call(E, kind, pls, 5, record_every=bad)
            assert [c for c in fake.calls[n:] if c[0].startswith(ISSUED)] == []
    pls = [make(E, "tdm", 0), make(E, "tdm", 1), make(E, "tdm", 2, num_vis_state_rollouts=5)]
    assert [p.num_vis_state_rollouts for p in pls] == [8, 8, 5]
    n = len(fake.calls)
    with pytest.raises(ValueError, match="planner 2 has num_vis_state_rollouts 5, planner 0 8"):
        call(E, "tdm", pls, 5, record_every=2)
    batch = E.MPPI_StochasticBatch(pls)
    with pytest.raises(ValueError, match="get_state_rollout: planner 2 has num_vis_state_rollouts 5, planner 0 8"):
        batch.get_state_rollout()
    pls = [make(E, "det", k) for k in range(3)]
    batch = E.MPPI_Batch(pls)
    pls[1].params_set = False
    with pytest.raises(ValueError, match="planner 1: MPPI parameters are not set"):
        batch.get_state_rollout()
    assert [c for c in fake.calls[n:] if c[0].startswith(ISSUED)] == []


@pytest.mark.parametrize("kind", ["det", "tdm", "barebone"])
def test_batch_get_state_rollout(host, kind):
    E, fake = host
    pls = [make(E, kind, k) for k in range(3)]
    batch = E.MPPI_StochasticBatch(pls) if kind == "tdm" else E.MPPI_Batch(pls)
    V, T = pls[0].num_vis_state_rollouts, pls[0].num_steps
    fake.pods.clear()
    out = batch.get_state_rollout()
    assert out.dtype == np.float32 and out.shape == (3, V, T + 1, 3)
    assert fake.calls[-1] == ("batch_get_state_rollout", (3, out.nbytes))
    assert len(fake.pods) == 3                       # every planner's params uploaded before the one call
    for k in range(3):
        assert (out[k] == k).all()
