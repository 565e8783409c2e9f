"""Recorded and barebone trial sequences without a GPU: the C-ABI of b200mppi_batch_run_trial_sequences_ex against the
ctypes mirror and its refusals, and run_trial_sequences(record_every=n) / run_barebone_trial_sequences on a fake
backend: the arguments handed to the library, the records returned in the (K, Emax, ...) layout the library writes, the
per-slot contact counts spread to (K, Emax) with 0 where no episode exists, logs, the caller's order of a mixed batch, unrecorded sequences
still going through b200mppi_batch_run_trial_sequences, and every refusal issuing nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.fake_backend import disarm
from tests.test_batch_host_cpu import barebone_planner, det_planner
from tests.test_mixed_batch_host_cpu import KINDS, ORDER, MixedFake

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_matches_ctypes(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    assert "b200mppi_batch_run_trial_sequences_ex" in _lib.EXPORTS
    src = tmp_path / "abi.c"
    src.write_text('#include "b200mppi.h"\n'
                   "int (*f)(b200mppi_batch*, int32_t, const b200mppi_trial_desc*, const int32_t*, int32_t, int32_t, "
                   "double*, float*, b200mppi_trial_result*, int32_t*, int32_t, float*, size_t, int32_t*) = "
                   "b200mppi_batch_run_trial_sequences_ex;\nint main(void) { return 0; }\n")
    r = subprocess.run(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "abi"),
                        "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    fn = _lib.lib.b200mppi_batch_run_trial_sequences_ex
    assert fn.restype is C.c_int and len(fn.argtypes) == 14
    assert fn.argtypes[2] is C.POINTER(_lib.TrialDesc) and fn.argtypes[8] is C.POINTER(_lib.TrialResult)
    assert fn.argtypes[12] is C.c_size_t


def test_library_refusals_before_any_work():
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    L = _lib.lib
    res = (_lib.TrialResult * 1)()
    E = (C.c_int32 * 1)(1)
    args = (None, None, res, None, 0, None, 0, None)
    assert L.b200mppi_batch_run_trial_sequences_ex(None, _lib.TRIALS_MAP, None, E, 5, 0, *args) == -1
    assert "null batch" in L.b200mppi_last_error().decode()


def _arr(p, ctype, shape):
    addr = p.value if isinstance(p, C.c_void_p) else C.cast(p, C.c_void_p).value
    return np.ctypeslib.as_array(C.cast(addr, C.POINTER(ctype)), shape)


class ExFake(MixedFake):
    """Plays b200mppi_batch_run_trial_sequences_ex: slot j runs j % 3 + 2 steps and ends max_steps; contacts[j] =
    10 + j; the records of slot j that the library writes hold 100 j + r at (planner, episode), the rest NaN (as the
    library fills them)."""
    V = None

    def b200mppi_batch_run_trial_sequences_ex(self, h, kind, descs, episodes, max_steps, reset_x0, xh, uh, res,
                                              contacts, every, recs, nbytes, issued):
        K = len(self.members)
        E = _arr(episodes, C.c_int32, (K,)).copy()
        slots = int(E.sum())
        self.ex = dict(kind=kind, episodes=E.tolist(), max_steps=max_steps, reset_x0=reset_x0, every=every,
                       nbytes=nbytes, contacts=contacts is not None, recs=recs is not None,
                       x0=[list(descs[j].x0) for j in range(slots)], dt=[descs[j].dt for j in range(slots)])
        self.calls.append(("batch_run_trial_sequences_ex", (K, max_steps)))
        xa = _arr(xh, C.c_double, (slots, max_steps + 1, 3))
        xa[:] = np.nan
        for j in range(slots):
            n = j % 3 + 2
            xa[j, :n + 1] = j
            res[j].steps, res[j].status, res[j].cum_dist_to_goal, res[j].dist_to_goal = n, 2, 1.0, 0.5
        if contacts is not None:
            _arr(contacts, C.c_int32, (slots,))[:] = 10 + np.arange(slots)
        if recs is not None:                          # (K, Emax, R, ...): slot first[k] + e at (k, e)
            R, Emax = -(-max_steps // every), int(E.max())
            per = nbytes // (4 * K * Emax * R)
            ra = _arr(recs, C.c_float, (K, Emax, R, per))
            ra[:] = np.nan
            first = np.concatenate([[0], np.cumsum(E)])
            for k in range(K):
                for e in range(E[k]):
                    j = first[k] + e
                    for r in range(-(-(j % 3 + 2) // every)):
                        ra[k, e, r] = 100 * j + r
        C.cast(issued, C.POINTER(C.c_int32))[0] = 7
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
    fake = ExFake()
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    made = []
    real_create = BT.MPPI_Batch._create

    def create(self, *a):
        made.append(self)
        return real_create(self, *a)
    monkeypatch.setattr(BT.MPPI_Batch, "_create", create)
    yield E, fake
    for b in made:                                   # fake handles must never reach the real destroy function
        b._handle = None
    disarm(fake)


def grids(E, n, seed=0):
    rng = np.random.default_rng(seed)
    return [E.TractionGrid(rng.uniform(0.2, 1.0, (20, 20)), rng.uniform(0.2, 1.0, (20, 20)), res=0.25)
            for _ in range(n)]


def check_records(out, first, eps, every, S, V, T):
    R = -(-S // every)
    rec = out["state_rollouts"]
    assert rec.dtype == np.float32 and rec.shape == (len(eps), max(eps), R, V, T + 1, 3)
    assert out["rollout_steps"].tolist() == [r * every for r in range(R)]
    for k, n in enumerate(eps):
        assert np.isnan(rec[k, n:]).all()           # episodes that do not exist
        for e in range(n):
            j = first[k] + e
            done = -(-(j % 3 + 2) // every)
            for r in range(done):
                assert (rec[k, e, r] == 100 * j + r).all()
            assert np.isnan(rec[k, e, done:]).all()


@pytest.mark.parametrize("every", [1, 3, 50])
def test_recorded_sequence_marshalling(host, every):
    E, fake = host
    pls = [det_planner(E, k) for k in range(3)]
    V, T = int(pls[0].num_vis_state_rollouts), pls[0].num_steps
    batch = E.MPPI_Batch(pls)
    eps, S = [1, 3, 2], 8
    out = batch.run_trial_sequences([grids(E, n, k) for k, n in enumerate(eps)], S, reset_x0=True, record_every=every)
    R = -(-S // every)
    x = fake.ex
    assert x["kind"] == E._lib.TRIALS_MAP and x["episodes"] == eps and x["every"] == every and x["reset_x0"] == 1
    assert x["nbytes"] == 3 * 3 * R * V * (T + 1) * 3 * 4 and x["recs"] and not x["contacts"]   # (K, Emax, R, ...)
    assert batch.steps_issued == 7 and "batch_run_trial_sequences" not in fake.names()
    check_records(out, [0, 1, 4], eps, every, S, V, T)
    assert out["xhist"].shape == (3, 3, S + 1, 3) and "contact_steps" not in out
    # without recording: the call b200mppi_batch_run_trial_sequences always took
    fake.calls.clear()
    out = batch.run_trial_sequences([grids(E, 1, k) for k in range(3)], S)
    assert "batch_run_trial_sequences" in fake.names() and "batch_run_trial_sequences_ex" not in fake.names()
    assert "state_rollouts" not in out and "rollout_steps" not in out


def test_mixed_records_in_callers_order(host):
    E, fake = host
    P = [det_planner(E, k, mode=m) for k, m in enumerate(KINDS)]
    V, T = int(P[0].num_vis_state_rollouts), P[0].num_steps
    b = E.MPPI_MixedBatch(P)
    out = b.run_trial_sequences([[g] for g in grids(E, len(P))], 5, record_every=2)
    assert fake.ex["kind"] == E._lib.TRIALS_MIXED
    for j, i in enumerate(ORDER):                    # batch-order slot j is caller planner ORDER[j]'s
        done = -(-(j % 3 + 2) // 2)
        assert (out["state_rollouts"][i, 0, :done] == 100 * j + np.arange(done)[:, None, None, None]).all()
        assert out["steps"][i, 0] == j % 3 + 2
    assert out["state_rollouts"].shape == (len(P), 1, 3, V, T + 1, 3)
    with pytest.raises(ValueError, match="MPPI_MixedBatch.run_barebone_trial_sequences: a mixed batch holds no"):
        b.run_barebone_trial_sequences(2, 5)


@pytest.mark.parametrize("record", [None, 2])
def test_barebone_sequences(host, record):
    E, fake = host
    pls = [barebone_planner(k) for k in range(3)]
    x0s = [p.params["x0"].copy() for p in pls]
    batch = E.MPPI_Batch(pls)
    out = batch.run_barebone_trial_sequences([2, 1, 3], 6, dt=0.05, record_every=record)
    x = fake.ex
    assert x["kind"] == E._lib.TRIALS_BAREBONE and x["episodes"] == [2, 1, 3] and x["contacts"]
    assert x["every"] == (record or 0) and x["recs"] == (record is not None)
    assert x["x0"] == [[float(v) for v in x0s[k]] for k, n in enumerate([2, 1, 3]) for _ in range(n)]
    assert x["dt"] == [0.05] * 6
    first = [0, 2, 3]
    want = np.zeros((3, 3), np.int64)
    for k, n in enumerate([2, 1, 3]):
        want[k, :n] = 10 + first[k] + np.arange(n)
        for e in range(n):
            log = out["logs"][k][e]
            assert log["contact_steps"] == want[k, e] and "cum_obj" not in log
        assert out["status"][k] == ["max_steps"] * n and out["episodes_run"][k] == n
    assert out["contact_steps"].tolist() == want.tolist()
    if record:
        check_records(out, first, [2, 1, 3], record, 6, int(pls[0].num_vis_state_rollouts), pls[0].num_steps)
    out = batch.run_barebone_trial_sequences(4, 6)
    assert fake.ex["episodes"] == [4, 4, 4] and out["contact_steps"].shape == (3, 4)


def test_refusals_issue_nothing(host):
    E, fake = host
    pls = [det_planner(E, k) for k in range(3)]
    batch = E.MPPI_Batch(pls)
    g = grids(E, 2)
    with pytest.raises(ValueError, match="MPPI_Batch.run_trial_sequences: record_every 0 < 1"):
        batch.run_trial_sequences([g] * 3, 5, record_every=0)
    other = det_planner(E, 2)
    other.num_vis_state_rollouts = 3
    odd = E.MPPI_Batch(pls[:2] + [other])
    with pytest.raises(ValueError, match="planner 2 has num_vis_state_rollouts 3"):
        odd.run_trial_sequences([g] * 3, 5, record_every=2)
    with pytest.raises(ValueError, match="run_barebone_trial_sequences: planner 0 is a det planner"):
        batch.run_barebone_trial_sequences(2, 5)
    bb = E.MPPI_Batch([barebone_planner(0), barebone_planner(1)])
    with pytest.raises(ValueError, match="run_trial_sequences: planner 0 is a barebone planner"):
        bb.run_trial_sequences([g, g], 5, record_every=2)
    with pytest.raises(ValueError, match="planner 1: episode count 0 < 1"):
        bb.run_barebone_trial_sequences([2, 0], 5)
    with pytest.raises(ValueError, match="3 episode counts for 2 planners"):
        bb.run_barebone_trial_sequences([2, 2, 2], 5)
    with pytest.raises(ValueError, match="max_steps 0 < 1"):
        bb.run_barebone_trial_sequences(2, 0)
    with pytest.raises(ValueError, match="record_every -1 < 1"):
        bb.run_barebone_trial_sequences(2, 5, record_every=-1)
    with pytest.raises(ValueError, match="planner 0, episode 0: dt 0.0 not finite and positive"):
        bb.run_barebone_trial_sequences(1, 5, dt=0.0)
    assert "batch_run_trial_sequences_ex" not in fake.names() and "batch_run_trial_sequences" not in fake.names()
