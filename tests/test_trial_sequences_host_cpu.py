"""Trial sequences without a GPU: the C-ABI of b200mppi_batch_run_trial_sequences (prototype and NOT_RUN against the
ctypes mirrors, refusals of the C entry point), and run_trial_sequences on a fake backend: marshalling of the per-slot
descriptors, output shapes and NaN padding, logs (None for an episode that did not run), params['x0'] afterwards and
every refusal issuing nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.fake_backend import disarm
from tests.test_batch_host_cpu import BatchFake, barebone_planner, det_planner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sequence_abi_matches_ctypes(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    assert "b200mppi_batch_run_trial_sequences" in _lib.EXPORTS
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include "b200mppi.h"\n'
                   "int (*f)(b200mppi_batch*, int32_t, const b200mppi_trial_desc*, const int32_t*, int32_t, int32_t, "
                   "double*, float*, b200mppi_trial_result*, int32_t*) = b200mppi_batch_run_trial_sequences;\n"
                   'int main(void) { printf("%d\\n", B200MPPI_TRIAL_NOT_RUN); return 0; }\n')
    exe = tmp_path / "abi"
    r = subprocess.run(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                        "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)], capture_output=True, text=True).stdout.strip() == str(_lib.TRIAL_NOT_RUN)
    fn = _lib.lib.b200mppi_batch_run_trial_sequences
    assert fn.restype is C.c_int and len(fn.argtypes) == 10
    assert fn.argtypes[2] is C.POINTER(_lib.TrialDesc) and fn.argtypes[8] is C.POINTER(_lib.TrialResult)


def test_library_refusals_before_any_work():
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    L = _lib.lib
    res = (_lib.TrialResult * 1)()
    E = (C.c_int32 * 1)(1)
    assert L.b200mppi_batch_run_trial_sequences(None, _lib.TRIALS_MAP, None, E, 5, 0, None, None, res, None) == -1
    assert "null batch" in L.b200mppi_last_error().decode()


class SeqFake(BatchFake):
    """Plays b200mppi_batch_run_trial_sequences: episode e of planner k runs k + e + 1 steps (xhist row t = (t, k, e),
    u = (t, -e)) and ends goal, except planner 2's episode 0 ends left_map (later episodes not_run without reset_x0)."""

    def b200mppi_batch_run_trial_sequences(self, h, kind, descs, episodes, max_steps, reset_x0, xh, uh, res, issued):
        K = len(self.members)
        E = np.ctypeslib.as_array(C.cast(episodes, C.POINTER(C.c_int32)), (K,)).copy()
        slots = int(E.sum())
        self.seq = dict(kind=kind, episodes=E.tolist(), max_steps=max_steps, reset_x0=reset_x0,
                        x0=[list(descs[j].x0) for j in range(slots)], dt=[descs[j].dt for j in range(slots)],
                        xlo=[descs[j].xlo for j in range(slots)])
        self.calls.append(("batch_run_trial_sequences", (K, max_steps)))
        xa = np.ctypeslib.as_array(C.cast(xh, C.POINTER(C.c_double)), (slots, max_steps + 1, 3))
        ua = np.ctypeslib.as_array(C.cast(uh, C.POINTER(C.c_float)), (slots, max_steps, 2))
        xa[:], ua[:] = np.nan, np.nan
        j = 0
        for k in range(K):
            stop = False
            for e in range(E[k]):
                r = res[j]
                if stop:
                    r.steps, r.status = 0, 4
                else:
                    n = k + e + 1
                    xa[j, :n + 1] = [[t, k, e] for t in range(n + 1)]
                    ua[j, :n] = [[t, -e] for t in range(n)]
                    left = k == 2 and e == 0
                    r.cum_obj, r.cum_dist_to_goal, r.dist_to_goal = 1.0 + e, 0.5 * n, (2.0 if left else -0.1)
                    r.steps, r.status = n, (3 if left else 1)
                    stop = left and not reset_x0
                j += 1
        C.cast(issued, C.POINTER(C.c_int32))[0] = 9
        return 0


@pytest.fixture()
def seqs(monkeypatch):
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    import mppi_numba_b200.barebone as B
    import mppi_numba_b200.batch as BT
    import mppi_numba_b200.mppi as M
    import mppi_numba_b200.terrain as T
    fake = SeqFake()
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    made = []
    real_create = BT.MPPI_Batch._create

    def create(self, *a):
        made.append(self)
        real_create(self, *a)
    monkeypatch.setattr(BT.MPPI_Batch, "_create", create)
    yield E, fake
    for b in made:                                   # fake handles must never reach the real destroy function
        b._handle = None
    disarm(fake)


def grids(E, n, seed=0):
    rng = np.random.default_rng(seed)
    return [E.TractionGrid(rng.uniform(0, 1, (5, 7)), rng.uniform(0, 1, (5, 7)), res=0.5, xlimits=(-1.0 - i, 2.5))
            for i in range(n)]


@pytest.mark.parametrize("reset_x0", [False, True])
def test_marshalling_outputs_logs_and_x0(seqs, reset_x0):
    E, fake = seqs
    pls = [det_planner(E, k) for k in range(3)]
    batch = E.MPPI_Batch(pls)
    x0s = [p.params["x0"].copy() for p in pls]
    eps = [1, 2, 3]
    out = batch.run_trial_sequences([grids(E, n, k) for k, n in enumerate(eps)], 8, dt=0.05, reset_x0=reset_x0)
    s = fake.seq
    assert s["kind"] == 0 and s["episodes"] == eps and s["max_steps"] == 8 and s["reset_x0"] == int(reset_x0)
    assert s["x0"] == [[float(v) for v in x0s[k]] for k, n in enumerate(eps) for _ in range(n)]
    assert s["dt"] == [0.05] * 6 and s["xlo"] == [-1.0, -1.0, -2.0, -1.0, -2.0, -3.0]
    assert out["xhist"].shape == (3, 3, 9, 3) and out["xhist"].dtype == np.float64
    assert out["uhist"].shape == (3, 3, 8, 2) and out["uhist"].dtype == np.float32
    assert batch.steps_issued == 9
    want_run = [1, 2, 3 if reset_x0 else 1]
    assert out["episodes_run"].tolist() == want_run
    for k, n in enumerate(eps):
        run = want_run[k]
        assert len(out["logs"][k]) == len(out["status"][k]) == n
        assert out["status"][k][run:] == ["not_run"] * (n - run) and out["logs"][k][run:] == [None] * (n - run)
        assert np.isnan(out["xhist"][k, run:]).all() and np.isnan(out["uhist"][k, run:]).all()
        assert (out["steps"][k, run:] == 0).all()
        for e in range(run):
            m = k + e + 1
            assert out["steps"][k, e] == m
            assert np.array_equal(out["xhist"][k, e, :m + 1], [[t, k, e] for t in range(m + 1)])
            assert np.isnan(out["xhist"][k, e, m + 1:]).all() and np.isnan(out["uhist"][k, e, m:]).all()
            log = out["logs"][k][e]
            if k == 2 and e == 0:
                assert out["status"][k][e] == "left_map" and log["success"] is False
                assert log["cum_obj"] == 1.0 + 2.0 / pls[k].params["v_post_rollout"]
            else:
                assert out["status"][k][e] == "goal" and log["success"] is True and np.isnan(log["dist_to_goal"])
                assert log["time_to_goal"] == m * 0.05 and log["cum_obj"] == 1.0 + e
            assert log["avg_dist_to_goal"] == 0.5
        last = run - 1
        assert np.array_equal(pls[k].params["x0"], [k + last + 1, k, last]) and pls[k].params["x0"].dtype == np.float64
        assert pls[k].u_prev_d is pls[k]._u_prev_buf
    names = fake.names()
    assert names.index("batch_run_trial_sequences") > max(i for i, n in enumerate(names) if n == "planner_set_params")


def test_refusals_issue_nothing(seqs, capsys):
    E, fake = seqs
    pls = [det_planner(E, k) for k in range(3)]
    batch = E.MPPI_Batch(pls)
    g = grids(E, 2)
    with pytest.raises(ValueError, match="2 lists of traction grids for 3 planners"):
        batch.run_trial_sequences([g, g], 5)
    with pytest.raises(ValueError, match="planner 1: empty list of traction grids"):
        batch.run_trial_sequences([g, [], g], 5)
    with pytest.raises(ValueError, match="max_steps 0 < 1"):
        batch.run_trial_sequences([g] * 3, 0)
    pls[1].params["num_opt"] = 0
    with pytest.raises(ValueError, match="planner 1 has num_opt 0 < 1"):
        batch.run_trial_sequences([g] * 3, 5)
    pls[1].params["num_opt"] = 1
    pls[2].params["x0"] = np.array([-50.0, 0.0, 0.0])
    with pytest.raises(ValueError, match="planner 2 cannot solve"):
        batch.run_trial_sequences([g] * 3, 5)
    assert "not within padded xlimits" in capsys.readouterr().out
    pls[2].params["x0"] = pls[0].params["x0"].copy()
    g32 = E.TractionGrid(np.ones((4, 4), np.float32), np.ones((4, 4), np.float32))
    with pytest.raises(ValueError, match="planner 1, episode 1: traction grid of dtype float32"):
        batch.run_trial_sequences([g, [g[0], g32], g], 5)
    with pytest.raises(ValueError, match="planner 0 is a barebone planner"):
        E.MPPI_Batch([barebone_planner(0), barebone_planner(1)]).run_trial_sequences([g, g], 5)
    assert "batch_run_trial_sequences" not in fake.names()
