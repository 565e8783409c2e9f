"""Barebone closed-loop trials without a GPU: the C-ABI of b200mppi_batch_run_barebone_trials (prototype, the ctypes
binding, a null batch refused), and MPPI_Batch.run_barebone_trials on a fake backend -- the descriptors it passes, the
dt default and override, the logs built from the results, the state it leaves on the Python side, and every refusal,
each naming its planner and issuing nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.fake_backend import disarm
from tests.test_batch_host_cpu import BatchFake, barebone_planner, det_planner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_barebone_trial_abi(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    proto = tmp_path / "proto.c"
    proto.write_text('#include "b200mppi.h"\n'
                     "int (*f)(b200mppi_batch*, const b200mppi_trial_desc*, int32_t, double*, float*, "
                     "b200mppi_trial_result*, int32_t*, int32_t*) = b200mppi_batch_run_barebone_trials;\n")
    r = subprocess.run(["gcc", "-c", "-Werror", "-I", os.path.join(ROOT, "include"), str(proto), "-o",
                        str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    fn = _lib.lib.b200mppi_batch_run_barebone_trials
    assert fn.restype is C.c_int and len(fn.argtypes) == 8
    res = (_lib.TrialResult * 1)()
    assert fn(None, None, 5, None, None, res, None, None) == -1
    assert "null batch" in _lib.lib.b200mppi_last_error().decode()


class BareboneTrialFake(BatchFake):
    """Plays b200mppi_batch_run_barebone_trials: planner k runs k + 1 steps (xhist row t = (t, k, 0.5 t), u = (t, -k)),
    ends with status (goal, max_steps)[k % 2] and touched obstacles on 2 k steps."""

    def b200mppi_batch_run_barebone_trials(self, h, descs, max_steps, xh, uh, res, contacts, issued):
        K = len(self.members)
        self.trials = [{f: (list(getattr(descs[i], f)) if hasattr(getattr(descs[i], f), "__len__") else
                            getattr(descs[i], f)) for f, _ in descs[i]._fields_} for i in range(K)]
        self.calls.append(("batch_run_barebone_trials", (K, max_steps)))
        xa = np.ctypeslib.as_array(C.cast(xh, C.POINTER(C.c_double)), (K, max_steps + 1, 3))
        ua = np.ctypeslib.as_array(C.cast(uh, C.POINTER(C.c_float)), (K, max_steps, 2))
        ca = np.ctypeslib.as_array(C.cast(contacts, C.POINTER(C.c_int32)), (K,))
        for k in range(K):
            n = k + 1
            xa[k] = np.nan
            ua[k] = np.nan
            xa[k, :n + 1] = [[t, k, 0.5 * t] for t in range(n + 1)]
            ua[k, :n] = [[t, -k] for t in range(n)]
            r = res[k]
            r.cum_obj, r.cum_dist_to_goal, r.dist_to_goal = 10.0 + k, 2.0 * k, (-0.1 if k % 2 == 0 else 1.5 + k)
            r.steps, r.status = n, (1, 2)[k % 2]
            ca[k] = 2 * k
        C.cast(issued, C.POINTER(C.c_int32))[0] = K + 2
        return 0


@pytest.fixture()
def trials(monkeypatch):
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    import mppi_numba_b200.barebone as B
    import mppi_numba_b200.batch as BT
    import mppi_numba_b200.mppi as M
    import mppi_numba_b200.terrain as T
    fake = BareboneTrialFake()
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    made = []
    real_init = BT.MPPI_Batch.__init__

    def init(self, planners):
        made.append(self)
        real_init(self, planners)
    monkeypatch.setattr(BT.MPPI_Batch, "__init__", init)
    yield E, fake, BT
    for b in made:                                   # fake handles must never reach the real destroy function
        b._handle = None
    disarm(fake)


def with_obstacles(p):
    p.params["obstacle_positions"] = np.array([[5.0, 4.5], [2.0, 1.0]])
    p.params["obstacle_radius"] = np.array([1.5, 1.0])
    return p


def test_descriptors_logs_and_planner_state(trials):
    E, fake, BT = trials
    pls = [with_obstacles(barebone_planner(k)) for k in range(3)]
    pls[1].params["dt"] = 0.05
    batch = E.MPPI_Batch(pls)
    x0s = [np.asarray(p.params["x0"], dtype=np.float64).copy() for p in pls]
    out = batch.run_barebone_trials(6)
    t = fake.trials
    for k, p in enumerate(pls):
        assert t[k]["lin"] is None and t[k]["ang"] is None and t[k]["height"] == 0 and t[k]["width"] == 0
        assert t[k]["x0"] == [float(v) for v in x0s[k]]
        assert t[k]["xgoal"] == [float(v) for v in p.params["xgoal"]]
        assert t[k]["goal_tolerance"] == p.params["goal_tolerance"]
        assert t[k]["dt"] == float(p.params["dt"])                 # the default: each planner's own dt
        assert p.u_prev_d is p._u_prev_buf
        assert np.array_equal(p.params["x0"], [k + 1, k, 0.5 * (k + 1)]) and p.params["x0"].dtype == np.float64
    assert [t[k]["dt"] for k in range(3)] == [0.1, 0.05, 0.1]
    assert fake.uploads["set_obstacles"]["rad"].tolist() == [1.5, 1.0]
    names = fake.names()
    assert names.index("batch_run_barebone_trials") > max(i for i, n in enumerate(names) if n == "planner_set_params")
    assert names.index("batch_run_barebone_trials") > max(i for i, n in enumerate(names) if n == "planner_set_obstacles")
    assert out["steps"].tolist() == [1, 2, 3] and out["status"] == ["goal", "max_steps", "goal"]
    assert out["contact_steps"].tolist() == [0, 2, 4]
    assert np.isnan(out["xhist"][0, 2:]).all() and not np.isnan(out["xhist"][2, :4]).any()
    assert np.isnan(out["uhist"][1, 2:]).all() and out["uhist"].dtype == np.float32
    assert batch.steps_issued == 5
    L = out["logs"]
    for k in (0, 2):
        assert L[k]["success"] is True and np.isnan(L[k]["dist_to_goal"])
        assert L[k]["time_to_goal"] == (k + 1) * t[k]["dt"]
    assert L[1]["success"] is False and np.isnan(L[1]["time_to_goal"]) and L[1]["dist_to_goal"] == 2.5
    for k in range(3):
        assert "cum_obj" not in L[k] and L[k]["contact_steps"] == 2 * k
        assert L[k]["cum_dist_to_goal"] == 2.0 * k and L[k]["avg_dist_to_goal"] == 2.0 * k / (k + 1)
    out = batch.run_barebone_trials(4, dt=0.025)                   # the override, for every planner
    assert [tr["dt"] for tr in fake.trials] == [0.025] * 3
    assert out["logs"][0]["time_to_goal"] == 0.025


def test_refusals_name_the_planner_and_issue_nothing(trials, capsys):
    E, fake, BT = trials
    pls = [barebone_planner(k) for k in range(3)]
    batch = E.MPPI_Batch(pls)
    with pytest.raises(ValueError, match="max_steps 0 < 1"):
        batch.run_barebone_trials(0)
    pls[1].params["num_opt"] = 0
    with pytest.raises(ValueError, match="planner 1 has num_opt 0 < 1"):
        batch.run_barebone_trials(5)
    pls[1].params["num_opt"] = 1
    for key, bad in (("x0", np.array([0.0, np.nan, 0.0])), ("x0", np.array([0.0, 0.0, np.inf])),
                     ("xgoal", np.array([np.inf, 1.0])), ("goal_tolerance", np.nan)):
        keep = pls[2].params[key]
        pls[2].params[key] = bad
        with pytest.raises(ValueError, match="planner 2: start pose, goal or goal_tolerance not finite"):
            batch.run_barebone_trials(5)
        pls[2].params[key] = keep
    for dt in (0.0, -0.1, np.nan, np.inf):
        with pytest.raises(ValueError, match="planner 0: dt .* not finite and positive"):
            batch.run_barebone_trials(5, dt=dt)
    pls[0].params["dt"] = np.nan
    with pytest.raises(ValueError, match="planner 0: dt nan not finite and positive"):
        batch.run_barebone_trials(5)
    pls[0].params["dt"] = 0.1
    pls[1].params_set = False
    with pytest.raises(ValueError, match="planner 1 cannot solve"):
        batch.run_barebone_trials(5)
    assert "MPPI parameters are not set" in capsys.readouterr().out
    pls[1].params_set = True
    det = E.MPPI_Batch([det_planner(E, k) for k in range(2)])
    with pytest.raises(ValueError, match="planner 0 is a det planner"):
        det.run_barebone_trials(5)
    with pytest.raises(ValueError, match="planner 0 is a barebone planner"):            # run_trials still refuses
        batch.run_trials([None] * 3, 5)
    stochastic = BT.MPPI_StochasticBatch.__new__(BT.MPPI_StochasticBatch)
    with pytest.raises(ValueError, match="MPPI_StochasticBatch.run_barebone_trials: barebone trials run barebone"):
        stochastic.run_barebone_trials(5)
    assert "batch_run_barebone_trials" not in fake.names() and "batch_run_trials" not in fake.names()
