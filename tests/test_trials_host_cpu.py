"""Closed-loop trials without a GPU: the C-ABI of b200mppi_batch_run_trials (prototype, descriptor and result layouts
against the ctypes mirrors), MPPI_Batch.run_trials on a fake backend (refusals, argument marshalling, the trial logs
and their NaN conventions, the state it leaves on the Python side), and the active-planner gating of the batched
kernels, emulated on the host."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.fake_backend import disarm
from tests.test_batch_host_cpu import BatchFake, barebone_planner, det_planner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_trial_abi_matches_ctypes(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    assert "b200mppi_batch_run_trials" in _lib.EXPORTS
    src = tmp_path / "abi.c"
    fields = [f for f, _ in _lib.TrialDesc._fields_]
    rfields = [f for f, _ in _lib.TrialResult._fields_]
    proto = tmp_path / "proto.c"
    proto.write_text('#include "b200mppi.h"\n'
                     "int (*f)(b200mppi_batch*, const b200mppi_trial_desc*, int32_t, double*, float*, "
                     "b200mppi_trial_result*, int32_t*) = b200mppi_batch_run_trials;\n")
    r = subprocess.run(["gcc", "-c", "-Werror", "-I", os.path.join(ROOT, "include"), str(proto), "-o",
                        str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200mppi.h"\nint main(void) {\n' +
                   '  printf("%zu %zu\\n", sizeof(b200mppi_trial_desc), sizeof(b200mppi_trial_result));\n' +
                   "".join('  printf("%%zu\\n", offsetof(b200mppi_trial_desc, %s));\n' % f for f in fields) +
                   "".join('  printf("%%zu\\n", offsetof(b200mppi_trial_result, %s));\n' % f for f in rfields) +
                   '  printf("%d %d %d\\n", B200MPPI_TRIAL_GOAL, B200MPPI_TRIAL_MAX_STEPS, B200MPPI_TRIAL_LEFT_MAP);\n'
                   "  return 0;\n}\n")
    exe = tmp_path / "abi"
    r = subprocess.run(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True).stdout.split("\n")
    assert out[0] == "%d %d" % (C.sizeof(_lib.TrialDesc), C.sizeof(_lib.TrialResult))
    offs = [int(v) for v in out[1:1 + len(fields) + len(rfields)]]
    assert offs == [getattr(_lib.TrialDesc, f).offset for f in fields] + [getattr(_lib.TrialResult, f).offset
                                                                           for f in rfields]
    assert out[1 + len(fields) + len(rfields)] == "%d %d %d" % (_lib.TRIAL_GOAL, _lib.TRIAL_MAX_STEPS,
                                                               _lib.TRIAL_LEFT_MAP)
    fn = _lib.lib.b200mppi_batch_run_trials
    assert fn.restype is C.c_int and len(fn.argtypes) == 7


class TrialFake(BatchFake):
    """Plays b200mppi_batch_run_trials: planner k runs k + 1 steps (xhist row t = (t, k, 0.5 t), u = (t, -k)) and ends
    with status (goal, max_steps, left_map)[k % 3]."""

    def b200mppi_batch_run_trials(self, h, descs, max_steps, xh, uh, res, issued):
        K = len(self.members)
        self.trials = [{f: (list(getattr(descs[i], f)) if hasattr(getattr(descs[i], f), "__len__") else
                            getattr(descs[i], f)) for f, _ in descs[i]._fields_} for i in range(K)]
        self.grids = [np.ctypeslib.as_array(C.cast(descs[i].lin, C.POINTER(C.c_double)),
                                            (descs[i].height, descs[i].width)).copy() for i in range(K)]
        self.calls.append(("batch_run_trials", (K, max_steps)))
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
def trials(monkeypatch):
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
    real_init = BT.MPPI_Batch.__init__

    def init(self, planners):
        made.append(self)
        real_init(self, planners)
    monkeypatch.setattr(BT.MPPI_Batch, "__init__", init)
    yield E, fake, BT
    for b in made:                                   # fake handles must never reach the real destroy function
        b._handle = None
    disarm(fake)


def test_run_trials_marshalling_logs_and_nan_padding(trials):
    E, fake, BT = trials
    pls = [det_planner(E, k) for k in range(3)]
    batch = E.MPPI_Batch(pls)
    rng = np.random.default_rng(0)
    grids = [E.TractionGrid(rng.uniform(0, 1, (5, 7)), rng.uniform(0, 1, (5, 7)), res=0.5, xlimits=(-1.0, 2.5)),
             E.TractionGrid(rng.uniform(0, 1, (5, 7)), rng.uniform(0, 1, (5, 7)), use_int8=True),
             E.TractionGrid(rng.uniform(0, 1, (4, 4)), rng.uniform(0, 1, (4, 4)), res=0.25)]
    x0s = [p.params["x0"].copy() for p in pls]
    out = batch.run_trials(grids, 6, dt=0.05)
    assert [tr["x0"] for tr in fake.trials] == [[float(v) for v in x] for x in x0s]
    t = fake.trials
    assert t[0]["xlo"] == -1.0 and t[0]["res"] == 0.5 and (t[0]["height"], t[0]["width"]) == (5, 7)
    assert np.array_equal(fake.grids[1], grids[1].lin_traction.astype(np.float64))
    for k, p in enumerate(pls):
        assert t[k]["dt"] == 0.05 and t[k]["goal_tolerance"] == p.params["goal_tolerance"]
        assert t[k]["xgoal"] == [float(v) for v in p.params["xgoal"]]
        assert t[k]["pxlim"] == [float(v) for v in p.lin_tdm.padded_xlimits]
        assert p.u_prev_d is p._u_prev_buf
        assert np.array_equal(p.params["x0"], [k + 1, k, 0.5 * (k + 1)]) and p.params["x0"].dtype == np.float64
    assert out["steps"].tolist() == [1, 2, 3] and out["status"] == ["goal", "max_steps", "left_map"]
    assert np.isnan(out["xhist"][0, 2:]).all() and not np.isnan(out["xhist"][2, :4]).any()
    assert np.isnan(out["uhist"][1, 2:]).all() and out["uhist"].dtype == np.float32
    L = out["logs"]
    assert L[0]["success"] is True and np.isnan(L[0]["dist_to_goal"]) and L[0]["time_to_goal"] == 1 * 0.05
    assert L[0]["cum_obj"] == 10.0 and L[0]["avg_dist_to_goal"] == 0.0
    for k in (1, 2):                                  # not reached: the d / v_post_rollout tail, no time to goal
        v_post = pls[k].params["v_post_rollout"]
        assert L[k]["success"] is False and np.isnan(L[k]["time_to_goal"]) and L[k]["dist_to_goal"] == 1.5 + k
        assert L[k]["cum_obj"] == 10.0 + k + (1.5 + k) / v_post
        assert L[k]["avg_dist_to_goal"] == 2.0 * k / (k + 1)
    names = fake.names()
    assert names.index("batch_run_trials") > max(i for i, n in enumerate(names) if n == "planner_set_params")
    assert batch.steps_issued == 3


def test_run_trials_refusals(trials, capsys):
    E, fake, BT = trials
    pls = [det_planner(E, k) for k in range(3)]
    batch = E.MPPI_Batch(pls)
    g = E.TractionGrid(np.ones((4, 4)), np.ones((4, 4)))
    with pytest.raises(ValueError, match="2 traction grids for 3 planners"):
        batch.run_trials([g, g], 5)
    with pytest.raises(ValueError, match="max_steps 0 < 1"):
        batch.run_trials([g] * 3, 0)
    pls[1].params["num_opt"] = 0
    with pytest.raises(ValueError, match="planner 1 has num_opt 0 < 1"):
        batch.run_trials([g] * 3, 5)
    pls[1].params["num_opt"] = 1
    pls[2].params["x0"] = np.array([-50.0, 0.0, 0.0])
    with pytest.raises(ValueError, match="planner 2 cannot solve"):
        batch.run_trials([g] * 3, 5)
    assert "not within padded xlimits" in capsys.readouterr().out
    pls[2].params["x0"] = pls[0].params["x0"].copy()
    g32 = E.TractionGrid(np.ones((4, 4), np.float32), np.ones((4, 4), np.float32))
    with pytest.raises(ValueError, match="planner 1: traction grid of dtype float32"):
        batch.run_trials([g, g32, g], 5)
    with pytest.raises(ValueError, match="planner 0 is a barebone planner"):
        E.MPPI_Batch([barebone_planner(0), barebone_planner(1)]).run_trials([g, g], 5)
    assert "batch_run_trials" not in fake.names()


def test_run_trials_refused_by_the_library_before_any_work():
    """Without a device: a null batch and bad arguments are refused by the C entry point."""
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    res = (_lib.TrialResult * 1)()
    assert _lib.lib.b200mppi_batch_run_trials(None, None, 5, None, None, res, None) == -1
    assert "null batch" in _lib.lib.b200mppi_last_error().decode()
