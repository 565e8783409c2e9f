"""Mixed batches without a GPU: the C-ABI of b200mppi_batch_create_mixed and b200mppi_batch_run_mixed_trials
(exports, header prototypes, B200MPPI_TRIALS_MIXED, argument refusals), and MPPI_MixedBatch on a fake backend -- the
internal order (one-map planners first), the planners, descriptors and trial kind handed to the library, the mapping
of every result back to the caller's order, and every refusal issuing nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.fake_backend import disarm
from tests.test_batch_host_cpu import BatchFake, barebone_planner, det_planner

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["tdm", "det", "spd", "tdm", "det", "spd"]      # caller order; the batch's: det, spd, det, spd, tdm, tdm
ORDER = [1, 2, 4, 5, 0, 3]


def test_abi_matches_header(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    for name in ("b200mppi_batch_create_mixed", "b200mppi_batch_run_mixed_trials"):
        assert name in _lib.EXPORTS
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include "b200mppi.h"\n'
                   "int (*f)(b200mppi_planner* const*, int32_t, b200mppi_batch**) = b200mppi_batch_create_mixed;\n"
                   "int (*g)(b200mppi_batch*, const b200mppi_trial_desc*, int32_t, double*, float*, "
                   "b200mppi_trial_result*, int32_t*) = b200mppi_batch_run_mixed_trials;\n"
                   'int main(void) { printf("%d\\n", B200MPPI_TRIALS_MIXED); return 0; }\n')
    exe = tmp_path / "abi"
    r = subprocess.run(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                        "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)], capture_output=True, text=True).stdout.strip() == str(_lib.TRIALS_MIXED)
    P, I32 = C.c_void_p, C.c_int32
    assert list(_lib.lib.b200mppi_batch_create_mixed.argtypes) == [C.POINTER(P), I32, C.POINTER(P)]
    fn = _lib.lib.b200mppi_batch_run_mixed_trials
    assert fn.restype is C.c_int and len(fn.argtypes) == 7 and fn.argtypes[1] is C.POINTER(_lib.TrialDesc)


def test_library_refusals_before_any_work():
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    L = _lib.lib
    h = C.c_void_p()
    assert L.b200mppi_batch_create_mixed((C.c_void_p * 1)(), 0, C.byref(h)) == -1
    assert "batch_create_mixed: count < 1" in L.b200mppi_last_error().decode()
    assert L.b200mppi_batch_create_mixed((C.c_void_p * 2)(None, None), 2, C.byref(h)) == -1
    assert "batch_create_mixed: planner 0 is null" in L.b200mppi_last_error().decode()
    assert not h.value
    res = (_lib.TrialResult * 1)()
    assert L.b200mppi_batch_run_mixed_trials(None, None, 5, None, None, res, None) == -1
    assert "null batch" in L.b200mppi_last_error().decode()


class MixedFake(BatchFake):
    """Plays the mixed batch: the solve fills u with the batch-order index, the trials give batch-order planner j
    j + 1 steps and the sequences one episode each."""

    def b200mppi_batch_create_mixed(self, arr, n, out):
        self.members = [arr[i] for i in range(n)]
        self.calls.append(("batch_create_mixed", (n,)))
        return self._handle_out(out)

    def b200mppi_batch_solve(self, h, u):
        n = len(self.members)
        self.calls.append(("batch_solve", (n,)))
        fill = np.repeat(np.arange(n, dtype=np.float32), self.T * 2)
        C.memmove(u.value if isinstance(u, C.c_void_p) else C.cast(u, C.c_void_p).value, fill.ctypes.data, fill.nbytes)
        return 0

    def _play(self, name, kind, descs, slots, max_steps, xh, uh, res):
        self.trial = dict(name=name, kind=kind, x0=[list(descs[j].x0) for j in range(slots)])
        self.calls.append((name, (slots, max_steps)))
        xs = np.full((slots, max_steps + 1, 3), np.nan)
        for j in range(slots):
            res[j].steps, res[j].status, res[j].cum_obj, res[j].cum_dist_to_goal = j + 1, 2, 1.0, float(j)
            xs[j, :j + 2] = j
        C.memmove(xh.value if isinstance(xh, C.c_void_p) else C.cast(xh, C.c_void_p).value, xs.ctypes.data, xs.nbytes)
        return 0

    def b200mppi_batch_run_mixed_trials(self, h, descs, max_steps, xh, uh, res, issued):
        return self._play("batch_run_mixed_trials", None, descs, len(self.members), max_steps, xh, uh, res)

    def b200mppi_batch_run_trial_sequences(self, h, kind, descs, episodes, max_steps, reset_x0, xh, uh, res, issued):
        return self._play("batch_run_trial_sequences", kind, descs, len(self.members), max_steps, xh, uh, res)


@pytest.fixture()
def host(monkeypatch):
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    import mppi_numba_b200.barebone as B
    import mppi_numba_b200.batch as BT
    import mppi_numba_b200.mppi as M
    import mppi_numba_b200.terrain as T
    fake = MixedFake()
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


def planners(E):
    return [det_planner(E, k, mode=m) for k, m in enumerate(KINDS)]


def grids(E, K):
    rng = np.random.default_rng(1)
    return [E.TractionGrid(rng.uniform(0.2, 1.0, (20, 20)), rng.uniform(0.2, 1.0, (20, 20)), res=0.25)
            for _ in range(K)]


def test_order_solve_and_mapping(host):
    E, fake = host
    P = planners(E)
    fake.T = P[0].num_steps
    b = E.MPPI_MixedBatch(P)
    assert b.order == ORDER and b.kind == "mixed"
    assert fake.members == [P[i]._handle.value for i in ORDER]
    for p in P:
        p.u_prev_d = None
    u = b.solve()
    for j, i in enumerate(ORDER):                    # batch-order row j is caller planner ORDER[j]'s
        assert (u[i] == j).all()
    for p, kind in zip(P, KINDS):                   # one-map planners alias u_prev_d as their own solve() does
        assert (p.u_prev_d is p._u_prev_buf) == (kind != "tdm")


def test_trials_descriptors_kind_and_mapping(host):
    E, fake = host
    P = planners(E)
    for k, p in enumerate(P):
        p.params["x0"] = np.array([1.0 + 0.1 * k, 2.0, 0.0])
    b = E.MPPI_MixedBatch(P)
    out = b.run_trials(grids(E, len(P)), 8)
    assert fake.trial["name"] == "batch_run_mixed_trials"
    assert [x[0] for x in fake.trial["x0"]] == [1.0 + 0.1 * i for i in ORDER]
    for j, i in enumerate(ORDER):
        assert out["steps"][i] == j + 1 and out["xhist"][i, 0, 0] == j and out["status"][i] == "max_steps"
        assert out["logs"][i]["cum_dist_to_goal"] == float(j)
        assert P[i].params["x0"][0] == j              # the final pose of its own episode
    out = b.run_trial_sequences([[g] for g in grids(E, len(P))], 8)
    assert fake.trial["kind"] == E._lib.TRIALS_MIXED
    for j, i in enumerate(ORDER):
        assert out["steps"][i, 0] == j + 1 and out["episodes_run"][i] == 1


class Ranked(object):
    use_det_dynamics, world_size = True, 2


def test_refusals_issue_nothing(host, capsys):
    E, fake = host
    P = planners(E)
    with pytest.raises(ValueError, match="planner 6 is a barebone planner"):
        E.MPPI_MixedBatch(P + [barebone_planner(0)])
    with pytest.raises(ValueError, match="planner 6 has world_size 2"):
        E.MPPI_MixedBatch(P + [Ranked()])
    other = det_planner(E, 9, mode="spd")
    other.num_steps += 1
    with pytest.raises(ValueError, match="planner 6 has num_steps"):
        E.MPPI_MixedBatch(P + [other])
    other = det_planner(E, 9, mode="tdm")
    other.num_grid_samples += 1
    with pytest.raises(ValueError, match="planner 6 has num_grid_samples"):
        E.MPPI_MixedBatch(P + [other])
    assert not [c for c in fake.calls if c[0] == "batch_create_mixed"]
    b = E.MPPI_MixedBatch(P)
    n = len(fake.calls)
    P[3].params["num_opt"] = 2
    with pytest.raises(ValueError, match="planner 3 has num_opt 2"):
        b.solve()
    with pytest.raises(ValueError, match="planner 3 has num_opt 2"):
        b.run_trials(grids(E, len(P)), 8)
    P[3].params["num_opt"] = 1
    saved = P[0].ang_tdm
    P[0].ang_tdm = P[4].lin_tdm                      # a use_tdm planner on a det planner's TDM
    for share in (False, True):
        b.share_tdms = share
        with pytest.raises(ValueError, match="planners 0 and 4 share a TDM"):
            b.run_trial_sequences([[g] for g in grids(E, len(P))], 8)
    P[0].ang_tdm = saved
    P[5].num_vis_state_rollouts += 1
    with pytest.raises(ValueError, match="planner 5 has num_vis_state_rollouts"):
        b.run_trials(grids(E, len(P)), 8, record_every=2)
    with pytest.raises(ValueError, match="planner 5 has num_vis_state_rollouts"):
        b.get_state_rollout()
    with pytest.raises(ValueError, match="barebone"):
        b.run_barebone_trials(8)
    issued = [c[0] for c in fake.calls[n:]]
    assert not [c for c in issued if c.startswith("batch_")], issued
