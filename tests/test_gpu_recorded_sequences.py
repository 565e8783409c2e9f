"""Recorded trial sequences on the GPU (run with ``-m gpu``): run_trial_sequences(record_every=n) against the host
sequence loop (tests/recorded_sequence_loop.py) replayed on identical twins with the device trajectory, calling
get_state_rollout() at each episode's steps t with t % n == 0 (after solve(), before shift_and_update) -- every record
bit for bit, NaN after an episode's last step and for episodes that did not run or do not exist, state_rollout_batch_d and every planner's snapshot --
while everything else equals the same sequence without recording; one-episode sequences against run_trials with
record_every; det-dynamics, speed-map, use_tdm, mixed-geometry, MPPI_MixedBatch and share_tdms batches; the same loop
driven by its own plant step; the launch formulas; the refusals."""
import ctypes as C
import functools

import numpy as np
import pytest

from tests import test_gpu_mixed_batch as MB
from tests import test_gpu_mixed_geometry_trials as MG
from tests import test_gpu_shared_tdm as SH
from tests.gpu_harness import assert_same, eng, quiet, snapshot, solve_in_batch_of_one, tdm_scenario  # noqa: F401
from tests.recorded_sequence_loop import recorded_sequence
from tests.test_gpu_device_realisations import drawn
from tests.test_gpu_trial_sequences import EPISODES, MAX_STEPS, episode_grids, setup

pytestmark = pytest.mark.gpu


def with_vis(p):
    d = snapshot(p)
    d["state_rollout"] = p.state_rollout_batch_d.copy_to_host()
    return d


def triplets(E, case):
    """Three identical sets (recorded, host replay, plain), per-episode base grids, batch class, host solve of one
    planner, episode counts.  "mixed": MPPI_MixedBatch of interleaved det, spd and use_tdm planners (one-map planners
    first inside the batch, so the stochastic launches index their flags from K1 > 0).  "shared": MPPI_StochasticBatch
    with share_tdms, planners 0..3 on one pair with goals reached at different steps and unequal episode counts (the
    members record at different episode steps), replayed on twins with private pairs."""
    if case == "tdm_mixed":
        specs = MG.SPECS[:5]
        sets = [MG.build(E, "tdm", specs) for _ in range(3)]
        grids = [MG.grid_of(E, k, s) for k, s in enumerate(specs)]
        return sets, grids, E.MPPI_StochasticBatch, solve_in_batch_of_one, [2, 5, 1, 3, 2]
    if case == "mixed":
        A, B, grids, kinds = MB.twin_sets(E, js=(0, 2, 4))
        _, Cw, _, _ = MB.twin_sets(E, js=(0, 2, 4))
        tdm = {id(p) for p, k in zip(B, kinds) if k == "tdm"}

        def solve_one(p):
            return solve_in_batch_of_one(p) if id(p) in tdm else p.solve()
        return [A, B, Cw], grids, E.MPPI_MixedBatch, solve_one, [2, 1, 3, 3, 2, 1, 2, 3, 2]
    if case == "shared":
        sc = tdm_scenario(1, H=128)
        A, Cw = (SH.build(E, sc, len(SH.GOALS), shared=True, goals=SH.GOALS) for _ in range(2))
        B = SH.build(E, sc, len(SH.GOALS), shared=False, goals=SH.GOALS)
        SH.same_start(A, B)
        return ([A, B, Cw], SH._grids(E, len(SH.GOALS), 128, 0.2),
                functools.partial(E.MPPI_StochasticBatch, share_tdms=True), solve_in_batch_of_one, [3, 1, 2, 2, 2])
    A, B, grids, cls, solve_one = setup(E, case)
    _, Cw, _, _, _ = setup(E, case)
    return [A, B, Cw], grids, cls, solve_one, EPISODES


def replay_records(A, B, out, seqs, solve_one, reset_x0, every, shared=False):
    """tests/recorded_sequence_loop on twins B, fed with the device trajectory: u[0] of every solve, every record, NaN
    where nothing was recorded, then every planner and its state_rollout_batch_d.  shared: B are private-pair twins of
    the shared members, so each planner is compared without its pair and box, and the shared pair against the private
    pair of the member that ran the most steps in all."""
    rec = out["state_rollouts"]
    for k, p in enumerate(B):
        run = int(out["episodes_run"][k])
        assert np.isnan(rec[k, run:]).all(), "planner %d: records of episodes that did not run" % k
        with quiet():
            host = recorded_sequence(p, seqs[k], MAX_STEPS, every, reset_x0=reset_x0, solve=solve_one,
                                     replay=(out["xhist"][k], out["steps"][k], run))
        for e, h in enumerate(host[:run]):
            n = int(out["steps"][k, e])
            assert_same({"u": h[1]}, {"u": out["uhist"][k, e]}, "planner %d episode %d: u[0]" % (k, e))
            assert_same({"r": h[4]}, {"r": rec[k, e]}, "planner %d episode %d: records" % (k, e))
            assert not np.isnan(rec[k, e, :-(-n // every)]).any()
            assert np.isnan(rec[k, e, -(-n // every):]).all(), "planner %d episode %d: records after step %d" % (k, e, n)
        if shared:
            want = dict(SH.planner_state(p), state_rollout=p.state_rollout_batch_d.copy_to_host())
            got = dict(SH.planner_state(A[k]), state_rollout=A[k].state_rollout_batch_d.copy_to_host())
            assert_same(got, want, "planner %d after the host loop" % k)
        else:
            assert_same(with_vis(A[k]), with_vis(p), "planner %d after the host loop" % k)
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=p.params["x0"]), "planner %d: x0" % k)
    if shared:
        K = len(A)
        longest = int(np.argmax(out["steps"][:K - 1].sum(axis=1)))
        for k in range(K - 1):
            assert_same(SH.pair_state(A[k]), SH.pair_state(B[longest]), "the shared pair (planner %d)" % k)
        assert_same(SH.pair_state(A[K - 1]), SH.pair_state(B[K - 1]), "the lone planner's pair")


CASES = [("det", 1, False), ("det", 3, True), ("det", 25, False), ("spd", 3, False), ("spd", 2, True),
         ("tdm", 1, True), ("tdm", 3, False), ("tdm_mixed", 3, False), ("mixed", 3, False), ("mixed", 2, True),
         ("shared", 3, False), ("shared", 2, True)]


@pytest.mark.parametrize("case,every,reset_x0", CASES)
def test_records_against_host_loop(eng, case, every, reset_x0):
    E = eng
    (A, B, Cw), grids, cls, solve_one, episodes = triplets(E, case)
    seqs = [episode_grids(E, g, k, n) for k, (g, n) in enumerate(zip(grids, episodes))]
    ba, bc = cls(A), cls(Cw)
    with quiet():
        out = ba.run_trial_sequences(seqs, MAX_STEPS, reset_x0=reset_x0, record_every=every)
        plain = bc.run_trial_sequences(seqs, MAX_STEPS, reset_x0=reset_x0)
    print(case, every, reset_x0, "steps", out["steps"].tolist(), "status", out["status"])
    K, Emax, R = len(A), max(episodes), -(-MAX_STEPS // every)
    V, T = A[0].num_vis_state_rollouts, A[0].num_steps
    assert out["state_rollouts"].shape == (K, Emax, R, V, T + 1, 3) and out["state_rollouts"].dtype == np.float32
    assert out["rollout_steps"].tolist() == [r * every for r in range(R)]
    for k in range(K):                                # episodes that do not exist
        assert np.isnan(out["state_rollouts"][k, episodes[k]:]).all()
    if not reset_x0 and case != "shared":
        assert any("left_map" in s[:-1] and s[-1] == "not_run" for s in out["status"])
    if case == "shared":                              # the members' episodes end at different steps
        assert len(set(out["steps"][:K - 1, 0].tolist())) > 1, out["steps"]
    # everything else as without recording
    assert set(out) == set(plain) | {"state_rollouts", "rollout_steps"}
    for key in ("xhist", "uhist", "steps", "episodes_run"):
        assert_same({key: out[key]}, {key: plain[key]}, "%s vs plain" % key)
    assert out["status"] == plain["status"] and ba.steps_issued == bc.steps_issued
    for k in range(K):
        for e, (lo, lp) in enumerate(zip(out["logs"][k], plain["logs"][k])):
            assert (lo is None) == (lp is None)
            if lo is not None:
                assert_same({x: np.float64(v) for x, v in lo.items()}, {x: np.float64(v) for x, v in lp.items()},
                            "planner %d episode %d: log" % (k, e))
        assert_same(snapshot(A[k]), snapshot(Cw[k]), "planner %d vs plain" % k)
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=Cw[k].params["x0"]), "planner %d: x0" % k)
        if case in ("tdm", "tdm_mixed", "shared"):
            assert list(A[k].sample_box()) == list(Cw[k].sample_box())
    if case in ("tdm", "shared"):
        assert any(p.sample_box()[0] != 0 for p in A)
    # launches: the plain sequence's, plus 1 + C2 at every step
    C2 = {"tdm": 1, "tdm_mixed": 2, "mixed": 1, "shared": 1}.get(case, 0)
    assert ba.launch_count() == bc.launch_count() + (1 + C2) * ba.steps_issued
    replay_records(A, B, out, seqs, solve_one, reset_x0, every, shared=case == "shared")


@pytest.mark.parametrize("reset_x0", [False, True])
def test_against_independent_host_loop(eng, reset_x0):
    """Against tests/recorded_sequence_loop driven by its own numpy plant step on twins: the same status and steps,
    trajectories within 1e-9 and records within 1e-5 (the plant steps round differently in the last bits)."""
    E = eng
    A, B, grids, cls, _ = setup(E, "det")
    seqs = [episode_grids(E, g, k, n) for k, (g, n) in enumerate(zip(grids, EPISODES))]
    every = 3
    with quiet():
        out = cls(A).run_trial_sequences(seqs, MAX_STEPS, reset_x0=reset_x0, record_every=every)
        host = [recorded_sequence(p, s, MAX_STEPS, every, reset_x0=reset_x0) for p, s in zip(B, seqs)]
    for k, eps in enumerate(host):
        for e, h in enumerate(eps):
            if h is None:
                assert out["status"][k][e] == "not_run" and np.isnan(out["state_rollouts"][k, e]).all()
                continue
            xh, uh, n, status, recs = h
            assert out["status"][k][e] == status and out["steps"][k, e] == n, (k, e)
            assert np.allclose(out["xhist"][k, e], xh, rtol=0, atol=1e-9, equal_nan=True)
            assert np.allclose(out["state_rollouts"][k, e], recs, rtol=0, atol=1e-5, equal_nan=True), (k, e)


@pytest.mark.parametrize("mode", ["det", "tdm"])
def test_one_episode_equals_run_trials(eng, mode):
    E = eng
    A, B, grids, cls, _ = setup(E, mode)
    ba, bb = cls(A), cls(B)
    every = 3
    with quiet():
        out = ba.run_trial_sequences([[g] for g in grids], MAX_STEPS, record_every=every)
        f = bb.run_stochastic_trials if mode == "tdm" else bb.run_trials
        want = f(grids, MAX_STEPS, record_every=every)
    assert_same(dict(r=out["state_rollouts"][:, 0], x=out["xhist"][:, 0], u=out["uhist"][:, 0], n=out["steps"][:, 0]),
                dict(r=want["state_rollouts"], x=want["xhist"], u=want["uhist"], n=want["steps"]), "outputs")
    assert out["rollout_steps"].tolist() == want["rollout_steps"].tolist()
    for k in range(len(A)):
        assert_same(with_vis(A[k]), with_vis(B[k]), "planner %d" % k)
    # the same steps; the sequence issues the record launches at every step, run_trials at recorded steps only
    C2 = 1 if mode == "tdm" else 0
    n = ba.steps_issued
    assert n == bb.steps_issued
    assert ba.launch_count() - bb.launch_count() == (1 + C2) * (n - -(-n // every))


def test_refusals_issue_nothing(eng):
    E = eng
    from mppi_numba_b200 import _lib as L
    A, _, grids, cls, _ = setup(E, "det")
    batch = cls(A)
    seqs = [[g] for g in grids]
    before = [with_vis(p) for p in A]
    with pytest.raises(ValueError, match="record_every 0 < 1"):
        batch.run_trial_sequences(seqs, 5, record_every=0)
    V = A[0].num_vis_state_rollouts
    A[3].num_vis_state_rollouts = V + 1
    with pytest.raises(ValueError, match="planner 3 has num_vis_state_rollouts %d" % (V + 1)):
        batch.run_trial_sequences(seqs, 5, record_every=2)
    A[3].num_vis_state_rollouts = V
    with pytest.raises(ValueError, match="planner 1: empty list"):
        batch.run_trial_sequences([[grids[0]], [], [grids[2]], [grids[3]], [grids[4]]], 5, record_every=2)
    # the C entry point: a wrong record byte count, a negative record_every, contact counts for a map batch
    K, T = len(A), A[0].num_steps
    descs = (L.TrialDesc * K)()
    keep = []
    from mppi_numba_b200.batch import _fill_desc
    for i, p in enumerate(A):
        p.move_mppi_task_vars_to_device()
        _fill_desc("p", p, grids[i], None, descs[i], keep)
    eps = np.ones(K, np.int32)
    xh, uh = np.empty((K, 6, 3)), np.empty((K, 5, 2), np.float32)
    res, issued, con = (L.TrialResult * K)(), C.c_int32(-1), np.zeros(K, np.int32)
    good = np.empty((K, 3, V, T + 1, 3), np.float32)
    for every, nbytes, contacts, msg in ((2, good.nbytes - 4, None, "rollouts buffer of"),
                                         (-1, good.nbytes, None, "record_every -1 < 0"),
                                         (2, good.nbytes, L.ptr(con), "contact_steps given")):
        rc = L.lib.b200mppi_batch_run_trial_sequences_ex(batch._handle, L.TRIALS_MAP, descs, L.ptr(eps), 5, 0,
                                                         L.ptr(xh), L.ptr(uh), res, contacts, every, L.ptr(good),
                                                         nbytes, C.byref(issued))
        assert rc != 0 and msg in L.lib.b200mppi_last_error().decode(), (msg, L.lib.b200mppi_last_error())
    assert issued.value == -1 and batch.launch_count() == 0
    for p, b in zip(A, before):
        assert_same(with_vis(p), b, "untouched")


def test_unrecorded_launches_unchanged(eng):
    """An unrecorded sequence issues the parent's launches: 5 per det step (3 num_opt + 1 + C1)."""
    E = eng
    A, _, grids, cls, _ = setup(E, "det")
    batch = cls(A)
    seqs = [episode_grids(E, g, k, n) for k, (g, n) in enumerate(zip(grids, EPISODES))]
    with quiet():
        batch.run_trial_sequences(seqs, MAX_STEPS)
    assert batch.launch_count() == 5 * batch.steps_issued


@pytest.mark.parametrize("reset_x0", [False, True])
def test_device_grids(eng, reset_x0):
    """Records on DeviceTractionGrid realisations equal those on the same realisations' host grids."""
    E = eng
    A, B, grids, cls, _ = setup(E, "tdm")
    with quiet():
        dev, host = drawn(E, 3, H=64)
    seqs_d = [[dev[(k + e) % 3] for e in range(2)] for k in range(len(A))]
    seqs_h = [[host[(k + e) % 3] for e in range(2)] for k in range(len(A))]
    with quiet():
        out = cls(A).run_trial_sequences(seqs_d, MAX_STEPS, reset_x0=reset_x0, record_every=4)
        want = cls(B).run_trial_sequences(seqs_h, MAX_STEPS, reset_x0=reset_x0, record_every=4)
    for key in ("state_rollouts", "xhist", "uhist", "steps"):
        assert_same({key: out[key]}, {key: want[key]}, key)
    for k in range(len(A)):
        assert_same(with_vis(A[k]), with_vis(B[k]), "planner %d" % k)
