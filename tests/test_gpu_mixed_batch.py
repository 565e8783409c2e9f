"""Mixed batches on the GPU (run with ``-m gpu``): MPPI_MixedBatch of interleaved det-dynamics, speed-map and use_tdm
planners against the per-kind batches (MPPI_Batch of the det planners, MPPI_Batch of the speed-map planners,
MPPI_StochasticBatch of the use_tdm planners) on identical twins -- every output and every planner's full snapshot
bit for bit -- plus launch accounting and the refusals."""
import numpy as np
import pytest

from tests import gpu_harness as H
from tests import test_gpu_shared_tdm as SH
from tests.gpu_harness import assert_same, eng, quiet, snapshot, tdm_scenario, tdm_trial_setup  # noqa: F401
from tests.scenarios import make_scenario
from tests.test_gpu_trials import trial_setup

pytestmark = pytest.mark.gpu

KINDS = ("det", "spd", "tdm")
N, T = 256, 16                 # trial_setup's one-map shape; the use_tdm planners take it too (their maps: 64 x 64)
MAX_STEPS = 20


def planner(E, kind, j, num_opt=1):
    """Planner j of a kind and its ground-truth grid: j = 0 reaches its goal at step 1, j = 2 runs to max_steps, j = 4
    leaves the map (tests/test_gpu_trials.trial_setup, tests/gpu_harness.tdm_trial_setup)."""
    if kind == "tdm":                                    # V 1, as a one-map planner of one map sample has
        real = H.tdm_scenario
        H.tdm_scenario = lambda *a, **kw: dict(real(*a, **kw), cfg=dict(real(*a, **kw)["cfg"], num_vis_state_rollouts=1))
        try:
            return tdm_trial_setup(E, j, num_opt=num_opt, N=N, T=T)
        finally:
            H.tdm_scenario = real
    pl, grid = trial_setup(E, kind, j)
    pl.params["num_opt"] = num_opt
    return pl, grid


def twin_sets(E, js=(0, 2, 4), kinds=KINDS, num_opt=1):
    """(A, B, grids, kinds): the planners det j, spd j, tdm j for each j of js, interleaved, twice."""
    order = [(kind, j) for j in js for kind in kinds]
    with quiet():
        A = [planner(E, kind, j, num_opt) for kind, j in order]
        B = [planner(E, kind, j, num_opt) for kind, j in order]
    return [a[0] for a in A], [b[0] for b in B], [a[1] for a in A], [kind for kind, _ in order]


def per_kind(E, B, kinds, share=False):
    """[(kind, indices, batch)]: the batch of each kind present among the twins B."""
    out = []
    for kind in KINDS:
        idx = [i for i, k in enumerate(kinds) if k == kind]
        if idx:
            cls = E.MPPI_StochasticBatch if kind == "tdm" else E.MPPI_Batch
            out.append((kind, idx, cls([B[i] for i in idx], share_tdms=share)))
    return out


def log_bytes(log):
    return np.array([float(log[k]) for k in sorted(log)]).tobytes()


def assert_planner_out(got, want, i, j, what):
    """Planner i of the mixed result ``got`` against planner j of a per-kind result ``want``, bit for bit."""
    for key in ("xhist", "uhist", "steps", "episodes_run", "state_rollouts"):
        if key in want:
            x, y = got[key][i], want[key][j]
            if "episodes_run" in want and key != "episodes_run":   # episode axes padded to each call's longest list
                m = min(len(x), len(y))
                assert np.isnan(x[m:]).all() if x.dtype.kind == "f" else not x[m:].any()
                x, y = x[:m], y[:m]
            assert_same({key: x}, {key: y}, "%s planner %d" % (what, i))
    assert got["status"][i] == want["status"][j], (what, i)
    logs = lambda L: [log_bytes(x) if x is not None else None for x in (L if isinstance(L, list) else [L])]
    assert logs(got["logs"][i]) == logs(want["logs"][j]), (what, i)


def trials_per_kind(groups, call, grids):
    """The per-kind call on each group's grids: {kind: (indices, result)}."""
    out = {}
    for kind, idx, batch in groups:
        f = call(batch, kind)
        with quiet():
            out[kind] = (idx, f([grids[i] for i in idx]))
    return out


def check_all(A, B, got, ref, what):
    for kind, (idx, want) in ref.items():
        for j, i in enumerate(idx):
            assert_planner_out(got, want, i, j, "%s (%s)" % (what, kind))
    for i in range(len(A)):
        assert_same(snapshot(A[i]), snapshot(B[i]), "%s planner %d" % (what, i))
        assert_same(dict(x0=A[i].params["x0"]), dict(x0=B[i].params["x0"]), "%s planner %d" % (what, i))
        assert (A[i].u_prev_d is A[i]._u_prev_buf) == (B[i].u_prev_d is B[i]._u_prev_buf)


def test_solve_rounds(eng):
    """Three rounds of solve() + shift_and_update on interleaved det / spd / use_tdm planners: u and every snapshot."""
    E = eng
    A, B, _, kinds = twin_sets(E)
    mixed, groups = E.MPPI_MixedBatch(A), per_kind(E, B, kinds)
    assert [kinds[i] for i in mixed.order] == ["det", "spd"] * 3 + ["tdm"] * 3     # det and spd: per-descriptor rollout
    with quiet():
        for r in range(3):
            um = mixed.solve()
            us = np.empty_like(um)
            for _, idx, batch in groups:
                us[idx] = batch.solve()
            assert_same(dict(u=um), dict(u=us), "round %d" % r)
            for i in range(len(A)):
                assert_same(snapshot(A[i]), snapshot(B[i]), "round %d planner %d" % (r, i))
                x0 = np.asarray(A[i].params["x0"], dtype=np.float64) + np.array([0.03 * (i % 4), -0.02 * r, 0.05])
                A[i].shift_and_update(x0.copy(), um[i], 1)
                B[i].shift_and_update(x0.copy(), us[i], 1)


def _trial_call(batch, kind, record_every=None):
    if kind == "tdm":
        return lambda g: batch.run_stochastic_trials(g, MAX_STEPS, record_every=record_every)
    return lambda g: batch.run_trials(g, MAX_STEPS, record_every=record_every)


@pytest.mark.parametrize("grids,num_opt", [("host", 1), ("device", 1), ("host", 2)])
def test_run_trials(eng, grids, num_opt):
    """run_trials against the per-kind trial calls: goal at step 1, max_steps and left_map of every kind, on host grids
    and on DeviceTractionGrids, at num_opt 1 and 2; and the step's launches 6 n + 1 + C1 + 2 C2 (C1 = C2 = 1: one map
    geometry per kind, two geometries in all)."""
    E = eng
    A, B, g, kinds = twin_sets(E, num_opt=num_opt)
    if grids == "device":
        from tests.test_gpu_device_realisations import gt_pair
        lin, ang = gt_pair(E, H=64)
        dev = E.draw_traction_grids(lin, ang, 1)
        g = [dev[0]] * len(A)
    mixed, groups = E.MPPI_MixedBatch(A), per_kind(E, B, kinds)
    with quiet():
        out = mixed.run_trials(g, MAX_STEPS)
    ref = trials_per_kind(groups, _trial_call, g)
    check_all(A, B, out, ref, "run_trials")
    status = set(out["status"])
    if grids == "host":
        assert {"goal", "max_steps", "left_map"} <= status, status
        assert min(out["steps"]) == 1
    assert mixed.launch_count() == mixed.steps_issued * (6 * num_opt + 1 + 1 + 2)


def test_share_tdms(eng):
    """share_tdms on a mixed batch groups as the per-kind batches do: a cvar_alpha sweep of use_tdm planners on one
    pair (and one on its own) next to det planners of which two share a pair; solve and run_trials."""
    E = eng
    sc_t = tdm_scenario(0, N=N, T=T)
    sc_d = make_scenario("det", N=N, M=1, T=T, H=40, W=40, res=0.2, B=6, seed=41)

    def build():
        d = SH.build(E, sc_d, 3, shared=True)
        t = SH.build(E, sc_t, 4, shared=True)
        for k, p in enumerate(t):
            p.params["cvar_alpha"] = [0.1, 0.25, 0.5, 1.0][k]
        return [d[0], t[0], d[1], t[1], t[2], d[2], t[3]]
    A, B = build(), build()
    kinds = ["det", "tdm", "det", "tdm", "tdm", "det", "tdm"]
    mixed, groups = E.MPPI_MixedBatch(A, share_tdms=True), per_kind(E, B, kinds, share=True)
    with quiet():
        um = mixed.solve()
        us = np.empty_like(um)
        for _, idx, batch in groups:
            us[idx] = batch.solve()
    assert_same(dict(u=um), dict(u=us), "shared solve")
    grids = SH._grids(E, 3, 40, 0.2) + SH._grids(E, 4, 64, 0.2)
    grids = [grids[i] for i in (0, 3, 1, 4, 5, 2, 6)]
    with quiet():
        out = mixed.run_trials(grids, MAX_STEPS)
    ref = trials_per_kind(groups, _trial_call, grids)
    check_all(A, B, out, ref, "shared run_trials")


@pytest.mark.parametrize("reset_x0", [False, True])
def test_run_trial_sequences(eng, reset_x0):
    """run_trial_sequences with and without reset_x0 against the per-kind sequences, 1 to 3 episodes per planner."""
    E = eng
    A, B, g, kinds = twin_sets(E, js=(0, 1, 2))
    rng = np.random.default_rng(5)
    seqs = []
    for i, grid in enumerate(g):
        shape = grid.lin_traction.shape
        extra = [E.TractionGrid(rng.uniform(0.2, 1.0, shape), rng.uniform(0.2, 1.0, shape), res=grid.res,
                                xlimits=grid.xlimits, ylimits=grid.ylimits) for _ in range(i % 3)]
        seqs.append([grid] + extra)
    mixed, groups = E.MPPI_MixedBatch(A), per_kind(E, B, kinds)
    with quiet():
        out = mixed.run_trial_sequences(seqs, MAX_STEPS, reset_x0=reset_x0)
    ref = trials_per_kind(groups, lambda b, k: lambda s: b.run_trial_sequences(s, MAX_STEPS, reset_x0=reset_x0), seqs)
    check_all(A, B, out, ref, "sequences")


def test_record_every_and_get_state_rollout(eng):
    """record_every records and get_state_rollout() against the per-kind calls."""
    E = eng
    A, B, g, kinds = twin_sets(E, js=(1, 2))
    mixed, groups = E.MPPI_MixedBatch(A), per_kind(E, B, kinds)
    with quiet():
        out = mixed.run_trials(g, MAX_STEPS, record_every=3)
    ref = trials_per_kind(groups, lambda b, k: _trial_call(b, k, record_every=3), g)
    check_all(A, B, out, ref, "recorded")
    assert np.array_equal(out["rollout_steps"], np.arange(len(out["rollout_steps"])) * 3)
    with quiet():
        mixed.solve()
        for _, idx, batch in groups:
            batch.solve()
    vm = mixed.get_state_rollout()
    for _, idx, batch in groups:
        assert_same(dict(v=vm[idx]), dict(v=batch.get_state_rollout()), "get_state_rollout")
    for i in range(len(A)):
        assert_same(snapshot(A[i]), snapshot(B[i]), "after get_state_rollout planner %d" % i)


@pytest.mark.parametrize("kind", KINDS)
def test_single_kind(eng, kind):
    """A mixed batch of one kind equals the batch of that kind, launch counts included (solve, then run_trials)."""
    E = eng
    A, B, g, kinds = twin_sets(E, kinds=(kind,))
    mixed, [(_, _, batch)] = E.MPPI_MixedBatch(A), per_kind(E, B, kinds)
    with quiet():
        um, us = mixed.solve(), batch.solve()
    assert_same(dict(u=um), dict(u=us), "solve")
    assert mixed.launch_count() == batch.launch_count()
    with quiet():
        out = mixed.run_trials(g, MAX_STEPS)
        want = _trial_call(batch, kind)(g)
    check_all(A, B, out, {kind: (list(range(len(A))), want)}, "single kind")
    assert mixed.launch_count() == batch.launch_count()
    assert mixed.steps_issued == batch.steps_issued


def test_refusals(eng):
    """Refused before any work, naming the planner(s): a barebone planner, unequal T, unequal num_opt, a TDM used by
    two kinds, unequal num_vis_state_rollouts when recording; snapshots and launch counts unchanged."""
    E = eng
    A, _, g, kinds = twin_sets(E, js=(1,))
    from tests.test_batch_host_cpu import barebone_planner
    with quiet():
        bb = barebone_planner(0)
        other_T, _ = trial_setup(E, "det", 1)
    with pytest.raises(ValueError, match="planner 3 is a barebone planner"):
        E.MPPI_MixedBatch(A + [bb])
    other_T.num_steps += 1                              # as a planner of another T presents itself
    with pytest.raises(ValueError, match="planner 3 has num_steps"):
        E.MPPI_MixedBatch(A + [other_T])
    mixed = E.MPPI_MixedBatch(A)
    before = [snapshot(p) for p in A]
    A[2].params["num_opt"] = 2
    with pytest.raises(ValueError, match="planner 2 has num_opt 2"):
        mixed.solve()
    with pytest.raises(ValueError, match="planner 2 has num_opt 2"):
        mixed.run_trials(g, MAX_STEPS)
    A[2].params["num_opt"] = 1
    saved = A[2].lin_tdm
    A[2].lin_tdm = A[0].lin_tdm
    with pytest.raises(ValueError, match="planners 0 and 2 share a TDM"):
        mixed.run_trial_sequences([[x] for x in g], MAX_STEPS)
    A[2].lin_tdm = saved
    A[1].num_vis_state_rollouts += 1
    with pytest.raises(ValueError, match="planner 1 has num_vis_state_rollouts"):
        mixed.run_trials(g, MAX_STEPS, record_every=2)
    A[1].num_vis_state_rollouts -= 1
    assert mixed.launch_count() == 0
    for p, s in zip(A, before):
        assert_same(snapshot(p), s, "after the refusals")
