"""Batches whose planners share TDM pairs (``share_tdms=True``) on the GPU (run with ``-m gpu``).  Every case runs the
same planners twice: once on one shared pair of a map (plus a planner alone on its own pair), once each on a private
pair of that map (same PMF, masks and seed, hence the same generator states, which each case asserts first).  The
private batch is K solve() calls on private copies (tests/test_gpu_stochastic_batch.py), so the contract is checked
byte for byte: every planner's snapshot equals its private twin's; the shared TDMs' generator states and completed maps
equal each twin's (in trials: the longest-running twin's); ``sample_box()`` is the hull of the members' boxes; the pair
is sampled once per call, not once per planner."""
import numpy as np
import pytest

from tests.gpu_harness import assert_same, eng, quiet, snapshot, tdm_pair, tdm_scenario, vary  # noqa: F401
from tests.scenarios import make_scenario

pytestmark = pytest.mark.gpu

TDM_KEYS = ("lin_rng", "lin_map", "ang_rng", "ang_map")
# start offsets (m) of the members of the shared pair and of the planner alone on its pair (last)
OFFSETS = [(0.0, 0.0), (1.5, -1.0), (-1.2, 1.4), (0.6, 1.9), (-1.8, -0.7), (0.4, -0.3)]


def build(E, sc, K, shared, diverged=False, goals=None, edge=None):
    """K planners of scenario sc (planner k with vary(sc, k)'s lambda and u_std, start offset OFFSETS[k]): with
    ``shared`` planners 0 .. K-2 on one pair and planner K-1 on its own; else every planner on its own pair.
    ``diverged``: one public lin.sample_grids() on every pair first (unfused); ``goals``: per-planner goal offsets;
    ``edge``: index of a planner started near the map's corner (its box leaves the map)."""
    cfg = E.Config(**sc["cfg"])

    def pair():
        lin, ang = tdm_pair(E, cfg, sc["pmf_lin"], sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        if diverged:
            lin.sample_grids()
        return lin, ang

    common = pair() if shared else None
    out = []
    with quiet():
        for k in range(K):
            lin, ang = common if shared and k < K - 1 else pair()
            p = dict(vary(sc, k)["params"])
            x0 = np.asarray(sc["params"]["x0"], dtype=np.float64).copy()
            x0[:2] += OFFSETS[k % len(OFFSETS)]
            if k == edge:
                x0[:2] = [0.15, 0.3]
            p["x0"] = x0
            if goals is not None:
                p["xgoal"] = x0[:2] + np.asarray(goals[k], dtype=np.float64)
            pl = E.MPPI_Numba(cfg)
            pl.setup(p, lin, ang)
            if "u0" in sc:
                pl.u_cur_d.copy_to_device(sc["u0"])
            out.append(pl)
    return out


def same_start(A, B):
    """The private pairs start with the generator states (and maps) of the shared pair."""
    for a, b in zip(A, B):
        for name in ("lin_tdm", "ang_tdm"):
            x, y = getattr(a, name), getattr(b, name)
            assert x is not y
            assert_same(dict(rng=x.rng_states_d.copy_to_host(), maps=x.sample_grid_batch_d.copy_to_host()),
                        dict(rng=y.rng_states_d.copy_to_host(), maps=y.sample_grid_batch_d.copy_to_host()), name)


def planner_state(p):
    """snapshot(p) without the pair's buffers and the reach box (both compared on their own)."""
    return {k: v for k, v in snapshot(p).items() if k not in TDM_KEYS + ("box",)}


def pair_state(p):
    s = snapshot(p)
    return {k: s[k] for k in TDM_KEYS}


def hull(boxes, rows, cols):
    """The shared pair's box from its members' own decisions (their private twins' sample_box()): the rectangle hull,
    how the largest; whole maps if any member decided whole maps.  (The hull's launch fits at these map sizes.)"""
    if len(boxes) == 1:
        return list(boxes[0])
    if any(b[0] == 0 for b in boxes):
        return [0, 0, rows, 0, cols]
    b = np.asarray(boxes)
    return [int(b[:, 0].max()), int(b[:, 1].min()), int(b[:, 2].max()), int(b[:, 3].min()), int(b[:, 4].max())]


def shift_all(A, B, ua, ub, r):
    for k in range(len(A)):
        x0 = np.asarray(A[k].params["x0"], dtype=np.float64) + np.array([0.03 * (k + 1), -0.02 * r, 0.05])
        A[k].shift_and_update(x0.copy(), ua[k], 1)
        B[k].shift_and_update(x0.copy(), ub[k], 1)


STOCHASTIC_CASES = ["off", "static", "hull", "edge", "num_opt2", "diverged", "m2048"]


@pytest.mark.parametrize("case", STOCHASTIC_CASES)
def test_stochastic_solve(eng, case, monkeypatch):
    E = eng
    if case in ("off", "static"):
        monkeypatch.setenv("B200MPPI_SAMPLE_BOX", case)
    shape = dict(N=64, M=2048, T=10) if case == "m2048" else dict(N=200, M=24, T=20)
    sc = tdm_scenario(1, H=128, num_opt=2 if case == "num_opt2" else 1, **shape)
    K = 6
    kw = dict(diverged=case == "diverged", edge=2 if case == "edge" else None)
    A = build(E, sc, K, shared=True, **kw)
    B = build(E, sc, K, shared=False, **kw)
    same_start(A, B)
    num_opt = int(sc["params"]["num_opt"])
    rows, cols = (int(v) for v in A[0].lin_tdm.pmf_grid_d.shape[1:])
    with quiet():
        batch_a = E.MPPI_StochasticBatch(A, share_tdms=True)
        batch_b = E.MPPI_StochasticBatch(B)
        for r in range(3):
            n0 = batch_a.launch_count()
            ua, ub = batch_a.solve(), batch_b.solve()
            assert_same(dict(u=ua), dict(u=ub), "round %d" % r)
            for k in range(K):
                assert_same(planner_state(A[k]), planner_state(B[k]), "round %d planner %d" % (r, k))
                assert_same(pair_state(A[k]), pair_state(B[k]), "round %d planner %d: its pair" % (r, k))
            own = [list(B[k].sample_box()) for k in range(K)]
            want = hull(own[:K - 1], rows, cols)
            got = [list(A[k].sample_box()) for k in range(K)]
            print("round", r, "own boxes", own, "-> group box", got[0])
            assert all(g == want for g in got[:K - 1]), (got, want)
            assert got[K - 1] == own[K - 1]                      # alone on its pair: its own box
            sampler = batch_a.launch_count() - n0 - 4 * num_opt
            if case == "off":
                assert sampler == 2                              # one fused whole-map launch per group
            else:                                                # per group: sampler (+ state advance) (x 2: unfused)
                assert 2 <= sampler <= (8 if case == "diverged" else 4), sampler
            shift_all(A, B, ua, ub, r)
    if case == "hull":
        assert want[0] == 2 and want[2] - want[1] < rows         # a box from the reach statistic, inside the map
    if case == "edge":
        assert want[0] == 0 and got[K - 1][0] != 0


@pytest.mark.parametrize("mode", ["det", "spd"])
def test_onemap_solve(eng, mode):
    E = eng
    sc = make_scenario(mode, N=200, M=1, T=20, H=64, W=64, res=0.2, B=5, seed=3, warm_start=True)
    K = 5
    A = build(E, sc, K, shared=True)
    B = build(E, sc, K, shared=False)
    same_start(A, B)
    with quiet():
        batch_a = E.MPPI_Batch(A, share_tdms=True)
        batch_b = E.MPPI_Batch(B)
        for r in range(3):
            n0 = batch_a.launch_count()
            ua, ub = batch_a.solve(), batch_b.solve()
            assert_same(dict(u=ua), dict(u=ub), "round %d" % r)
            for k in range(K):
                assert (A[k].u_prev_d is A[k]._u_prev_buf) and (B[k].u_prev_d is B[k]._u_prev_buf)
                assert_same(snapshot(A[k]), snapshot(B[k]), "round %d planner %d" % (r, k))
            assert batch_a.launch_count() - n0 == 4                # noise, ONE sampler launch for both groups, ...
            shift_all(A, B, ua, ub, r)


def test_sharing_on_without_shared_pairs_and_default_refusal(eng):
    """Sharing on, no pair shared: byte-identical to sharing off, sample_box() and launch counts included.  Sharing
    off: a shared pair is refused as before, with nothing issued."""
    E = eng
    sc = tdm_scenario(1, H=128)
    K = 4
    A = build(E, sc, K, shared=False)
    B = build(E, sc, K, shared=False)
    with quiet():
        batch_a, batch_b = E.MPPI_StochasticBatch(A, share_tdms=True), E.MPPI_StochasticBatch(B)
        for r in range(3):
            ua, ub = batch_a.solve(), batch_b.solve()
            assert_same(dict(u=ua), dict(u=ub), "round %d" % r)
            for k in range(K):
                assert_same(snapshot(A[k]), snapshot(B[k]), "round %d planner %d" % (r, k))
            assert batch_a.launch_count() == batch_b.launch_count()
            shift_all(A, B, ua, ub, r)
    S = build(E, sc, 3, shared=True)
    batch = E.MPPI_StochasticBatch(S)
    with pytest.raises(E.B200MPPIError, match="planners 0 and 1 share a TDM"):
        batch.solve()
    assert batch.launch_count() == 0
    S[1].params["alpha_dyn"] = 0.7                               # the library's own refusal, behind the Python one
    for p in S:
        p.move_mppi_task_vars_to_device()
    shared = E.MPPI_StochasticBatch(S, share_tdms=True)
    rc = E._lib.lib.b200mppi_batch_solve(shared._handle, None)
    assert rc != 0 and "share a TDM pair but have alpha_dyn" in E._lib.lib.b200mppi_last_error().decode()
    assert shared.launch_count() == 0


def _grids(E, K, n, res, seed=300):
    rng = np.random.default_rng(seed)
    return [E.TractionGrid(rng.uniform(0.2, 1.0, (n, n)), rng.uniform(0.2, 1.0, (n, n)), res=res) for _ in range(K)]


# goals: two within a step, nearby, out of reach; the planner alone on its pair: nearby
GOALS = [(0.3, 0.3), (0.35, -0.2), (0.9, -0.4), (50.0, 50.0), (-0.8, 0.6)]


@pytest.mark.parametrize("record_every", [None, 1, 3])
def test_stochastic_trials(eng, record_every):
    E = eng
    sc = tdm_scenario(1, H=128)
    K, S = len(GOALS), 16
    A = build(E, sc, K, shared=True, goals=GOALS)
    B = build(E, sc, K, shared=False, goals=GOALS)
    same_start(A, B)
    grids = _grids(E, K, 128, 0.2)
    with quiet():
        batch_a = E.MPPI_StochasticBatch(A, share_tdms=True)
        out_a = batch_a.run_stochastic_trials(grids, S, record_every=record_every)
        out_b = E.MPPI_StochasticBatch(B).run_stochastic_trials(grids, S, record_every=record_every)
    steps = out_a["steps"]
    print("steps", steps.tolist(), "status", out_a["status"])
    assert steps[0] < steps[3] == S                               # members stop at different steps
    n = batch_a.steps_issued                                      # + 2 per recorded step
    assert batch_a.launch_count() == 7 * n + (2 * -(-n // record_every) if record_every else 0)
    keys = ["xhist", "uhist", "steps"] + (["state_rollouts", "rollout_steps"] if record_every else [])
    assert_same({k: out_a[k] for k in keys}, {k: out_b[k] for k in keys}, "histories")
    assert out_a["status"] == out_b["status"]
    for k in range(K):
        assert_same({n: np.asarray(v) for n, v in out_a["logs"][k].items()},
                    {n: np.asarray(v) for n, v in out_b["logs"][k].items()}, "planner %d: log" % k)
        assert_same(planner_state(A[k]), planner_state(B[k]), "planner %d" % k)
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=B[k].params["x0"]), "planner %d" % k)
    longest = int(np.argmax(steps[:K - 1]))
    for k in range(K - 1):
        assert_same(pair_state(A[k]), pair_state(B[longest]), "the shared pair (planner %d)" % k)
    assert_same(pair_state(A[K - 1]), pair_state(B[K - 1]), "the lone planner's pair")
    assert list(A[K - 1].sample_box()) == list(B[K - 1].sample_box())
    # the members running at the group's last step: the hull of their own boxes (one member: its own box)
    rows, cols = (int(v) for v in A[0].lin_tdm.pmf_grid_d.shape[1:])
    last = [k for k in range(K - 1) if steps[k] == steps[longest]]
    want = hull([list(B[k].sample_box()) for k in last], rows, cols)
    assert all(list(A[k].sample_box()) == want for k in last), ([list(A[k].sample_box()) for k in last], want)


def test_stochastic_trials_against_host_loop(eng):
    """No goal reached: the device episode against the host loop of the shared batch's solve(), replayed on the device's
    trajectory -- u[0] every step and, at the end, every planner byte for byte, the shared pair's box included (host
    and device decide the hull alike)."""
    E = eng
    sc = tdm_scenario(1, H=128)
    K, S = 4, 8
    goals = [(50.0, 50.0)] * K
    A = build(E, sc, K, shared=True, goals=goals)
    C = build(E, sc, K, shared=True, goals=goals)
    grids = _grids(E, K, 128, 0.2)
    with quiet():
        out = E.MPPI_StochasticBatch(A, share_tdms=True).run_stochastic_trials(grids, S)
        assert all(s == "max_steps" for s in out["status"])
        host = E.MPPI_StochasticBatch(C, share_tdms=True)
        for t in range(S):
            u = host.solve()
            for k in range(K):
                assert_same({"u[0]": u[k][0]}, {"u[0]": out["uhist"][k, t]}, "planner %d step %d" % (k, t))
                C[k].shift_and_update(out["xhist"][k, t + 1], u[k], 1)
    boxes = [list(p.sample_box()) for p in A]
    print("boxes", boxes)
    for k in range(K):
        assert_same(snapshot(A[k]), snapshot(C[k]), "planner %d" % k)
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=C[k].params["x0"]), "planner %d" % k)
    assert boxes[0][0] == 2 and all(b == boxes[0] for b in boxes[:K - 1])


@pytest.mark.parametrize("mode", ["det", "spd"])
def test_onemap_trials(eng, mode):
    E = eng
    sc = make_scenario(mode, N=200, M=1, T=20, H=64, W=64, res=0.2, B=5, seed=3, warm_start=True)
    K, S = len(GOALS), 16
    A = build(E, sc, K, shared=True, goals=GOALS)
    B = build(E, sc, K, shared=False, goals=GOALS)
    same_start(A, B)
    grids = _grids(E, K, 64, 0.2, seed=310)
    with quiet():
        batch_a = E.MPPI_Batch(A, share_tdms=True)
        out_a = batch_a.run_trials(grids, S)
        out_b = E.MPPI_Batch(B).run_trials(grids, S)
    steps = out_a["steps"]
    print("steps", steps.tolist(), "status", out_a["status"])
    assert batch_a.launch_count() == 5 * batch_a.steps_issued
    assert_same({k: out_a[k] for k in ("xhist", "uhist", "steps")}, {k: out_b[k] for k in ("xhist", "uhist", "steps")},
                "histories")
    assert out_a["status"] == out_b["status"]
    for k in range(K):
        assert_same(planner_state(A[k]), planner_state(B[k]), "planner %d" % k)
    longest = int(np.argmax(steps[:K - 1]))
    for k in range(K - 1):
        assert_same(pair_state(A[k]), pair_state(B[longest]), "the shared pair (planner %d)" % k)
    assert_same(pair_state(A[K - 1]), pair_state(B[K - 1]), "the lone planner's pair")
