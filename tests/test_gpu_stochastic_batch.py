"""Batched stochastic (use_tdm) solves on the GPU (run with ``-m gpu``): one MPPI_StochasticBatch.solve() of K planners
against K solve() calls on identical twins, bit for bit -- u, noise, per-(m, n) costs, costs, weights, RNG states, the
TDMs' RNG states and sampled maps, the reach box and the host-side solve state -- over closed-loop rounds; launch
counts; every refusal."""
import pytest

from tests.gpu_harness import (assert_same, batch_vs_sequential, eng, expected_batch_launches,  # noqa: F401
                               planner_launches, quiet, snapshot, tdm_planner, tdm_scenario, vary)
from tests.scenarios import make_scenario

pytestmark = pytest.mark.gpu


def test_stochastic_batch_equals_sequential_closed_loop(eng):
    scs = [tdm_scenario(k) for k in range(5)]
    A, B, batch = batch_vs_sequential(eng.MPPI_StochasticBatch, lambda k: tdm_planner(eng, vary(scs[k], k)), 5)
    assert all(p.sample_box()[0] == 2 for p in A)                         # the dynamic box was used
    # per round: 1 noise + 5 x (boxed sampler + the fused pair's advance) + rollout + CVaR + update; solve(): 6 each
    assert [planner_launches(p) for p in B] == [3 * 6] * 5
    assert batch.launch_count() == 3 * (1 + 5 * 2 + 3) == expected_batch_launches(B, 3, 1)
    assert planner_launches(A[0]) == 0


def test_stochastic_batch_of_one_and_num_opt(eng):
    sc = tdm_scenario(0)
    batch_vs_sequential(eng.MPPI_StochasticBatch, lambda k: tdm_planner(eng, vary(sc, k)), 1, rounds=2)
    scs = [tdm_scenario(k, num_opt=2) for k in range(3)]                 # static box, two iterations
    A, B, batch = batch_vs_sequential(eng.MPPI_StochasticBatch, lambda k: tdm_planner(eng, vary(scs[k], k)), 3,
                                      rounds=2)
    assert all(p.sample_box()[0] in (0, 1) for p in A)
    assert batch.launch_count() == expected_batch_launches(B, 2, 2)
    scs = [tdm_scenario(k, num_opt=0) for k in range(2)]                 # maps sampled, u returned unchanged
    A, B, batch = batch_vs_sequential(eng.MPPI_StochasticBatch, lambda k: tdm_planner(eng, vary(scs[k], k)), 2,
                                      rounds=1)


def test_stochastic_batch_edge_diverged_and_mixed_masks(eng):
    scs = [tdm_scenario(0), tdm_scenario(1, edge=True), tdm_scenario(2, masks03=True), tdm_scenario(3)]
    make = lambda k: tdm_planner(eng, vary(scs[k], k), diverged=(k == 3))      # noqa: E731
    A, B, batch = batch_vs_sequential(eng.MPPI_StochasticBatch, make, 4)
    assert A[1].sample_box()[0] == 0                                      # whole maps near the edge
    assert A[3].sample_box()[0] == 2
    assert batch.launch_count() == expected_batch_launches(B, 3, 1)


def test_stochastic_batch_config3_shape(eng):
    scs = [tdm_scenario(k, N=1024, M=64, T=64, H=512, res=0.1) for k in range(2)]
    make = lambda k: tdm_planner(eng, vary(scs[k % 2], k))                      # noqa: E731
    batch_vs_sequential(eng.MPPI_StochasticBatch, make, 32, rounds=2, check_every=False)


def test_stochastic_batch_refusals_issue_nothing(eng, capsys):
    E = eng
    scs = [tdm_scenario(k) for k in range(3)]
    with quiet():
        pls = [tdm_planner(E, vary(scs[k], k)) for k in range(3)]
        det = make_scenario("det", N=200, M=1, T=20, H=64, W=64, res=0.2, B=5, seed=3)
        dp = tdm_planner(E, det)
    with pytest.raises(ValueError, match="planner 1 is a det planner"):
        E.MPPI_StochasticBatch([pls[0], dp])
    with pytest.raises(ValueError, match="planner 1 uses use_tdm: the stochastic mode is not batched"):
        E.MPPI_Batch([dp, pls[0]])
    other = make_scenario("tdm", N=200, M=16, T=20, H=64, W=64, res=0.2, B=5, seed=4)
    with quiet():
        pm = tdm_planner(E, vary(other, 0))
    with pytest.raises(E.B200MPPIError, match="planner 1 has num_grid_samples 16, planner 0 24"):
        E.MPPI_StochasticBatch([pls[0], pm])
    batch = E.MPPI_StochasticBatch(pls)
    before = [snapshot(p) for p in pls]
    with pytest.raises(ValueError, match="trials run det-dynamics or speed-map"):
        batch.run_trials([None] * 3, 5)
    res = (E._lib.TrialResult * 3)()
    rc = E._lib.lib.b200mppi_batch_run_trials(batch._handle, (E._lib.TrialDesc * 3)(), 5, None, None, res, None)
    assert rc != 0 and "planner 0 is MODE_TDM" in E._lib.lib.b200mppi_last_error().decode()
    pls[2].params["num_opt"] = 2
    with pytest.raises(E.B200MPPIError, match="planner 2 has num_opt 2"):
        batch.solve()
    pls[2].params["num_opt"] = 1
    with quiet():
        pls[1].setup(pls[1].params, pls[1].lin_tdm, pls[0].lin_tdm)
    with pytest.raises(E.B200MPPIError, match="share a TDM"):
        batch.solve()
    assert batch.launch_count() == 0
    for p, b in zip(pls[:1], before[:1]):
        assert_same(snapshot(p), b, "refused planner")
