"""Stochastic batches of more than 1024 sampled maps on the GPU (run with ``-m gpu``): above the warp CVaR kernel's
limit the batch's one CVaR launch runs the CTA kernel (cvar_large_batch_kernel).  MPPI_StochasticBatch.solve() against
K solve() calls on identical twins, bit for bit (u, noise, per-(m, n) costs, CVaR costs, weights, RNG states, both
TDMs' states and sampled maps, sample_box()), at M 1025, 2048 and 15000 (the largest Config allows); and
run_stochastic_trials at M 2048 against the host loop replayed from the device's trajectory."""
import pytest

from tests.test_gpu_stochastic_batch import (_quiet, batch_vs_sequential, expected_batch_launches, tdm_planner,
                                             tdm_scenario)
from tests.test_gpu_stochastic_trials import replay, twins

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    assert E.device_count() >= 1, "GPU tests need a CUDA device"
    return E


@pytest.mark.parametrize("M", [1025, 2048])
def test_large_m_batch_equals_sequential(eng, M):
    """K 3: alphas 0.5, 0.25, 1.0; planner 1 warm-started, planner 2 with 0..3 masks; three closed-loop rounds."""
    scs = [tdm_scenario(k, N=96, M=M, T=12, H=48, masks03=(k == 2)) for k in range(3)]
    assert ["u0" in sc for sc in scs] == [False, True, False]
    assert len({sc["params"]["cvar_alpha"] for sc in scs}) == 3
    A, B, batch = batch_vs_sequential(eng, lambda k: tdm_planner(eng, scs[k], k), 3)
    assert batch.launch_count() == expected_batch_launches(eng, B, 3, 1)


def test_largest_m_batch_equals_sequential(eng):
    """K 2 at M 15000 on a 24 x 24-cell map."""
    scs = [tdm_scenario(k, N=64, M=15000, T=8, H=24) for k in range(2)]
    with _quiet():
        assert eng.Config(**scs[0]["cfg"]).num_grid_samples == 15000
    A, B, batch = batch_vs_sequential(eng, lambda k: tdm_planner(eng, scs[k], k), 2)
    assert batch.launch_count() == expected_batch_launches(eng, B, 3, 1)


def test_large_m_trials_equal_host_replay(eng):
    """K 4 at M 2048: planner 0 reaches its goal at step 1, planner 1 later, planner 2 runs to max_steps, planner 3
    starts near the map's corner (whole-map steps)."""
    E = eng
    A, B, grids = twins(E, K=4, N=96, M=2048, T=12)
    batch = E.MPPI_StochasticBatch(A)
    with _quiet():
        out = batch.run_stochastic_trials(grids, 8)
    steps, status = out["steps"], out["status"]
    print("steps", steps.tolist(), "status", status, "boxes", [list(p.sample_box()) for p in A])
    assert status[0] == "goal" and steps[0] == 1
    assert status[2] == "max_steps" and steps[2] == 8
    assert A[3].sample_box()[0] == 0                             # whole maps near the corner
    assert batch.launch_count() == 7 * batch.steps_issued
    replay(E, A, B, out)
