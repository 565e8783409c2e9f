"""Batched stochastic (use_tdm) solves on the GPU (run with ``-m gpu``): one MPPI_StochasticBatch.solve() of K planners
against K solve() calls on identical twins, bit for bit -- u, noise, per-(m, n) costs, costs, weights, RNG states, the
TDMs' RNG states and sampled maps, the reach box and the host-side solve state -- over closed-loop rounds; launch
counts; every refusal."""
import contextlib
import ctypes as C
import io

import numpy as np
import pytest

from tests.scenarios import make_scenario

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    assert E.device_count() >= 1, "GPU tests need a CUDA device"
    return E


def _quiet():
    return contextlib.redirect_stdout(io.StringIO())


def tdm_scenario(k, N=200, M=24, T=20, H=64, res=0.2, num_opt=1, edge=False, masks03=False):
    sc = make_scenario("tdm", N=N, M=M, T=T, H=H, W=H, res=res, B=5, seed=23 + 5 * k, warm_start=(k % 2 == 1),
                       cvar_alpha=[0.5, 0.25, 1.0, 0.1][k % 4])
    p = sc["params"]
    p["num_opt"] = num_opt
    p["obs_penalty"], p["unknown_penalty"] = 1e3 + 10 * k, 50.0 + k
    p["dt"] = [0.1, 0.08, 0.12][k % 3]
    if edge:                                             # the reach box would leave the map: whole maps
        p["x0"] = np.array([0.15, 0.3, 0.4])
    if masks03:                                          # mask values 0..3: the general penalty variant
        rng = np.random.default_rng(90 + k)
        sc["obstacle"] = (rng.integers(0, 4, sc["obstacle"].shape) * (rng.random(sc["obstacle"].shape) < 0.05)).astype(np.int8)
    return sc


def tdm_planner(E, sc, k, diverged=False):
    with _quiet():
        cfg = E.Config(**sc["cfg"])
        lin, ang = E.TDM_Numba(cfg), E.TDM_Numba(cfg)
        lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        if diverged:                                     # the pair's streams differ: each TDM sampled on its own
            lin.sample_grids()
        pl = E.MPPI_Numba(cfg)
    params = dict(sc["params"])
    params["lambda_weight"] = [1.0, 0.5, 2.0, 0.8, 1.3][k % 5]
    params["u_std"] = np.array([2.0, 3.0]) * (1.0 + 0.1 * (k % 7))
    pl.setup(params, lin, ang)
    if "u0" in sc:
        pl.u_cur_d.copy_to_device(sc["u0"])
    return pl


def planner_launches(E, p):
    n = C.c_int64()
    E._lib.check(E._lib.lib.b200mppi_planner_launch_count(p._handle, C.byref(n)))
    return int(n.value)


def snapshot(p):
    """Everything a solve() writes.  Per-(m, n) costs only once a rollout ran: with num_opt = 0 no solve writes them and
    the buffer holds whatever its allocation held."""
    d = dict(u_cur=p.u_cur_d.copy_to_host(), u_prev=p.u_prev_d.copy_to_host(), noise=p.noise_samples_d.copy_to_host(),
             costs=p.costs_d.copy_to_host(), costs_nm=p.costs_nm_d.copy_to_host(), weights=p.weights_d.copy_to_host(),
             rng=p.rng_states_d.copy_to_host(), box=np.asarray(p.sample_box()))
    if int(p.params["num_opt"]) < 1:
        del d["costs_nm"]
    for name, t in (("lin", p.lin_tdm), ("ang", p.ang_tdm)):
        d[name + "_rng"] = t.rng_states_d.copy_to_host()
        d[name + "_map"] = t.sample_grid_batch_d.copy_to_host()       # completes a boxed sampling
    return d


def assert_same(a, b, what):
    """Bit for bit: an untouched buffer may hold NaN patterns (what its allocation held), which == never equates."""
    assert a.keys() == b.keys()
    for key in a:
        x, y = np.asarray(a[key]), np.asarray(b[key])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), "%s: %s differs" % (what, key)


def batch_vs_sequential(E, make, K, rounds=3, check_every=True):
    with _quiet():
        A = [make(k) for k in range(K)]
        B = [make(k) for k in range(K)]
        batch = E.MPPI_StochasticBatch(A)
        for r in range(rounds):
            ub = batch.solve()
            us = np.stack([p.solve() for p in B])
            assert ub.shape == us.shape and ub.dtype == np.float32
            assert np.array_equal(ub, us), "round %d: u differs" % r
            for k in range(K):                           # the Python layer leaves u_prev_d as solve() does
                assert (A[k].u_prev_d is A[k]._u_prev_buf) == (B[k].u_prev_d is B[k]._u_prev_buf)
            if check_every or r == rounds - 1:
                for k in range(K):
                    assert_same(snapshot(A[k]), snapshot(B[k]), "round %d planner %d" % (r, k))
            for k in range(K):
                x0 = np.asarray(A[k].params["x0"], dtype=np.float64) + np.array([0.03 * (k + 1), -0.02 * r, 0.05])
                A[k].shift_and_update(x0.copy(), ub[k], 1)
                B[k].shift_and_update(x0.copy(), us[k], 1)
    return A, B, batch


def expected_batch_launches(E, B, rounds, num_opt):
    """1 noise + 1 rollout + 1 CVaR + 1 update per iteration, plus every planner's own sampler launches (its solve()
    issues those same sampler launches next to its 4 per iteration)."""
    per_iter = 4 * num_opt * rounds
    return per_iter + sum(planner_launches(E, p) - per_iter for p in B)


def test_stochastic_batch_equals_sequential_closed_loop(eng):
    scs = [tdm_scenario(k) for k in range(5)]
    A, B, batch = batch_vs_sequential(eng, lambda k: tdm_planner(eng, scs[k], k), 5)
    assert all(p.sample_box()[0] == 2 for p in A)                         # the dynamic box was used
    # per round: 1 noise + 5 x (boxed sampler + the fused pair's advance) + rollout + CVaR + update; solve(): 6 each
    assert [planner_launches(eng, p) for p in B] == [3 * 6] * 5
    assert batch.launch_count() == 3 * (1 + 5 * 2 + 3) == expected_batch_launches(eng, B, 3, 1)
    assert planner_launches(eng, A[0]) == 0


def test_stochastic_batch_of_one_and_num_opt(eng):
    sc = tdm_scenario(0)
    batch_vs_sequential(eng, lambda k: tdm_planner(eng, sc, k), 1, rounds=2)
    scs = [tdm_scenario(k, num_opt=2) for k in range(3)]                 # static box, two iterations
    A, B, batch = batch_vs_sequential(eng, lambda k: tdm_planner(eng, scs[k], k), 3, rounds=2)
    assert all(p.sample_box()[0] in (0, 1) for p in A)
    assert batch.launch_count() == expected_batch_launches(eng, B, 2, 2)
    scs = [tdm_scenario(k, num_opt=0) for k in range(2)]                 # maps sampled, u returned unchanged
    A, B, batch = batch_vs_sequential(eng, lambda k: tdm_planner(eng, scs[k], k), 2, rounds=1)


def test_stochastic_batch_edge_diverged_and_mixed_masks(eng):
    scs = [tdm_scenario(0), tdm_scenario(1, edge=True), tdm_scenario(2, masks03=True), tdm_scenario(3)]
    make = lambda k: tdm_planner(eng, scs[k], k, diverged=(k == 3))     # noqa: E731
    A, B, batch = batch_vs_sequential(eng, make, 4)
    assert A[1].sample_box()[0] == 0                                      # whole maps near the edge
    assert A[3].sample_box()[0] == 2
    assert batch.launch_count() == expected_batch_launches(eng, B, 3, 1)


def test_stochastic_batch_config3_shape(eng):
    scs = [tdm_scenario(k, N=1024, M=64, T=64, H=512, res=0.1) for k in range(2)]
    make = lambda k: tdm_planner(eng, scs[k % 2], k)                     # noqa: E731
    batch_vs_sequential(eng, make, 32, rounds=2, check_every=False)


def test_stochastic_batch_refusals_issue_nothing(eng, capsys):
    E = eng
    scs = [tdm_scenario(k) for k in range(3)]
    with _quiet():
        pls = [tdm_planner(E, scs[k], k) for k in range(3)]
        det = make_scenario("det", N=200, M=1, T=20, H=64, W=64, res=0.2, B=5, seed=3)
        cfg = E.Config(**det["cfg"])
        lin, ang = E.TDM_Numba(cfg), E.TDM_Numba(cfg)
        lin.set_TDM_from_PMF_grid(det["pmf_lin"], det["tdm_dict"], det["obstacle"], det["unknown"])
        ang.set_TDM_from_PMF_grid(det["pmf_ang"], det["tdm_dict"], det["obstacle"], det["unknown"])
        dp = E.MPPI_Numba(cfg)
        dp.setup(det["params"], lin, ang)
    with pytest.raises(ValueError, match="planner 1 is a det planner"):
        E.MPPI_StochasticBatch([pls[0], dp])
    with pytest.raises(ValueError, match="planner 1 uses use_tdm: the stochastic mode is not batched"):
        E.MPPI_Batch([dp, pls[0]])
    other = make_scenario("tdm", N=200, M=16, T=20, H=64, W=64, res=0.2, B=5, seed=4)
    with _quiet():
        pm = tdm_planner(E, other, 0)
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
    with _quiet():
        pls[1].setup(pls[1].params, pls[1].lin_tdm, pls[0].lin_tdm)
    with pytest.raises(E.B200MPPIError, match="share a TDM"):
        batch.solve()
    assert batch.launch_count() == 0
    for p, b in zip(pls[:1], before[:1]):
        assert_same(snapshot(p), b, "refused planner")
