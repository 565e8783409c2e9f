"""Batched one-map solves on the GPU (run with ``-m gpu``): one MPPI_Batch.solve() of K planners against K solve()
calls on identical twins, bit for bit -- the returned u, every planner buffer solve() writes, the planners' and their
TDMs' RNG states and the sampled maps -- over several closed-loop rounds; launch counts; every rejection path."""
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


# ----------------------------------------------------------------------------- planners and their state
def map_planner(E, sc, k):
    """One det / speed-map planner of scenario `sc`, varied by its index k (lambda, u_std, warm start)."""
    with _quiet():
        cfg = E.Config(**sc["cfg"])
        lin, ang = E.TDM_Numba(cfg), E.TDM_Numba(cfg)
        lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        pl = E.MPPI_Numba(cfg)
    params = dict(sc["params"])
    params["lambda_weight"] = [1.0, 0.5, 2.0, 0.8, 1.3][k % 5]
    params["u_std"] = np.array([2.0, 3.0]) * (1.0 + 0.1 * (k % 7))
    pl.setup(params, lin, ang)
    if "u0" in sc:
        pl.u_cur_d.copy_to_device(sc["u0"])
    return pl


def map_scenario(mode, k, N=256, T=24, H=48, res=0.2, B=6, det_alpha=1.0, num_opt=1):
    sc = make_scenario(mode, N=N, M=1, T=T, H=H, W=H, res=res, B=B, seed=11 + 7 * k, det_alpha=det_alpha,
                       warm_start=(k % 2 == 1))
    sc["params"]["num_opt"] = num_opt
    return sc


def barebone_planner(E, k, N=300, T=20, num_opt=1):
    from mppi_numba_b200 import barebone as BB
    with _quiet():
        pl = BB.MPPI_Numba(BB.Config(T=T * 0.1 + 0.05, dt=0.1, num_control_rollouts=N, num_vis_state_rollouts=4,
                                     seed=3 + k))
    rng = np.random.default_rng(40 + k)
    params = dict(dt=0.1, x0=np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(-np.pi, np.pi)]),
                  xgoal=np.array([6.0 + k, 4.0 - 0.5 * k]), goal_tolerance=0.5, dist_weight=10,
                  lambda_weight=[1.0, 0.5, 2.0, 0.8, 1.3][k % 5], num_opt=num_opt,
                  u_std=np.array([1.0, 1.0]) * (1.0 + 0.1 * k), vrange=np.array([0.0, 2.0]),
                  wrange=np.array([-np.pi, np.pi]), obstacle_positions=rng.uniform(1, 5, (1 + k % 3, 2)),
                  obstacle_radius=rng.uniform(0.3, 1.0, 1 + k % 3), obs_penalty=1e6)
    pl.setup(params)
    if k % 2:
        pl.u_cur_d.copy_to_device(np.stack([rng.uniform(0, 2, pl.num_steps), rng.uniform(-1, 1, pl.num_steps)], 1))
    return pl


def planner_launches(E, p):
    n = C.c_int64()
    E._lib.check(E._lib.lib.b200mppi_planner_launch_count(p._handle, C.byref(n)))
    return int(n.value)


def snapshot(p):
    d = dict(u_cur=p.u_cur_d.copy_to_host(), u_prev=p.u_prev_d.copy_to_host(), noise=p.noise_samples_d.copy_to_host(),
             costs=p.costs_d.copy_to_host(), weights=p.weights_d.copy_to_host(), rng=p.rng_states_d.copy_to_host())
    if getattr(p, "lin_tdm", None) is not None:
        for name, t in (("lin", p.lin_tdm), ("ang", p.ang_tdm)):
            d[name + "_rng"] = t.rng_states_d.copy_to_host()
            d[name + "_map"] = t.sample_grid_batch_d.copy_to_host()
    return d


def assert_same(a, b, what):
    assert a.keys() == b.keys()
    for key in a:
        assert np.array_equal(a[key], b[key]), "%s: %s differs" % (what, key)


def batch_vs_sequential(E, make, K, rounds=3):
    """Twins built by make(k); batch solve on one set, K solve() calls on the other, `rounds` closed-loop rounds."""
    with _quiet():
        A = [make(k) for k in range(K)]
        B = [make(k) for k in range(K)]
        batch = E.MPPI_Batch(A)
        for r in range(rounds):
            ub = batch.solve()
            us = np.stack([p.solve() for p in B])
            assert ub.shape == us.shape and ub.dtype == np.float32
            assert np.array_equal(ub, us), "round %d: u differs" % r
            for k in range(K):
                assert_same(snapshot(A[k]), snapshot(B[k]), "round %d planner %d" % (r, k))
            for k in range(K):
                x0 = np.asarray(A[k].params["x0"], dtype=np.float64) + np.array([0.03 * (k + 1), -0.02 * r, 0.05])
                A[k].shift_and_update(x0.copy(), ub[k], 1)
                B[k].shift_and_update(x0.copy(), us[k], 1)
    return A, B, batch


# ----------------------------------------------------------------------------- equality with sequential solves
@pytest.mark.parametrize("mode", ["det", "spd", "barebone"])
def test_batch_equals_sequential_closed_loop(eng, mode):
    if mode == "barebone":
        make = lambda k: barebone_planner(eng, k)                       # noqa: E731
    else:
        scs = [map_scenario(mode, k, det_alpha=0.5 if mode == "det" else 1.0) for k in range(5)]
        make = lambda k: map_planner(eng, scs[k], k)                    # noqa: E731
    A, B, batch = batch_vs_sequential(eng, make, 5)
    # the batch keeps its own launch counter: one launch per stage per round, whatever K
    assert batch.launch_count() == 3 * (3 if mode == "barebone" else 4)
    assert planner_launches(eng, A[0]) == 0 and planner_launches(eng, B[0]) == batch.launch_count()


def test_batch_of_one_and_num_opt_two(eng):
    sc = map_scenario("det", 0)
    batch_vs_sequential(eng, lambda k: map_planner(eng, sc, k), 1, rounds=2)
    scs = [map_scenario("det", k, num_opt=2) for k in range(3)]
    A, B, batch = batch_vs_sequential(eng, lambda k: map_planner(eng, scs[k], k), 3, rounds=2)
    assert batch.launch_count() == 2 * (4 + 3)                          # sampler in the first iteration only
    bb = batch_vs_sequential(eng, lambda k: barebone_planner(eng, k, num_opt=2), 3, rounds=1)[2]
    assert bb.launch_count() == 6
    scs = [map_scenario("det", k, num_opt=0) for k in range(2)]         # maps sampled, u returned unchanged
    A, B, batch = batch_vs_sequential(eng, lambda k: map_planner(eng, scs[k], k), 2, rounds=1)
    assert batch.launch_count() == 1


def test_batch_heterogeneous_map_sizes_take_the_sampler_fallback(eng):
    """Pairs whose map geometry differs from the first pair's are sampled by their own launches: same results,
    one sampler launch more per such pair."""
    scs = [map_scenario("det", k, H=[40, 56, 40, 56][k]) for k in range(4)]
    A, B, batch = batch_vs_sequential(eng, lambda k: map_planner(eng, scs[k], k), 4, rounds=2)
    assert batch.launch_count() == 2 * (1 + (1 + 2) + 1 + 1)
    scs = [map_scenario("det", k, H=48) for k in range(4)]
    A, B, batch = batch_vs_sequential(eng, lambda k: map_planner(eng, scs[k], k), 4, rounds=2)
    assert batch.launch_count() == 2 * 4


def test_batch_launch_count_does_not_grow_with_k(eng):
    """Config-2 shape (N 1024, T 64, 256 x 256, nominal 2-bin maps): K = 16 issues the launches of K = 1."""
    scs = [map_scenario("det", k, N=1024, T=64, H=256, B=2) for k in range(16)]
    with _quiet():
        one = map_planner(eng, scs[0], 0)
        l0 = one.launch_count()
        one.solve()
        single = one.launch_count() - l0
        planners = [map_planner(eng, scs[k], k) for k in range(16)]
        batch = eng.MPPI_Batch(planners)
        assert batch.solve() is not None
    assert single == 4 and batch.launch_count() == single


def test_batch_config4_shape_k32_equals_sequential(eng):
    """Config-4 shape: N 4096, T 128, 512 x 512 PMF, 32 bins, det alpha 0.3; K = 32 planners."""
    scs = [make_scenario("det", N=4096, M=1, T=128, H=512, W=512, res=0.2, B=32, seed=100 + k, det_alpha=0.3,
                         warm_start=(k % 3 == 0)) for k in range(32)]
    batch_vs_sequential(eng, lambda k: map_planner(eng, scs[k], k), 32, rounds=1)


# ----------------------------------------------------------------------------- rejections
def _raw_create(L, pls):
    arr = (C.c_void_p * len(pls))(*[(p._handle.value if p is not None else None) for p in pls])
    h = C.c_void_p()
    rc = L.lib.b200mppi_batch_create(arr, len(pls), C.byref(h))
    return rc, L.lib.b200mppi_last_error().decode(), h


def test_batch_rejections_launch_nothing_and_leave_state_untouched(eng, capsys):
    L = eng._lib
    scs = [map_scenario("det", k) for k in range(3)]
    with _quiet():
        dets = [map_planner(eng, scs[k], k) for k in range(3)]
        spd = map_planner(eng, map_scenario("spd", 0), 0)
        other_n = map_planner(eng, map_scenario("det", 5, N=128), 0)
        other_t = map_planner(eng, map_scenario("det", 5, T=20), 0)
        tdm_sc = make_scenario("tdm", N=256, M=4, T=24, H=48, W=48, res=0.2, B=6, seed=2)
        tdm = map_planner(eng, tdm_sc, 0)
    for p in dets:
        p.move_mppi_task_vars_to_device()
    for pls, want in (([dets[0], tdm], "planner 1 is MODE_TDM: the stochastic mode is not batched"),
                      ([dets[0], spd], "planner 1 has mode 2, planner 0 mode 1"),
                      ([dets[0], other_n], "planner 1 has num_control_rollouts 128"),
                      ([dets[0], other_t], "planner 1 has num_steps 20"),
                      ([dets[0], dets[1], dets[0]], "planner 2 is planner 0 again"),
                      ([dets[0], None], "planner 1 is null")):
        rc, msg, h = _raw_create(L, pls)
        assert rc == -1                                                        # B200MPPI_EINVAL
        assert want in msg, msg
        assert not h.value
    rc, msg, _ = _raw_create(L, [])
    assert rc == -1 and "count < 1" in msg
    # a single-rank batch only: a planner built as rank 0 of 2
    pod = L.ConfigPOD(num_steps=24, num_control_rollouts=256, num_grid_samples=1, max_map_rows=60, max_map_cols=60,
                      tdm_thread_x=16, tdm_thread_y=16, num_vis_state_rollouts=1, mode=L.MODE_DET_DYN, device=0,
                      rank=0, world_size=2, seed=1)
    hr = C.c_void_p()
    L.check(L.lib.b200mppi_planner_create(C.byref(pod), C.byref(hr)))
    try:
        arr = (C.c_void_p * 2)(dets[0]._handle.value, hr.value)
        h = C.c_void_p()
        assert L.lib.b200mppi_batch_create(arr, 2, C.byref(h)) == -1
        assert "planner 1 has world_size 2" in L.lib.b200mppi_last_error().decode()
    finally:
        L.lib.b200mppi_planner_destroy(hr)
    # Python constructor errors
    for pls, want in (([dets[0], tdm], "stochastic mode is not batched"), ([dets[0], spd], "cannot be mixed")):
        with pytest.raises(ValueError, match=want):
            eng.MPPI_Batch(pls)

    # solve-time rejections: nothing launched, every member's state as before
    before = [snapshot(p) for p in dets]
    counts = [p.launch_count() for p in dets]
    batch = eng.MPPI_Batch(dets)
    dets[2].params["num_opt"] = 2
    with pytest.raises(L.B200MPPIError, match="planner 2 has num_opt 2, planner 0 num_opt 1"):
        batch.solve()
    dets[2].params["num_opt"] = 1
    own_ang = dets[1].ang_tdm
    dets[1].ang_tdm = dets[0].ang_tdm                                          # two planners share a TDM
    with pytest.raises(L.B200MPPIError, match="planners 0 and 1 share a TDM"):
        batch.solve()
    dets[1].ang_tdm = own_ang
    for p in dets:
        p.move_mppi_task_vars_to_device()
    assert batch.launch_count() == 0
    for k, p in enumerate(dets):
        assert p.launch_count() == counts[k]
        assert_same(snapshot(p), before[k], "planner %d after a rejected solve" % k)
    # a member that fails its preconditions: None and the reason, nothing solved
    dets[2].params_set = False
    capsys.readouterr()
    assert batch.solve() is None
    out = capsys.readouterr().out
    assert "MPPI parameters are not set" in out and "planner 2" in out
    assert batch.launch_count() == 0
