"""Ground-truth realisations drawn on the GPU (run with ``-m gpu``): ``draw_traction_grids`` against the reference
notebook's ``sample_traction_grid`` helper on a twin TDM pair (every plane bit for bit, both TDMs' generator states and
sampled maps afterwards), and every trial call given device realisations against the same call given the twin's host
grids: histories, logs, records, steps_issued, launch counts and every planner and TDM bit for bit.  Refusals issue
nothing."""
import functools
import gc

import numpy as np
import pytest

from tests import test_gpu_mixed_geometry_trials as MG
from tests import test_gpu_shared_tdm as SH
from tests.gpu_harness import assert_same, eng, quiet, snapshot, tdm_pair, tdm_trial_setup, twins  # noqa: F401
from tests.scenarios import make_scenario
from tests.test_gpu_trials import trial_setup

pytestmark = pytest.mark.gpu

S = 16


def gt_pair(E, M=3, H=40, res=0.2, extra=(0, 0), scale=1.0, seed=77):
    """A ground-truth TDM pair (use_tdm, M maps); ``extra`` cells of allocation beyond the padded map (rows, cols);
    bin values and bounds times ``scale``.  Equal arguments give twin pairs."""
    sc = make_scenario("tdm", N=64, M=M, T=8, H=H, W=H, res=res, B=5, seed=seed)
    cfg = dict(sc["cfg"])
    cfg["max_map_dim"] = (cfg["max_map_dim"][0] + extra[0], cfg["max_map_dim"][1] + extra[1])
    td = dict(sc["tdm_dict"], bin_values=sc["tdm_dict"]["bin_values"] * scale,
              bin_values_bounds=sc["tdm_dict"]["bin_values_bounds"] * scale)
    with quiet():
        return tdm_pair(E, E.Config(**cfg), sc["pmf_lin"], sc["pmf_ang"], td)


def helper(E, lin_tdm, ang_tdm):
    """The reference notebook's sample_traction_grid, with the float32 grids NumPy 2 gives widened to float64."""
    lq = lin_tdm.sample_grids().copy_to_host()[0]
    lin = lq * (lin_tdm.bin_values_bounds[1] - lin_tdm.bin_values_bounds[0]) / 100.0 + lin_tdm.bin_values_bounds[0]
    aq = ang_tdm.sample_grids().copy_to_host()[0]
    ang = aq * (ang_tdm.bin_values_bounds[1] - ang_tdm.bin_values_bounds[0]) / 100.0 + ang_tdm.bin_values_bounds[0]
    assert lin.dtype == np.float32 and ang.dtype == np.float32
    return E.TractionGrid(lin.astype(np.float64), ang.astype(np.float64), lin_tdm.res, xlimits=lin_tdm.padded_xlimits,
                          ylimits=lin_tdm.padded_ylimits)


def tdm_state(lin, ang):
    return {n + k: v for n, t in (("lin_", lin), ("ang_", ang))
            for k, v in (("rng", t.rng_states_d.copy_to_host()), ("map", t.sample_grid_batch_d.copy_to_host()))}


def drawn(E, count, **gt):
    """(device set, host grids): count realisations drawn on the GPU from one pair and by the helper on its twin."""
    ga, gb = gt_pair(E, **gt), gt_pair(E, **gt)
    dev = E.draw_traction_grids(ga[0], ga[1], count)
    host = [helper(E, *gb) for _ in range(count)]
    return dev, host


def assert_out_same(a, b, what):
    """Two trial results bit for bit (NaN patterns included)."""
    assert a.keys() == b.keys(), what
    for key in a:
        x, y = a[key], b[key]
        if key == "logs":
            flat = lambda L: [e for s in L for e in (s if isinstance(s, list) else [s])]   # noqa: E731
            for i, (la, lb) in enumerate(zip(flat(x), flat(y))):
                assert (la is None) == (lb is None), (what, i)
                if la is not None:
                    assert_same({k: np.asarray(v) for k, v in la.items()}, {k: np.asarray(v) for k, v in lb.items()},
                                "%s: log %d" % (what, i))
        elif isinstance(x, np.ndarray):
            assert_same({key: x}, {key: y}, what)
        else:
            assert x == y, (what, key)


def check_pair(A, B, out_a, out_b, batch_a, batch_b, what):
    assert_out_same(out_a, out_b, what)
    assert batch_a.steps_issued == batch_b.steps_issued, what
    assert batch_a.launch_count() == batch_b.launch_count(), what
    for k in range(len(A)):
        assert_same(snapshot(A[k]), snapshot(B[k]), "%s: planner %d" % (what, k))
        assert_same(dict(x0=A[k].params["x0"]), dict(x0=B[k].params["x0"]), "%s: planner %d" % (what, k))


# ----------------------------------------------------------------------------- the draw
@pytest.mark.parametrize("count, gt", [(1, dict(M=3)), (3, dict(M=3)), (3, dict(M=1)),
                                       (2, dict(M=2, extra=(5, 11))), (3, dict(M=3, same=True))],
                         ids=["count1", "count3", "m1", "smaller_than_allocation", "lin_is_ang"])
def test_draw_equals_helper(eng, count, gt):
    E = eng
    gt = dict(gt)
    same = gt.pop("same", False)
    ga, gb = gt_pair(E, **gt), gt_pair(E, **gt)
    if same:
        ga, gb = (ga[0], ga[0]), (gb[0], gb[0])
    dev = E.draw_traction_grids(ga[0], ga[1], count)
    assert len(dev) == count
    for i in range(count):
        want = helper(E, *gb)
        g = dev[i]
        lin, ang = g.get_grids()
        assert (g.height, g.width) == want.lin_traction.shape == tuple(ga[0].max_map_dim)
        assert g.res == want.res
        assert np.array_equal(g.xlimits, want.xlimits) and np.array_equal(g.ylimits, want.ylimits)
        assert_same(dict(lin=lin, ang=ang), dict(lin=want.lin_traction, ang=want.ang_traction), "realisation %d" % i)
    assert_same(tdm_state(*ga), tdm_state(*gb), "TDMs after the draw")
    if not same:                                      # the two planes differ: they come from two TDMs
        assert not np.array_equal(*dev[0].get_grids())


# ----------------------------------------------------------------------------- trial calls, device against host
def onemap(E, mode):
    A, B, _ = twins(functools.partial(trial_setup, E, mode), 5)
    return A, B, E.MPPI_Batch


def stochastic(E):
    A, B, _ = twins(functools.partial(tdm_trial_setup, E), 5)
    return A, B, E.MPPI_StochasticBatch


@pytest.mark.parametrize("mode", ["det", "spd", "tdm"])
def test_run_trials(eng, mode):
    E = eng
    A, B, cls = stochastic(E) if mode == "tdm" else onemap(E, mode)
    dev, host = drawn(E, 5, H=64 if mode == "tdm" else 40)
    ba, bb = cls(A), cls(B)
    run = "run_stochastic_trials" if mode == "tdm" else "run_trials"
    with quiet():
        out_a, out_b = getattr(ba, run)(list(dev), S), getattr(bb, run)(host, S)
    check_pair(A, B, out_a, out_b, ba, bb, mode)


@pytest.mark.parametrize("mode, reset_x0", [("det", False), ("det", True), ("tdm", False), ("tdm", True)])
def test_run_trial_sequences(eng, mode, reset_x0):
    """One set of 3 realisations shared by every planner's sequence."""
    E = eng
    A, B, cls = stochastic(E) if mode == "tdm" else onemap(E, mode)
    dev, host = drawn(E, 3, H=64 if mode == "tdm" else 40)
    ba, bb = cls(A), cls(B)
    with quiet():
        out_a = ba.run_trial_sequences([list(dev)] * len(A), S, reset_x0=reset_x0)
        out_b = bb.run_trial_sequences([host] * len(B), S, reset_x0=reset_x0)
    check_pair(A, B, out_a, out_b, ba, bb, "%s reset_x0=%s" % (mode, reset_x0))


@pytest.mark.parametrize("mode", ["det", "tdm"])
def test_record_every(eng, mode):
    E = eng
    A, B, cls = stochastic(E) if mode == "tdm" else onemap(E, mode)
    dev, host = drawn(E, 5, H=64 if mode == "tdm" else 40)
    ba, bb = cls(A), cls(B)
    run = "run_stochastic_trials" if mode == "tdm" else "run_trials"
    with quiet():
        out_a = getattr(ba, run)(list(dev), S, record_every=3)
        out_b = getattr(bb, run)(host, S, record_every=3)
    check_pair(A, B, out_a, out_b, ba, bb, mode)


def test_share_tdms(eng):
    E = eng
    sc = make_scenario("tdm", N=200, M=24, T=20, H=64, W=64, res=0.2, B=5, seed=41)
    goals = SH.GOALS
    A = SH.build(E, sc, 5, True, goals=goals)
    B = SH.build(E, sc, 5, True, goals=goals)
    dev, host = drawn(E, 5, H=64)
    ba, bb = E.MPPI_StochasticBatch(A, share_tdms=True), E.MPPI_StochasticBatch(B, share_tdms=True)
    with quiet():
        out_a, out_b = ba.run_stochastic_trials(list(dev), S), bb.run_stochastic_trials(host, S)
    check_pair(A, B, out_a, out_b, ba, bb, "share_tdms")


@pytest.mark.parametrize("mode", ["det", "tdm"])
def test_mixed_geometry(eng, mode):
    """Planners on maps of several sizes and resolutions, every one on the same realisation; most planners' maps differ
    from the ground truth's."""
    E = eng
    A, B = MG.build(E, mode, MG.SPECS), MG.build(E, mode, MG.SPECS)
    dev, host = drawn(E, 1, H=40)
    cls = E.MPPI_StochasticBatch if mode == "tdm" else E.MPPI_Batch
    ba, bb = cls(A), cls(B)
    run = "run_stochastic_trials" if mode == "tdm" else "run_trials"
    with quiet():
        out_a = getattr(ba, run)([dev[0]] * len(A), S)
        out_b = getattr(bb, run)([host[0]] * len(B), S)
    check_pair(A, B, out_a, out_b, ba, bb, mode)


def test_episode_leaves_the_map(eng):
    """Tractions up to 60: the robots are thrown off their maps."""
    E = eng
    A, B, cls = onemap(E, "det")
    dev, host = drawn(E, 5, H=40, scale=60.0)
    ba, bb = cls(A), cls(B)
    with quiet():
        out_a, out_b = ba.run_trials(list(dev), S), bb.run_trials(host, S)
    assert "left_map" in out_a["status"]
    check_pair(A, B, out_a, out_b, ba, bb, "left map")


def test_planner_beyond_the_ground_truth_plane(eng):
    """A ground-truth plane of 8 x 8 cells at 0.5 m ([-0.5, 3.5] a side) under planners whose padded maps reach 8.6 m
    and who start about 4 m from the origin: poses beyond the plane read no traction (the plant's bounds test), as with
    the host grids of that plane, while the stop rule keeps the planners' own limits."""
    E = eng
    A, B, cls = onemap(E, "det")
    dev, host = drawn(E, 5, H=6, res=0.5)
    assert (dev[0].height, dev[0].width) == (8, 8) and dev[0].xlimits[1] - dev[0].xlimits[0] == 4.0
    ba, bb = cls(A), cls(B)
    with quiet():
        out_a, out_b = ba.run_trials(list(dev), S), bb.run_trials(host, S)
    x = out_a["xhist"]
    beyond = (x[..., 0] >= dev[0].xlimits[1]) | (x[..., 1] >= dev[0].ylimits[1])
    assert beyond.any(), "no pose beyond the plane: the case does not test reads past it"
    check_pair(A, B, out_a, out_b, ba, bb, "beyond the plane")


def test_one_set_across_calls_and_mixed_grids(eng):
    """One set for every planner of a one-map batch, then a stochastic batch, then the first batch again; then host and
    device grids in one call."""
    E = eng
    A1, B1, _ = onemap(E, "det")
    A2, B2, _ = stochastic(E)
    dev, host = drawn(E, 2, H=64)
    ba1, bb1 = E.MPPI_Batch(A1), E.MPPI_Batch(B1)
    ba2, bb2 = E.MPPI_StochasticBatch(A2), E.MPPI_StochasticBatch(B2)
    with quiet():
        for r, (ba, bb, run, A, B) in enumerate([(ba1, bb1, "run_trials", A1, B1),
                                                 (ba2, bb2, "run_stochastic_trials", A2, B2),
                                                 (ba1, bb1, "run_trials", A1, B1)]):
            out_a = getattr(ba, run)([dev[r % 2]] * len(A), S)
            out_b = getattr(bb, run)([host[r % 2]] * len(B), S)
            check_pair(A, B, out_a, out_b, ba, bb, "round %d" % r)
        mixed_a = [dev[0], host[1], dev[1], host[0], dev[0]]
        mixed_b = [host[0], host[1], host[1], host[0], host[0]]
        out_a, out_b = ba1.run_trials(mixed_a, S), bb1.run_trials(mixed_b, S)
    check_pair(A1, B1, out_a, out_b, ba1, bb1, "mixed")


# ----------------------------------------------------------------------------- refusals
def refused(E, batch, A, grids, match):
    before = [snapshot(p) for p in A]
    count = batch.launch_count()
    with quiet(), pytest.raises(E.B200MPPIError, match=match):
        batch.run_trials(grids, S)
    assert batch.launch_count() == count
    for k, p in enumerate(A):
        assert_same(snapshot(p), before[k], "planner %d" % k)


def test_refusals(eng):
    E = eng
    A, _, cls = onemap(E, "det")
    batch = cls(A)
    dev, _ = drawn(E, 2, H=40)
    g = dev[1]
    grids = [dev[0]] * len(A)
    # device memory that is no realisation: a TDM's sample buffer
    other = A[0].lin_tdm.sample_grid_batch_d.__cuda_array_interface__["data"][0]
    g._lin_ptr, saved = other, g._lin_ptr
    refused(E, batch, A, grids[:2] + [g] + grids[3:], "device memory but not a plane")
    g._lin_ptr = saved
    # the middle of a plane
    g._ang_ptr, saved = g._ang_ptr + 8, g._ang_ptr
    refused(E, batch, A, grids[:3] + [g] + grids[4:], "middle of a realisation plane")
    g._ang_ptr = saved
    # a destroyed set
    gone = E.draw_traction_grids(*gt_pair(E, H=40), 1)
    ptrs = gone[0]._lin_ptr, gone[0]._ang_ptr
    del gone
    gc.collect()
    g._lin_ptr, g._ang_ptr = ptrs
    refused(E, batch, A, grids[:4] + [g], "destroyed realisation set")


def test_refusal_other_device(eng):
    E = eng
    if E.device_count() < 2:
        pytest.skip("one GPU: a realisation set on another device needs a second one")
    A, _, cls = onemap(E, "det")
    batch = cls(A)
    sc = make_scenario("tdm", N=64, M=2, T=8, H=40, W=40, res=0.2, B=5, seed=77)
    with quiet():
        lin, ang = E.TDM_Numba(E.Config(**sc["cfg"]), device=1), E.TDM_Numba(E.Config(**sc["cfg"]), device=1)
        lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"])
        ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"])
    dev = E.draw_traction_grids(lin, ang, 1)
    refused(E, batch, A, [dev[0]] * len(A), "on device 1")


def test_python_refusals(eng):
    E = eng
    lin, ang = gt_pair(E, H=40)
    with pytest.raises(ValueError, match="count 0 < 1"):
        E.draw_traction_grids(lin, ang, 0)
    before = tdm_state(lin, ang)
    lin.reset()
    with pytest.raises(ValueError, match="lin_tdm has no PMF grid set"):
        E.draw_traction_grids(lin, ang, 1)
    assert_same(tdm_state(lin, ang), before, "TDMs after a refusal")
