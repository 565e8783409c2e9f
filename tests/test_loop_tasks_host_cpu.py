"""A device loop's task updates without a GPU: ``set_goals`` and ``set_obstacles`` marshalled on a fake backend --
shape, dtype, stride and device refusals before anything is issued, the obstacle capacity (``max_obstacles``) and its
refusals, ``set_obstacles`` refused on det, use_tdm and mixed loops, and what close commits into each planner's params
(float64 goals as taken, float32 goals widened, obstacle sets as (n, 2) positions and (n,) radii, planners that took
nothing untouched) and the "bad_obstacles" status."""
import ctypes as C
import types

import numpy as np
import pytest

from tests.fake_backend import disarm
from tests.test_batch_host_cpu import barebone_planner, det_planner
from tests.test_device_loop_host_cpu import Arr, LoopFake
from tests.test_mixed_batch_host_cpu import MixedFake
from tests.test_stochastic_batch_host_cpu import planner as tdm_planner

GOAL64, GOAL32 = 0.1, float(np.float32(0.1))


class TaskFake(LoopFake, MixedFake):
    """LoopFake with the task entry points: records their arguments; the capacity is max(max_obstacles, cap0); close_ex
    reports planner 0 with a float64 goal and two obstacles, planner 1 with a float32 goal (widened), no obstacles and
    status bad_obstacles, and every other planner with nothing taken."""

    cap0 = 2
    max_obstacles = 0

    def b200mppi_batch_create_stochastic(self, arr, n, out):
        self.members = [arr[i] for i in range(n)]
        return self._handle_out(out)

    def b200mppi_batch_loop_open(self, h, kind, limits, rows, out):
        self.max_obstacles = 0
        return super().b200mppi_batch_loop_open(h, kind, limits, rows, out)

    def b200mppi_batch_loop_open_ex(self, h, kind, limits, rows, max_obstacles, out):
        self.max_obstacles = max_obstacles
        self.calls.append(("loop_open_ex", (kind, max_obstacles)))
        return self._handle_out(out)

    def b200mppi_loop_obstacle_capacity(self, h, cap):
        cap._obj.value = self.capacity()
        return 0

    def capacity(self):
        return max(self.max_obstacles, self.cap0)

    def b200mppi_loop_set_goals(self, h, g, dtype, stride):
        self.calls.append(("loop_set_goals", (g.value, dtype, stride)))
        return 0

    def b200mppi_loop_set_obstacles(self, h, obs, dtype, count, stride, counts):
        self.calls.append(("loop_set_obstacles", (obs.value, dtype, count, stride, counts.value if counts else None)))
        return 0

    def b200mppi_loop_close_ex(self, h, S, tasks, obs):
        self.b200mppi_loop_close(h, S)
        self.calls[-1] = ("loop_close_ex", ())
        K = len(self.members)
        S[1].status = 6
        tasks[0].took_goal, tasks[0].goal[:] = 1, [GOAL64, -2.5]
        tasks[1].took_goal, tasks[1].goal[:] = 1, [GOAL32, 3.0]
        tasks[0].took_obstacles, tasks[0].num_obstacles = 1, 2
        tasks[1].took_obstacles, tasks[1].num_obstacles = 1, 0
        if obs:
            O = self.capacity()
            a = np.arange(K * O * 3, dtype=np.float64).reshape(K, O, 3) + GOAL64
            C.memmove(obs.value, a.ctypes.data, a.nbytes)
        return 0


@pytest.fixture()
def host(monkeypatch):
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    import mppi_numba_b200.barebone as B
    import mppi_numba_b200.batch as BT
    import mppi_numba_b200.mppi as M
    import mppi_numba_b200.terrain as T
    fake = TaskFake()
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    yield E, fake
    import gc
    for obj in gc.get_objects():                       # fake handles must never reach the real destroy functions
        if isinstance(obj, (BT.MPPI_Batch, BT.DeviceLoop)):
            h = getattr(obj, "_handle", None)
            if h is not None and getattr(h, "value", None) in fake.issued:
                obj._handle = None
    disarm(fake)


def last(fake, name):
    return [a for n, a in fake.calls if n == name][-1]


def det_batch(E, fake, K=3):
    pls = [det_planner(E, k) for k in range(K)]
    fake.T = pls[0].num_steps
    return E.MPPI_Batch(pls), pls


def bb_batch(E, fake, K=3):
    pls = [barebone_planner(k) for k in range(K)]
    fake.T = pls[0].num_steps
    return E.MPPI_Batch(pls), pls


def test_set_goals_marshalling_and_refusals(host):
    E, fake = host
    batch, _ = det_batch(E, fake)
    with batch.device_loop() as loop:
        loop.set_goals(Arr((3, 2), "<f8"))
        assert last(fake, "loop_set_goals") == (0x7000, 0, 16)
        loop.set_goals(Arr((3, 2), "<f4", data=0x7100))
        assert last(fake, "loop_set_goals") == (0x7100, 1, 8)
        loop.set_goals(Arr((3, 2), "<f8", strides=(32, 8)))             # g[:, :2] of a (3, 4) array
        assert last(fake, "loop_set_goals") == (0x7000, 0, 32)
        n = len(fake.calls)
        for bad, what in ((Arr((3, 2), "<f8", strides=(32, 16)), "strides"), (Arr((3, 3), "<f8"), "shape"),
                          (Arr((2, 2), "<f8"), "shape"), (Arr((3, 2), "<i4"), "dtype"),
                          (Arr((3, 2), "<f8", device=types.SimpleNamespace(type="cuda", index=1)), "device"),
                          (Arr((3, 2), "<f8", device=types.SimpleNamespace(type="cpu", index=None)), "device")):
            with pytest.raises(ValueError, match=what):
                loop.set_goals(bad)
        with pytest.raises(TypeError, match="cuda_array_interface"):
            loop.set_goals(np.zeros((3, 2)))
        assert len(fake.calls) == n, "a refused call issued something"
        loop.set_goals(Arr((3, 2), "<f8", stream=0x6000))
        assert fake.calls[-2] == ("loop_wait", (0x6000,)) and fake.calls[-1][0] == "loop_set_goals"
    for call in (lambda: loop.set_goals(Arr((3, 2), "<f8")), lambda: loop.set_obstacles(Arr((3, 1, 3), "<f8"))):
        with pytest.raises(ValueError, match="closed"):
            call()


def test_set_obstacles_marshalling_and_refusals(host):
    E, fake = host
    batch, _ = bb_batch(E, fake, K=2)
    with batch.device_loop(max_obstacles=4) as loop:
        assert loop.max_obstacles == 4
        loop.set_obstacles(Arr((2, 3, 3), "<f8"))
        assert last(fake, "loop_set_obstacles") == (0x7000, 0, 3, 72, None)
        loop.set_obstacles(Arr((2, 4, 3), "<f4"), Arr((2,), "<i4", data=0x8000))
        assert last(fake, "loop_set_obstacles") == (0x7000, 1, 4, 48, 0x8000)
        loop.set_obstacles(Arr((2, 1, 3), "<f4", strides=(64, 12, 4)))  # planner rows 64 bytes apart
        assert last(fake, "loop_set_obstacles") == (0x7000, 1, 1, 64, None)
        loop.set_obstacles(Arr((2, 0, 3), "<f8", data=0))                  # no obstacles for anyone
        assert last(fake, "loop_set_obstacles") == (None, 0, 0, 0, None)
        n = len(fake.calls)
        for bad, counts, what in ((Arr((2, 5, 3), "<f8"), None, "capacity is 4"),
                                  (Arr((2, 3, 2), "<f8"), None, "shape"), (Arr((3, 3, 3), "<f8"), None, "shape"),
                                  (Arr((2, 3), "<f8"), None, "shape"), (Arr((2, 3, 3), "<i4"), None, "dtype"),
                                  (Arr((2, 3, 3), "<f8", strides=(72, 32, 8)), None, "strides"),
                                  (Arr((2, 3, 3), "<f8"), Arr((2,), "<i8"), "dtype"),
                                  (Arr((2, 3, 3), "<f8"), Arr((3,), "<i4"), "shape"),
                                  (Arr((2, 3, 3), "<f8", device=types.SimpleNamespace(type="cuda", index=1)), None,
                                   "device")):
            with pytest.raises(ValueError, match=what):
                loop.set_obstacles(bad, counts)
        with pytest.raises(TypeError, match="cuda_array_interface"):
            loop.set_obstacles(np.zeros((2, 3, 3)))
        assert len(fake.calls) == n, "a refused call issued something"


def test_capacity_rule(host):
    E, fake = host
    batch, _ = bb_batch(E, fake, K=2)
    with batch.device_loop() as loop:                  # max_obstacles 0: the plain open, which equals open_ex with 0
        assert fake.calls[-1][0] == "loop_open" and "loop_open_ex" not in fake.names()
        assert loop.max_obstacles == fake.cap0         # the largest obstacle count of the planners, from the library
    with batch.device_loop(max_obstacles=5) as loop:
        assert last(fake, "loop_open_ex") == (2, 5) and loop.max_obstacles == 5
        with pytest.raises(ValueError, match="capacity is 5"):
            loop.set_obstacles(Arr((2, 6, 3), "<f8"))
    with pytest.raises(ValueError, match="max_obstacles -1"):
        batch.device_loop(max_obstacles=-1)
    det, _ = det_batch(E, fake)
    n = len(fake.calls)
    with pytest.raises(ValueError, match="barebone"):
        det.device_loop(max_obstacles=3)
    assert len(fake.calls) == n and det._loop is None


def test_set_obstacles_refused_on_other_kinds(host):
    E, fake = host
    from tests.test_mixed_batch_host_cpu import planners as mixed_planners
    for make in (lambda: det_batch(E, fake)[0], lambda: E.MPPI_StochasticBatch([tdm_planner(E, k) for k in range(2)]),
                 lambda: E.MPPI_MixedBatch(mixed_planners(E))):
        batch = make()                                 # the fake's members: this batch's
        K = len(batch.planners)
        with batch.device_loop() as loop:
            n = len(fake.calls)
            with pytest.raises(ValueError, match="only barebone planners take obstacles"):
                loop.set_obstacles(Arr((K, 1, 3), "<f8"))
            assert len(fake.calls) == n
            loop.set_goals(Arr((K, 2), "<f8"))        # goals: every kind
            assert fake.calls[-1][0] == "loop_set_goals"


def test_commit_into_params_and_status(host):
    E, fake = host
    batch, pls = bb_batch(E, fake)
    before = [{k: np.array(v, copy=True) if isinstance(v, np.ndarray) else v for k, v in p.params.items()} for p in pls]
    with pytest.raises(KeyError):
        with batch.device_loop(max_obstacles=3) as loop:
            loop.set_goals(Arr((3, 2), "<f4"))
            raise KeyError("plant")
    assert fake.calls[-1] == ("loop_close_ex", ()) and batch._loop is None
    assert loop.status == ["running", "bad_obstacles", "stopped"]
    g0, g1 = pls[0].params["xgoal"], pls[1].params["xgoal"]
    assert g0.dtype == np.float64 and g0.tolist() == [GOAL64, -2.5]
    assert g1.dtype == np.float64 and g1.tolist() == [GOAL32, 3.0] and g1[0] != GOAL64   # the float32 widened
    obs = np.arange(3 * 3 * 3, dtype=np.float64).reshape(3, 3, 3) + GOAL64
    pos, rad = pls[0].params["obstacle_positions"], pls[0].params["obstacle_radius"]
    assert pos.dtype == np.float64 and pos.shape == (2, 2) and pos.tolist() == obs[0, :2, :2].tolist()
    assert rad.dtype == np.float64 and rad.tolist() == obs[0, :2, 2].tolist()
    assert pls[1].params["obstacle_positions"].shape == (0, 2) and pls[1].params["obstacle_radius"].shape == (0,)
    for key in ("xgoal", "obstacle_positions", "obstacle_radius"):      # planner 2 took nothing
        a, b = pls[2].params.get(key), before[2].get(key)
        assert (a is None and b is None) or np.array_equal(a, b)
    # the next host solve uploads what was committed: planner 1 with no obstacles
    with _quiet():
        pls[1].solve()
    assert fake.uploads["set_obstacles"]["rad"].shape == (0,)
    assert fake.uploads["set_params"]["xgoal"] == [np.float32(GOAL32), 3.0]


def test_loop_without_task_calls_closes_as_before(host):
    E, fake = host
    batch, pls = bb_batch(E, fake)
    goals = [p.params["xgoal"].copy() for p in pls]
    with batch.device_loop() as loop:
        loop.solve()
    assert fake.calls[-1] == ("loop_close", ()) and "loop_close_ex" not in fake.names()
    assert all(np.array_equal(p.params["xgoal"], g) for p, g in zip(pls, goals))
    assert "obstacle_positions" not in pls[0].params


def _quiet():
    import contextlib
    import io
    return contextlib.redirect_stdout(io.StringIO())


def test_abi_of_the_task_calls():
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    for name in ("b200mppi_batch_loop_open_ex", "b200mppi_loop_obstacle_capacity", "b200mppi_loop_set_goals",
                 "b200mppi_loop_set_obstacles", "b200mppi_loop_close_ex"):
        assert name in _lib.EXPORTS
    assert C.sizeof(_lib.LoopTask) == 32 and _lib.LoopTask.goal.offset == 16
    L = _lib.lib
    # refusals before any work, without a GPU: null loop and null arguments
    assert L.b200mppi_loop_set_goals(None, None, 0, 16) == _lib.EINVAL
    assert L.b200mppi_loop_set_obstacles(None, None, 0, 0, 0, None) == _lib.EINVAL
    assert L.b200mppi_loop_obstacle_capacity(None, None) == _lib.EINVAL
    assert L.b200mppi_batch_loop_open_ex(None, 2, None, None, 4, None) == _lib.EINVAL
    assert L.b200mppi_loop_close_ex(None, None, None, None) == _lib.EINVAL
