"""Device loops without a GPU: DeviceLoop's marshalling on a fake backend -- the __cuda_array_interface__ parsing
(dtype, shape, strides, device and stream), what the open hands the library (kind, padded limits, rows), every refusal
while a loop is open and after it closed, the commit when the ``with`` body raises, and what close leaves in Python
(params['x0'] as float64, the u_prev_d alias, solves / shifts / status)."""
import ctypes as C
import types

import numpy as np
import pytest

from tests.fake_backend import disarm
from tests.test_batch_host_cpu import BatchFake, barebone_planner, det_planner

U_PTR, ACT_PTR, STREAM = 0xbeef0000, 0xace00000, 0x5000


class LoopFake(BatchFake):
    """Plays the device-loop entry points: records their arguments; close reports planner k with 2 solves, 1 shift,
    status (running, left_map, stopped)[k % 3] and the last pose (1.5, 2.5, 0.25 k)."""

    def b200mppi_batch_loop_open(self, h, kind, limits, rows, out):
        K = len(self.members)
        lim = None if limits is None else self._bytes(limits, 32 * K, np.float64, (K, 4))
        self.opened = dict(kind=kind, limits=lim, rows=self._bytes(rows, 4 * K, np.int32, (K,)))
        self.calls.append(("loop_open", (kind,)))
        return self._handle_out(out)

    def b200mppi_loop_controls(self, h, u, st):
        u._obj.value, st._obj.value = U_PTR, STREAM
        return 0

    def b200mppi_loop_active(self, h, a):
        a._obj.value = ACT_PTR
        return 0

    def b200mppi_loop_solve(self, h, u):
        self.calls.append(("loop_solve", (u.value,)))
        return 0

    def b200mppi_loop_shift_and_update(self, h, x, dtype, stride):
        self.calls.append(("loop_shift", (x.value, dtype, stride)))
        return 0

    def b200mppi_loop_stop(self, h, m, eb):
        self.calls.append(("loop_stop", (m.value, eb)))
        return 0

    def b200mppi_loop_wait_stream(self, h, s):
        self.calls.append(("loop_wait", (s.value,)))
        return 0

    def b200mppi_loop_close(self, h, S):
        self.calls.append(("loop_close", ()))
        for k in range(len(self.members)):
            S[k].solves, S[k].shifts, S[k].status = 2, 1, (0, 3, 5)[k % 3]
            S[k].x[:] = [1.5, 2.5, 0.25 * k]
        return 0


class Arr(object):
    """A device array seen only through its __cuda_array_interface__."""

    def __init__(self, shape, typestr, strides=None, stream=None, data=0x7000, device=None):
        self.__cuda_array_interface__ = dict(shape=shape, typestr=typestr, data=(data, False), version=3,
                                             strides=strides, stream=stream)
        if device is not None:
            self.device = device


@pytest.fixture()
def host(monkeypatch):
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    import mppi_numba_b200.barebone as B
    import mppi_numba_b200.batch as BT
    import mppi_numba_b200.mppi as M
    import mppi_numba_b200.terrain as T
    fake = LoopFake()
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


def det_batch(E, fake, K=3):
    pls = [det_planner(E, k) for k in range(K)]
    fake.T = pls[0].num_steps
    return E.MPPI_Batch(pls), pls


def last(fake, name):
    return [a for n, a in fake.calls if n == name][-1]


def test_open_marshals_kind_limits_and_rows(host):
    E, fake = host
    batch, pls = det_batch(E, fake)
    with batch.device_loop():
        o = fake.opened
        assert o["kind"] == 0 and o["rows"].tolist() == [0, 1, 2]
        want = [list(p.lin_tdm.padded_xlimits) + list(p.lin_tdm.padded_ylimits) for p in pls]
        assert o["limits"].tolist() == np.asarray(want, np.float64).tolist()
    bb = E.MPPI_Batch([barebone_planner(k) for k in range(2)])
    with bb.device_loop():
        assert fake.opened["kind"] == 2 and fake.opened["limits"] is None


def test_interface_parsing(host):
    E, fake = host
    batch, _ = det_batch(E, fake)
    T = batch.num_steps
    with batch.device_loop() as loop:
        u = loop.solve()
        cai = u.__cuda_array_interface__
        assert cai["shape"] == (3, T, 2) and cai["typestr"] == "<f4" and cai["data"][0] == U_PTR
        assert cai["stream"] == STREAM and last(fake, "loop_solve") == (U_PTR,)
        assert loop.active.__cuda_array_interface__["data"][0] == ACT_PTR
        out = Arr((3, T, 2), "<f4", data=0x9000)
        assert loop.solve(out=out) is out and last(fake, "loop_solve") == (0x9000,)
        loop.shift_and_update(Arr((3, 3), "<f8"))
        assert last(fake, "loop_shift") == (0x7000, 0, 24)
        loop.shift_and_update(Arr((3, 3), "<f4"))
        assert last(fake, "loop_shift") == (0x7000, 1, 12)
        loop.shift_and_update(Arr((3, 3), "<f8", strides=(32, 8)))           # x[:, :3] of a (3, 4) array
        assert last(fake, "loop_shift") == (0x7000, 0, 32)
        n = len(fake.calls)
        for bad, what in ((Arr((3, 3), "<f8", strides=(48, 16)), "strides"), (Arr((3, 4), "<f8"), "shape"),
                          (Arr((2, 3), "<f8"), "shape"), (Arr((3, 3), "<i4"), "dtype"),
                          (Arr((3, 3), "<f8", device=types.SimpleNamespace(type="cuda", index=1)), "device"),
                          (Arr((3, 3), "<f8", device=types.SimpleNamespace(type="cpu", index=None)), "device")):
            with pytest.raises(ValueError, match=what):
                loop.shift_and_update(bad)
        with pytest.raises(TypeError, match="cuda_array_interface"):
            loop.shift_and_update(np.zeros((3, 3)))
        with pytest.raises(ValueError, match="C-contiguous"):
            loop.solve(out=Arr((3, T, 2), "<f4", strides=(T * 8 + 8, 8, 4)))
        assert len(fake.calls) == n, "a refused call issued something"
        loop.shift_and_update(Arr((3, 3), "<f8", stream=0x6000))
        assert fake.calls[-2] == ("loop_wait", (0x6000,)) and fake.calls[-1][0] == "loop_shift"
        loop.stop(Arr((3,), "|b1"))
        assert last(fake, "loop_stop") == (0x7000, 1)
        loop.stop(Arr((3,), "<i4"))
        assert last(fake, "loop_stop") == (0x7000, 4)
        with pytest.raises(ValueError, match="dtype"):
            loop.stop(Arr((3,), "<f4"))


def test_refusals_while_open_and_after_close(host):
    E, fake = host
    batch, pls = det_batch(E, fake)
    p = pls[1]
    with batch.device_loop() as loop:
        for call in (p.solve, lambda: p.set_params(p.params), lambda: p.setup(p.params, p.lin_tdm, p.ang_tdm),
                     lambda: p.shift_and_update(np.zeros(3), np.zeros((batch.num_steps, 2), np.float32)),
                     p.get_state, lambda: p.set_state({}), p.get_state_rollout, lambda: p.lin_tdm.sample_grids(),
                     lambda: p.ang_tdm.set_TDM_from_PMF_grid(None, None)):
            with pytest.raises(ValueError, match="planner 1"):
                call()
        for call in (batch.solve, batch.get_state_rollout, batch.device_loop, lambda: batch.set_stream(0),
                     lambda: batch.run_trials([None] * 3, 5)):
            with pytest.raises(ValueError, match="device loop is open"):
                call()
    for call in (loop.solve, lambda: loop.shift_and_update(Arr((3, 3), "<f8")), lambda: loop.stop(Arr((3,), "<i4"))):
        with pytest.raises(ValueError, match="closed"):
            call()
    loop.close()                                           # idempotent
    assert [n for n, _ in fake.calls].count("loop_close") == 1
    with _quiet():
        assert p.solve() is not None                       # free again


def test_commit_on_exception(host):
    E, fake = host
    batch, pls = det_batch(E, fake)
    with pytest.raises(KeyError):
        with batch.device_loop() as loop:
            loop.solve()
            raise KeyError("plant")
    assert fake.calls[-1] == ("loop_close", ()) and batch._loop is None
    assert loop.solves.tolist() == [2, 2, 2] and loop.shifts.tolist() == [1, 1, 1]
    assert loop.status == ["running", "left_map", "stopped"]
    for k, p in enumerate(pls):
        x0 = p.params["x0"]
        assert isinstance(x0, np.ndarray) and x0.dtype == np.float64 and x0.tolist() == [1.5, 2.5, 0.25 * k]
        assert p.u_prev_d is p._u_prev_buf                 # the u_prev_d alias of a det solve


def _quiet():
    import contextlib
    import io
    return contextlib.redirect_stdout(io.StringIO())


def test_abi_of_the_loop_calls():
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    for name in ("b200mppi_batch_loop_open", "b200mppi_loop_solve", "b200mppi_loop_shift_and_update",
                 "b200mppi_loop_stop", "b200mppi_loop_active", "b200mppi_loop_close", "b200mppi_loop_controls",
                 "b200mppi_loop_wait_stream"):
        assert name in _lib.EXPORTS
    assert C.sizeof(_lib.LoopSummary) == 40 and _lib.LoopSummary.x.offset == 16
