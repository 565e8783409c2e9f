"""MPPI_StochasticBatch without a GPU: the new C-ABI entry point (export, prototype as the header declares it, argument
errors before any device work) and the Python layer through a fake backend -- refusals naming the planner, run_trials
refused, the one batched call after every member's params upload, and u_prev_d left alone."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.fake_backend import FakeLib, disarm
from tests.scenarios import make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_create_stochastic_exported_with_header_prototype(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    name = "b200mppi_batch_create_stochastic"
    assert hasattr(C.CDLL(_lib.LIB_PATH), name) and name in _lib.EXPORTS
    src = tmp_path / "proto.c"
    src.write_text('#include "b200mppi.h"\n'
                   "int (*f)(b200mppi_planner* const*, int32_t, b200mppi_batch**) = b200mppi_batch_create_stochastic;\n")
    r = subprocess.run(["gcc", "-c", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                        str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    fn = getattr(_lib.lib, name)
    assert fn.restype is C.c_int and list(fn.argtypes) == [C.POINTER(C.c_void_p), C.c_int32, C.POINTER(C.c_void_p)]
    h = C.c_void_p()
    assert fn((C.c_void_p * 1)(), 0, C.byref(h)) == -1
    assert "count < 1" in _lib.lib.b200mppi_last_error().decode()
    assert fn((C.c_void_p * 2)(None, None), 2, C.byref(h)) == -1
    assert "batch_create_stochastic: planner 0 is null" in _lib.lib.b200mppi_last_error().decode()
    assert not h.value


class StochasticFake(FakeLib):
    def __init__(self):
        super().__init__()
        self.pods = []
        self.members = None

    def b200mppi_planner_set_params(self, h, pod):
        rc = super().b200mppi_planner_set_params(h, pod)
        self.pods.append(h.value)
        return rc

    def b200mppi_batch_create_stochastic(self, arr, n, out):
        self.members = [arr[i] for i in range(n)]
        self.calls.append(("batch_create_stochastic", (n,)))
        return self._handle_out(out)

    def b200mppi_batch_solve(self, h, u):
        self.calls.append(("batch_solve", (len(self.members),)))
        addr = u.value if isinstance(u, C.c_void_p) else C.cast(u, C.c_void_p).value
        fill = np.arange(len(self.members) * self.T * 2, dtype=np.float32)
        C.memmove(addr, fill.ctypes.data, fill.nbytes)
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
    fake = StochasticFake()
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    made = []
    for cls in (BT.MPPI_Batch, BT.MPPI_StochasticBatch):
        real = cls.__init__

        def init(self, planners, _real=real):
            made.append(self)
            _real(self, planners)
        monkeypatch.setattr(cls, "__init__", init)
    yield E, fake
    for b in made:                                   # fake handles must never reach the real destroy function
        b._handle = None
    disarm(fake)


def planner(E, k, mode="tdm", **cfg_extra):
    sc = make_scenario(mode, N=100, M=8 if mode == "tdm" else 1, T=10, H=20, W=20, res=0.25, B=4, seed=5 + k)
    cfg = E.Config(**dict(sc["cfg"], **cfg_extra))
    lin, ang = E.TDM_Numba(cfg), E.TDM_Numba(cfg)
    lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    pl = E.MPPI_Numba(cfg)
    pl.setup(dict(sc["params"], lambda_weight=0.5 + k), lin, ang)
    return pl


def test_refusals_name_the_planner(host):
    E, fake = host
    tdm = planner(E, 0)
    with pytest.raises(ValueError, match="MPPI_StochasticBatch: planner 1 is a det planner"):
        E.MPPI_StochasticBatch([tdm, planner(E, 1, mode="det")])
    sc = make_scenario("tdm", N=100, M=8, T=10, H=20, W=20, res=0.25, B=4, seed=9)
    ranked = E.MPPI_Numba(E.Config(**sc["cfg"]), rank=0, world_size=2)
    with pytest.raises(ValueError, match="MPPI_StochasticBatch: planner 1 has world_size 2"):
        E.MPPI_StochasticBatch([tdm, ranked])
    with pytest.raises(ValueError, match="no planners"):
        E.MPPI_StochasticBatch([])
    # MPPI_Batch keeps refusing use_tdm planners as before
    with pytest.raises(ValueError, match="planner 1 uses use_tdm: the stochastic mode is not batched"):
        E.MPPI_Batch([planner(E, 2, mode="det"), tdm])
    assert "batch_create_stochastic" not in fake.names() and "batch_create" not in fake.names()


def test_solve_one_call_after_every_upload_and_u_prev_untouched(host, capsys):
    E, fake = host
    pls = [planner(E, k) for k in range(3)]
    batch = E.MPPI_StochasticBatch(pls)
    assert fake.members == [p._handle.value for p in pls] and len(batch) == 3
    fake.T = pls[0].num_steps
    marker = object()
    for p in pls:
        p.u_prev_d = marker
    fake.pods.clear()
    u = batch.solve()
    assert u.shape == (3, pls[0].num_steps, 2) and np.array_equal(u.ravel(), np.arange(u.size, dtype=np.float32))
    assert fake.pods == [p._handle.value for p in pls]
    assert all(p.u_prev_d is marker for p in pls)
    names = fake.names()
    assert names.count("batch_solve") == 1 and "planner_solve" not in names
    pls[1].params_set = False
    capsys.readouterr()
    assert batch.solve() is None
    assert "MPPI_StochasticBatch: planner 1: MPPI solve condition not met" in capsys.readouterr().out
    assert names == fake.names()[:len(names)] and fake.names().count("batch_solve") == 1
    with pytest.raises(ValueError, match="MPPI_StochasticBatch.run_trials: closed-loop trials run det-dynamics"):
        batch.run_trials([None] * 3, 10)
