"""MPPI_Batch without a GPU: the C-ABI of the batched solve (exports, prototypes as the header declares them) and the
Python layer through a fake backend (tests/fake_backend.py) -- constructor validation, the print-and-return-None
convention when a member's preconditions fail, the params POD every member uploads before the one batched call, and
the re-pointing of u_prev_d afterwards."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.fake_backend import FakeLib, disarm
from tests.scenarios import make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH_SYMBOLS = ("b200mppi_batch_create", "b200mppi_batch_destroy", "b200mppi_batch_set_stream",
                 "b200mppi_batch_solve", "b200mppi_batch_launch_count")


# ----------------------------------------------------------------------------- C-ABI
def test_batch_symbols_exported_with_header_prototypes(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    raw = C.CDLL(_lib.LIB_PATH)
    for name in BATCH_SYMBOLS:
        assert hasattr(raw, name), name
        assert name in _lib.EXPORTS
    # the header's prototypes, checked by the C compiler against the exact function-pointer types
    src = tmp_path / "proto.c"
    src.write_text("""
#include "b200mppi.h"
int (*f_create)(b200mppi_planner* const*, int32_t, b200mppi_batch**) = b200mppi_batch_create;
int (*f_destroy)(b200mppi_batch*) = b200mppi_batch_destroy;
int (*f_stream)(b200mppi_batch*, void*) = b200mppi_batch_set_stream;
int (*f_solve)(b200mppi_batch*, float*) = b200mppi_batch_solve;
int (*f_count)(b200mppi_batch*, int64_t*) = b200mppi_batch_launch_count;
""")
    r = subprocess.run(["gcc", "-c", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                        str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # ... and the ctypes prototypes say the same
    P, I32, I64 = C.c_void_p, C.c_int32, C.c_int64
    want = {"b200mppi_batch_create": [C.POINTER(P), I32, C.POINTER(P)], "b200mppi_batch_destroy": [P],
            "b200mppi_batch_set_stream": [P, P], "b200mppi_batch_solve": [P, P],
            "b200mppi_batch_launch_count": [P, C.POINTER(I64)]}
    for name, args in want.items():
        fn = getattr(_lib.lib, name)
        assert fn.restype is C.c_int and list(fn.argtypes) == args, name


def test_batch_create_validates_before_touching_the_gpu():
    """Argument errors are reported without a device (count, null planner)."""
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    h = C.c_void_p()
    assert _lib.lib.b200mppi_batch_create((C.c_void_p * 1)(), 0, C.byref(h)) == -1
    assert "count < 1" in _lib.lib.b200mppi_last_error().decode()
    assert _lib.lib.b200mppi_batch_create((C.c_void_p * 2)(None, None), 2, C.byref(h)) == -1
    assert "planner 0 is null" in _lib.lib.b200mppi_last_error().decode()
    assert not h.value


# ----------------------------------------------------------------------------- Python layer on a fake backend
class BatchFake(FakeLib):
    """FakeLib that also records every params POD in call order and plays the batched solve."""

    def __init__(self):
        super().__init__()
        self.pods = []
        self.members = None

    def b200mppi_planner_set_params(self, h, pod):
        rc = super().b200mppi_planner_set_params(h, pod)
        self.pods.append((h.value, dict(self.uploads["set_params"])))
        return rc

    def b200mppi_batch_create(self, arr, n, out):
        self.members = [arr[i] for i in range(n)]
        self.calls.append(("batch_create", (n,)))
        return self._handle_out(out)

    def b200mppi_batch_solve(self, h, u):
        n = len(self.members)
        self.calls.append(("batch_solve", (n,)))
        addr = u.value if isinstance(u, C.c_void_p) else C.cast(u, C.c_void_p).value
        if addr:
            T = self.T
            fill = np.arange(n * T * 2, dtype=np.float32)
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
    fake = BatchFake()
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    made = []
    real_init = BT.MPPI_Batch.__init__

    def init(self, planners):
        made.append(self)
        real_init(self, planners)
    monkeypatch.setattr(BT.MPPI_Batch, "__init__", init)
    yield E, fake
    for b in made:                                   # fake handles must never reach the real destroy function
        b._handle = None
    disarm(fake)


def det_planner(E, k, mode="det", **cfg_extra):
    sc = make_scenario(mode, N=100, M=1, T=10, H=20, W=20, res=0.25, B=4, seed=5 + k)
    cfg = E.Config(**dict(sc["cfg"], **cfg_extra))
    lin, ang = E.TDM_Numba(cfg), E.TDM_Numba(cfg)
    lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    pl = E.MPPI_Numba(cfg)
    params = dict(sc["params"], lambda_weight=0.5 + k, u_std=np.array([1.0 + k, 2.0]))
    pl.setup(params, lin, ang)
    return pl


def barebone_planner(k):
    from mppi_numba_b200 import barebone as BB
    pl = BB.MPPI_Numba(BB.Config(T=1.0, dt=0.1, num_control_rollouts=100, seed=k))
    pl.setup(dict(dt=0.1, x0=np.array([0.0, 0.0, 0.1 * k]), xgoal=np.array([5.0, k]), goal_tolerance=0.5,
                  lambda_weight=1.0 + k, num_opt=1, u_std=np.array([1.0, 1.0]), vrange=np.array([0.0, 2.0]),
                  wrange=np.array([-np.pi, np.pi])))
    return pl


def test_constructor_rejections(host, capsys):
    E, fake = host
    det = det_planner(E, 0)
    with pytest.raises(ValueError, match="planner 1 uses use_tdm: the stochastic mode is not batched"):
        E.MPPI_Batch([det, det_planner(E, 1, mode="tdm")])
    with pytest.raises(ValueError, match="planner 1 is a spd planner, planner 0 a det planner"):
        E.MPPI_Batch([det, det_planner(E, 1, mode="spd")])
    with pytest.raises(ValueError, match="planner 1 is a barebone planner, planner 0 a det planner"):
        E.MPPI_Batch([det, barebone_planner(1)])
    sc = make_scenario("det", N=100, M=1, T=10, H=20, W=20, res=0.25, B=4, seed=9)
    ranked = E.MPPI_Numba(E.Config(**sc["cfg"]), rank=0, world_size=2)
    with pytest.raises(ValueError, match="planner 1 has world_size 2"):
        E.MPPI_Batch([det, ranked])
    with pytest.raises(ValueError, match="no planners"):
        E.MPPI_Batch([])
    assert "batch_create" not in fake.names()


@pytest.mark.parametrize("kind", ["det", "spd", "barebone"])
def test_solve_uploads_every_members_pod_then_one_call(host, kind):
    E, fake = host
    pls = [barebone_planner(k) if kind == "barebone" else det_planner(E, k, mode=kind) for k in range(3)]
    batch = E.MPPI_Batch(pls)
    assert fake.members == [p._handle.value for p in pls]
    fake.T = pls[0].num_steps
    for p in pls:
        p.u_prev_d = None                            # re-pointed by the batch solve as by solve()
    fake.pods.clear()
    u = batch.solve()
    assert u.shape == (3, pls[0].num_steps, 2) and u.dtype == np.float32
    assert np.array_equal(u.ravel(), np.arange(u.size, dtype=np.float32))
    assert [h for h, _ in fake.pods] == [p._handle.value for p in pls]
    for p, (_, pod) in zip(pls, fake.pods):
        assert pod["lambda_weight"] == np.float32(p.params["lambda_weight"])
        assert pod["x0"] == [np.float32(v) for v in p.params["x0"]]
        assert pod["u_std"] == [np.float32(v) for v in p.params["u_std"]]
        assert pod["num_opt"] == 1
        assert p.u_prev_d is p._u_prev_buf
    names = fake.names()
    assert names.count("batch_solve") == 1 and "planner_solve" not in names
    assert names.index("batch_solve") > max(i for i, n in enumerate(names) if n == "planner_set_params")


def test_failed_member_precondition_prints_index_and_returns_none(host, capsys):
    E, fake = host
    pls = [det_planner(E, k) for k in range(3)]
    batch = E.MPPI_Batch(pls)
    pls[1].params_set = False
    fake.pods.clear()
    capsys.readouterr()
    assert batch.solve() is None
    out = capsys.readouterr().out
    assert "MPPI parameters are not set. Cannot solve" in out
    assert "MPPI_Batch: planner 1: MPPI solve condition not met" in out
    assert "batch_solve" not in fake.names() and not fake.pods        # nothing uploaded, nothing solved
    pls[1].params_set = True
    pls[2].params["x0"] = np.array([-50.0, 0.0, 0.0])                 # outside the padded map
    capsys.readouterr()
    assert batch.solve() is None
    out = capsys.readouterr().out
    assert "not within padded xlimits" in out and "planner 2" in out
