"""Batches whose planners share TDM pairs (share_tdms=True), without a GPU: the new C-ABI entry point (export and
prototype as the header declares it) and the Python layer through a fake backend -- the setter called only when asked
for, the default leaving shared pairs to the library's refusal, and the overlaps sharing refuses (partial overlap,
unequal alpha_dyn on one stochastic pair) refused before any work, naming both planners."""
import ctypes as C
import os
import subprocess

import pytest

from tests.fake_backend import FakeLib, disarm
from tests.scenarios import make_scenario

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_share_tdms_exported_with_header_prototype(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    name = "b200mppi_batch_share_tdms"
    assert hasattr(C.CDLL(_lib.LIB_PATH), name) and name in _lib.EXPORTS
    src = tmp_path / "proto.c"
    src.write_text('#include "b200mppi.h"\nint (*f)(b200mppi_batch*, int32_t) = b200mppi_batch_share_tdms;\n')
    r = subprocess.run(["gcc", "-c", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                        str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    fn = getattr(_lib.lib, name)
    assert fn.restype is C.c_int and list(fn.argtypes) == [C.c_void_p, C.c_int32]
    assert fn(None, 1) == -1 and "null batch" in _lib.lib.b200mppi_last_error().decode()


class ShareFake(FakeLib):
    def __init__(self):
        super().__init__()
        self.members = None
        self.shared = []

    def _create(self, name, arr, n, out):
        self.members = [arr[i] for i in range(n)]
        self.calls.append((name, (n,)))
        return self._handle_out(out)

    def b200mppi_batch_create(self, arr, n, out):
        return self._create("batch_create", arr, n, out)

    def b200mppi_batch_create_stochastic(self, arr, n, out):
        return self._create("batch_create_stochastic", arr, n, out)

    def b200mppi_batch_share_tdms(self, h, enable):
        self.shared.append(int(enable))
        self.calls.append(("batch_share_tdms", (int(enable),)))
        return 0

    def b200mppi_batch_solve(self, h, u):
        self.calls.append(("batch_solve", (len(self.members),)))
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
    fake = ShareFake()
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    made = []
    for cls in (BT.MPPI_Batch, BT.MPPI_StochasticBatch):
        real = cls.__init__

        def init(self, planners, share_tdms=False, _real=real):
            made.append(self)
            _real(self, planners, share_tdms=share_tdms)
        monkeypatch.setattr(cls, "__init__", init)
    yield E, fake
    for b in made:                                   # fake handles must never reach the real destroy function
        b._handle = None
    disarm(fake)


def planners(E, mode, K, pair=None, seed=5):
    """K set-up planners of one scenario; pair: (lin, ang) every planner is set up with (else each its own)."""
    sc = make_scenario(mode, N=100, M=8 if mode == "tdm" else 1, T=10, H=20, W=20, res=0.25, B=4, seed=seed)
    cfg = E.Config(**sc["cfg"])
    out = []
    for k in range(K):
        if pair is None or k == 0:
            lin, ang = E.TDM_Numba(cfg), E.TDM_Numba(cfg)
            lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
            ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
            pair = (lin, ang) if pair is not None else None
        else:
            lin, ang = pair
        pl = E.MPPI_Numba(cfg)
        pl.setup(dict(sc["params"], lambda_weight=0.5 + k), lin, ang)
        out.append(pl)
    return out


@pytest.mark.parametrize("mode", ["det", "tdm"])
def test_setter_called_only_when_asked(host, mode):
    E, fake = host
    cls = E.MPPI_StochasticBatch if mode == "tdm" else E.MPPI_Batch
    pls = planners(E, mode, 3, pair=True)
    batch = cls(pls)                                  # the default: no setter call, the library refuses shared pairs
    assert fake.shared == [] and batch.share_tdms is False
    batch.solve()                                     # (the refusal itself is the library's: tests/test_gpu_batch.py)
    assert "batch_share_tdms" not in fake.names()
    shared = cls(pls, share_tdms=True)
    assert fake.shared == [1] and shared.share_tdms is True
    n = fake.names().count("batch_solve")
    shared.solve()
    assert fake.names().count("batch_solve") == n + 1


@pytest.mark.parametrize("mode", ["det", "tdm"])
def test_partial_overlap_refused_before_any_work(host, mode):
    E, fake = host
    cls = E.MPPI_StochasticBatch if mode == "tdm" else E.MPPI_Batch
    pls = planners(E, mode, 3)
    batch = cls(pls, share_tdms=True)
    own = pls[2].lin_tdm, pls[2].ang_tdm
    cases = [((pls[0].lin_tdm, own[1]), "planners 0 and 2 share lin_tdm but not ang_tdm"),
             ((own[0], pls[1].ang_tdm), "planners 1 and 2 share ang_tdm but not lin_tdm"),
             ((pls[0].ang_tdm, own[1]), "planners 0 and 2: a TDM is lin_tdm of one and ang_tdm of the other")]
    for (lin, ang), msg in cases:
        pls[2].lin_tdm, pls[2].ang_tdm = lin, ang
        before = list(fake.names())
        with pytest.raises(ValueError, match=msg):
            batch.solve()
        assert fake.names() == before                 # nothing issued: not even the params uploads
        if mode == "det":
            with pytest.raises(ValueError, match=msg):
                batch.run_trials([None] * 3, 5)
        else:
            with pytest.raises(ValueError, match=msg):
                batch.run_stochastic_trials([None] * 3, 5)
        assert fake.names() == before
    pls[2].lin_tdm, pls[2].ang_tdm = own


def test_unequal_alpha_dyn_refused_before_any_work(host):
    E, fake = host
    pls = planners(E, "tdm", 3, pair=True)
    batch = E.MPPI_StochasticBatch(pls, share_tdms=True)
    pls[1].params["alpha_dyn"] = 0.8
    before = list(fake.names())
    with pytest.raises(ValueError, match=r"planners 0 and 1 share a TDM pair but have alpha_dyn 1.0 and 0.8"):
        batch.solve()
    with pytest.raises(ValueError, match=r"planners 0 and 1 share a TDM pair but have alpha_dyn"):
        batch.run_stochastic_trials([None] * 3, 5)
    assert fake.names() == before
    for p in pls:                                     # equal alpha_dyn: accepted
        p.params["alpha_dyn"] = 0.8
    batch.solve()
    assert fake.names().count("batch_solve") == before.count("batch_solve") + 1
    # one-map batches always sample at 1.0: their alpha_dyn is not compared
    dets = planners(E, "det", 2, pair=True)
    dets[1].params["alpha_dyn"] = 0.3
    E.MPPI_Batch(dets, share_tdms=True).solve()
