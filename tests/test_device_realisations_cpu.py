"""Ground-truth realisations drawn on the device, without a GPU: the conversion kernel's real source through the
emulator against the NumPy expression of the reference notebook's sample_traction_grid (every int8 byte, several
float32 bound pairs, a whole plane of a map smaller than its allocation), the header's prototypes against the ctypes
mirrors, and the Python layer on a fake backend: device grids in the trial descriptors, host and device grids mixed in
one call, and every Python refusal issuing nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.emu_realisation import build
from tests.fake_backend import disarm
from tests.test_batch_host_cpu import det_planner
from tests.test_trials_host_cpu import TrialFake

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOUNDS = [(0.0, 1.0), (0.0, 60.0), (0.25, 1.75), (-3.5, 0.1), (1e-3, 7.3), (0.0, 1e-39), (-2.0, -1.0)]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build(str(tmp_path_factory.mktemp("emu_realisation")))


def helper_expression(q, lo, hi):
    """The notebook's q * (hi - lo) / 100.0 + lo for an int8 array and float32 bounds: float32 under NumPy 2."""
    lo, hi = np.float32(lo), np.float32(hi)
    out = q * (hi - lo) / 100.0 + lo
    assert out.dtype == np.float32
    return out.astype(np.float64)


def convert(emu, grids, pitch, bounds, rows, cols):
    n = len(grids)
    outs = [np.full((rows, cols), np.nan) for _ in range(n)]
    gp = (C.c_void_p * 2)(*[g.ctypes.data for g in grids] + [None] * (2 - n))
    op = (C.c_void_p * 2)(*[o.ctypes.data for o in outs] + [None] * (2 - n))
    emu.emu_realisation_convert(gp, (C.c_int * 2)(*(list(pitch) + [0] * (2 - n))),
                                (C.c_float * 2)(*[b[0] for b in bounds] + [0.0] * (2 - n)),
                                (C.c_float * 2)(*[b[1] for b in bounds] + [0.0] * (2 - n)), op, n, rows, cols)
    return outs


@pytest.mark.parametrize("lo, hi", BOUNDS)
def test_every_byte(emu, lo, hi):
    q = np.arange(-128, 128, dtype=np.int8).reshape(16, 16)
    got, = convert(emu, [q], [16], [(lo, hi)], 16, 16)
    want = helper_expression(q, lo, hi)
    assert got.tobytes() == want.tobytes()


def test_two_planes_of_a_map_smaller_than_its_allocation(emu):
    """Both planes in one launch, each with its own bounds and pitch, over the whole allocation: the bytes beyond the
    padded map (whatever the buffer holds there) are converted too, as copy_to_host()[0] returns them."""
    rng = np.random.default_rng(5)
    rows, cols = 37, 45
    lp, ap = 48, 64                                     # row pitches larger than the allocation's columns
    lg = rng.integers(-128, 128, (rows, lp)).astype(np.int8)
    ag = rng.integers(0, 101, (rows, ap)).astype(np.int8)
    lg[20:, :] = 7                                      # a sentinel beyond the map's rows
    got = convert(emu, [lg, ag], [lp, ap], [(0.0, 1.0), (0.25, 3.5)], rows, cols)
    assert got[0].tobytes() == helper_expression(lg[:, :cols], 0.0, 1.0).tobytes()
    assert got[1].tobytes() == helper_expression(ag[:, :cols], 0.25, 3.5).tobytes()


def test_rounding_is_not_contracted_or_flushed():
    """The cases above separate the exact rule from its neighbours: a fused multiply-add, a product by 0.01 instead of
    the division, and a flush of subnormals each give other values for some byte."""
    q = np.arange(-128, 128).astype(np.float32)
    hits = {"fma": False, "times_0.01": False, "ftz": False}
    for lo, hi in BOUNDS:
        lo, hi = np.float32(lo), np.float32(hi)
        exact = (q * (hi - lo) / np.float32(100) + lo).astype(np.float64)
        fma = ((q.astype(np.float64) * (hi - lo) / 100).astype(np.float32) + lo).astype(np.float64)
        prod = (q * (hi - lo) * np.float32(0.01) + lo).astype(np.float64)
        ftz = np.where(np.abs(exact) < np.finfo(np.float32).tiny, 0.0, exact)
        hits["times_0.01"] |= bool((prod != exact).any())
        hits["ftz"] |= bool((ftz != exact).any())
        hits["fma"] |= bool((fma != exact).any())
    assert all(hits.values()), hits


def test_abi_matches_ctypes(tmp_path):
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    src = tmp_path / "proto.c"
    src.write_text('#include "b200mppi.h"\n'
                   "int (*f0)(b200mppi_tdm*, b200mppi_tdm*, int32_t, b200mppi_realisations**) = "
                   "b200mppi_tdm_draw_realisations;\n"
                   "int (*f1)(b200mppi_realisations*) = b200mppi_realisations_destroy;\n"
                   "int (*f2)(const b200mppi_realisations*, int32_t*, int32_t*, int32_t*, double*, double*, double*, "
                   "int32_t*) = b200mppi_realisations_info;\n"
                   "int (*f3)(const b200mppi_realisations*, int32_t, const double**, const double**) = "
                   "b200mppi_realisations_planes;\n"
                   "int (*f4)(const b200mppi_realisations*, int32_t, double*, double*) = "
                   "b200mppi_realisations_copy_out;\n")
    r = subprocess.run(["gcc", "-c", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                        str(tmp_path / "proto.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for name, n in (("b200mppi_tdm_draw_realisations", 4), ("b200mppi_realisations_destroy", 1),
                    ("b200mppi_realisations_info", 8), ("b200mppi_realisations_planes", 4),
                    ("b200mppi_realisations_copy_out", 4)):
        assert name in _lib.EXPORTS
        fn = getattr(_lib.lib, name)
        assert fn.restype is C.c_int and len(fn.argtypes) == n, name


def test_library_refusals_without_a_device():
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    L = _lib.lib
    out = C.c_void_p()
    assert L.b200mppi_tdm_draw_realisations(None, None, 1, C.byref(out)) == -1
    assert "null argument" in L.b200mppi_last_error().decode()
    assert L.b200mppi_realisations_info(C.c_void_p(0x1234), None, None, None, None, None, None, None) == -1
    assert "not a live realisation set" in L.b200mppi_last_error().decode()
    assert L.b200mppi_realisations_destroy(C.c_void_p(0x1234)) == -1
    assert not out.value


# ----------------------------------------------------------------------------- Python layer on a fake backend
class RealisationFake(TrialFake):
    """TrialFake that also plays a realisation set of 2 realisations of 6 x 7 cells at fake device addresses."""
    BASE = 0x7f0000000000

    def b200mppi_tdm_draw_realisations(self, lin, ang, count, out):
        self.calls.append(("tdm_draw_realisations", (int(count),)))
        self.count = int(count)
        return self._handle_out(out)

    def b200mppi_realisations_info(self, h, count, height, width, res, xl, yl, device):
        for ref, v in ((count, self.count), (height, 6), (width, 7), (device, 0)):
            ref._obj.value = v
        return 0

    def b200mppi_realisations_planes(self, h, i, lin, ang):
        lin._obj.value = self.BASE + 2 * i * 6 * 7 * 8
        ang._obj.value = self.BASE + (2 * i + 1) * 6 * 7 * 8
        return 0

    def b200mppi_batch_run_trials(self, h, descs, max_steps, xh, uh, res, issued):
        K = len(self.members)
        self.descs = [(descs[i].lin, descs[i].ang, descs[i].height, descs[i].width, descs[i].xlo, descs[i].ylo,
                       descs[i].res) for i in range(K)]
        self.device_slots = [i for i in range(K) if descs[i].lin >= self.BASE]
        for i in self.device_slots:                      # TrialFake reads host grids: give it a host view instead
            descs[i].lin = descs[i].ang = self.stand_in.ctypes.data
        return super().b200mppi_batch_run_trials(h, descs, max_steps, xh, uh, res, issued)


@pytest.fixture()
def rhost(monkeypatch):
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    import mppi_numba_b200.barebone as B
    import mppi_numba_b200.batch as BT
    import mppi_numba_b200.mppi as M
    import mppi_numba_b200.terrain as T
    fake = RealisationFake()
    fake.stand_in = np.zeros((6, 7))
    for mod in (M, T, B, BT):
        monkeypatch.setattr(mod, "lib", fake)
    made = []
    yield E, fake, made
    for obj in made:
        obj._handle = None
    disarm(fake)


def test_device_grids_in_descriptors(rhost):
    E, fake, made = rhost
    planners = [det_planner(E, k) for k in range(3)]
    lin, ang = planners[0].lin_tdm, planners[0].ang_tdm
    dev = E.draw_traction_grids(lin, ang, 2)
    made.append(dev)
    batch = E.MPPI_Batch(planners)
    made.append(batch)
    assert len(dev) == 2 and (dev[1].height, dev[1].width) == (6, 7)
    assert dev[0].res == lin.res and np.array_equal(dev[0].xlimits, lin.padded_xlimits)
    host = E.TractionGrid(np.ones((5, 4)), np.ones((5, 4)), res=0.3, xlimits=(-1.0, 0.2), ylimits=(2.0, 3.5))
    out = batch.run_trials([dev[1], host, dev[0]], 4)
    assert fake.device_slots == [0, 2]
    base, plane = RealisationFake.BASE, 6 * 7 * 8
    assert fake.descs[0][:4] == (base + 2 * plane, base + 3 * plane, 6, 7)
    assert fake.descs[2][:4] == (base, base + plane, 6, 7)
    assert fake.descs[0][4:] == (float(lin.padded_xlimits[0]), float(lin.padded_ylimits[0]), float(lin.res))
    assert fake.descs[1][2:] == (5, 4, -1.0, 2.0, 0.3)
    assert out["xhist"].shape == (3, 5, 3)


def test_python_refusals_issue_nothing(rhost):
    E, fake, made = rhost
    p = det_planner(E, 0)
    q = det_planner(E, 1)
    n = len(fake.calls)
    with pytest.raises(ValueError, match="count 0 < 1"):
        E.draw_traction_grids(p.lin_tdm, p.ang_tdm, 0)
    q.ang_tdm.device = 1
    with pytest.raises(ValueError, match="lin_tdm is on device 0, ang_tdm on device 1"):
        E.draw_traction_grids(p.lin_tdm, q.ang_tdm, 1)
    q.ang_tdm.device = 0
    p.lin_tdm.pmf_grid_initialized = False
    with pytest.raises(ValueError, match="lin_tdm has no PMF grid set"):
        E.draw_traction_grids(p.lin_tdm, p.ang_tdm, 1)
    assert len(fake.calls) == n
