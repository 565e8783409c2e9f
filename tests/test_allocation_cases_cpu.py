"""The tables of tests/allocation_cases.py kept honest, and the rollout kernels' real source run on them.

- Every geometry keeps its allocation larger than the padded map in the intended axes, with distinct pitches where the
  columns differ.
- From each corner, the exact oracle's trajectories read allocation cells beyond the map through the side the corner
  faces, on every geometry whose allocation extends that way; a wrap by the map's dimensions instead of the
  allocation's (the oracle given only the map-shaped part of the allocation) changes the costs.
- The generic kernels (modes 0, 1, 2), the windowed kernel and the visualisation kernel, executed on the host by
  tests/emu_rollout.py and tests/emu_rollout_win.py with both geometries and both pitches, equal the exact oracle
  (libm provider) bit for bit on the small geometries.  A mismatch seen only on the GPU then points at the device
  build rather than at the test.
- The window-first cases, sampled on the host from the TDM's initial generator states: one flags maps, one stays
  inside the sampled rectangle and reads nothing beyond the map, and the wrap and old-samples cases read beyond the map
  without a flag.  On the small map set over the large map's samples, the reads land on those samples and the costs
  depend on them."""
import numpy as np
import pytest

from tests import allocation_cases as AC
from tests import emu_rollout, emu_rollout_win
from tests.test_exact_oracle_cpu import EXACT, assert_equal
from tests.test_rollout_emulated_cpu import _c, _fparams, _p, _ratios

F32 = np.float32


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("emu_allocation"))
    return emu_rollout.build(d), emu_rollout_win.build(d)


@pytest.mark.parametrize("geom", list(AC.GEOMETRIES))
def test_geometry(geom):
    rows, cols, Rmax, Cmax, res = AC.GEOMETRIES[geom]
    assert Rmax >= rows and Cmax >= cols and (Rmax, Cmax) != (rows, cols)
    assert (Rmax > rows) == (geom in ("rows", "both", "large")) and (Cmax > cols) == (geom in ("cols", "both", "large"))
    assert cols % 16
    if Cmax > cols:
        assert len({AC.pitch(Cmax), AC.pitch(cols), cols}) == 3
    if geom == "large":
        assert rows > 232 and cols > 240
    else:
        assert rows < 224 and cols < 240
    s = AC.raw_case(geom, "centre", 0, N=4, M=2, T=2)
    for w in ("lin", "ang"):
        g = s[w]
        bc, br = AC.beyond(g.shape, rows, cols)
        assert (g[bc] == AC.SENTINELS[w][0]).all() and (g[br] == AC.SENTINELS[w][1]).all()
        assert ((g[~(bc | br)] >= 0) & (g[~(bc | br)] <= 100)).all()
    assert len({*AC.SENTINELS["lin"], *AC.SENTINELS["ang"]}) == 4 and min(AC.SENTINELS["lin"] + AC.SENTINELS["ang"]) > 100
    assert s["obs"].max() == (3 if geom == AC.MASKS03 else 1)


@pytest.mark.parametrize("geom", list(AC.GEOMETRIES))
def test_corners_read_beyond_the_map(geom):
    """Each corner's rollouts read beyond the map through the side it faces, wherever the allocation extends that
    way."""
    rows, cols, Rmax, Cmax, _ = AC.GEOMETRIES[geom]
    for spot in AC.SPOTS:
        s = AC.raw_case(geom, spot, 0, N=32, M=2)
        want, states = AC.oracle(s, EXACT, return_states=True)
        got = AC.beyond_reads(states, s, EXACT)
        if spot in AC.SIDE:
            axis, side = AC.SIDE[spot]
            key = ("wrap_" if side == "low" else "clamp_") + axis
            assert got[key] == ((Cmax > cols) if axis == "x" else (Rmax > rows)), (geom, spot, got)
        if any(got.values()):                       # wrapped / clamped by the map instead: other costs
            crop = (s["lin"][:, :rows, :cols], s["ang"][:, :rows, :cols])
            assert (AC.oracle(s, EXACT, grids=crop) != want).any(), (geom, spot)


def _emu_inputs(s):
    """The kernels' device layout: sampled maps at the allocation's pitch, masks at the map's."""
    rows, cols, Rmax, Cmax = s["R"], s["C"], s["Rmax"], s["Cmax"]
    gp, mp = AC.pitch(Cmax), AC.pitch(cols)
    grids = []
    for w in ("lin", "ang"):
        g = np.full((s["M"], Rmax, gp), -1, np.int8)         # the row tails beyond Cmax are never read
        g[:, :, :Cmax] = s[w]
        grids.append(g)
    planes = []
    for k in ("obs", "unk", "risk"):
        m = np.full((rows, mp), -1, np.int8)
        m[:, :cols] = s[k]
        planes.append(m)
    pxl, pyl = AC.limits(s)
    f = _fparams(s["res"], pxl[0], pyl[0], s["dt"], s["x0"], s["goal"], s["tol"], 0.01, 1.0, [2, 3], s["vrange"],
                 [-np.pi, np.pi], 1e5, 1e2, 1.0, s["lb"][0], s["ab"][0])
    geo = _c([rows, cols, Rmax, Cmax, gp, mp, s["T"], s["N"], s["M"]], np.int32)
    return f, geo, _ratios(s["lb"], s["ab"]), grids, planes


@pytest.mark.parametrize("geom", AC.SMALL)
def test_emulated_kernels_equal_oracle(emu, geom):
    gen, win = emu
    for spot in AC.SPOTS:
        for mode in (0, 1, 2):
            s = AC.raw_case(geom, spot, mode, N=64, M=4, T=60)
            f, geo, ratios, (lin, ang), (obs, unk, risk) = _emu_inputs(s)
            N, M = s["N"], s["M"]
            cnm, costs = np.zeros((N, M), F32), np.zeros(N, F32)
            gen.emu_rollout(mode, _p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), _p(risk),
                            _p(s["noise"]), _p(s["u_cur"]), _p(cnm), _p(costs), None, 0)
            what = "%s %s mode %d" % (geom, spot, mode)
            got = cnm if mode == 0 else costs[:, None]
            assert_equal(got, AC.oracle(s, EXACT, ctrl_order="sequential"), what + ", generic kernel")
            if mode == 0:
                out = np.zeros((N, M), F32)
                assert win.emu_rollout_win(_p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(obs), _p(unk), _p(s["noise"]),
                                           _p(s["u_cur"]), _p(out), 0, 0, None, None, 0, 1, 0, 0,
                                           int(not s["masks03"])) == 0
                assert_equal(out, AC.oracle(s, EXACT), what + ", windowed kernel")
            V = 4
            vis = np.zeros((V, s["T"] + 1, 3), F32)
            gen.emu_state_rollout(mode, V, _p(f), _p(geo), _p(ratios), _p(lin), _p(ang), _p(s["noise"]), _p(s["u_cur"]),
                                  _p(s["u_prev"]), _p(vis))
            assert_equal(vis, AC.state_oracle(s, V, EXACT), what + ", state rollouts")


@pytest.mark.parametrize("case", list(AC.WF_CASES))
def test_window_first_cases(case):
    base = None
    if case == "old-samples":                             # the small map's allocation holds the large map's samples
        base = AC.host_maps(AC.wf_scenario(*AC.WF_MAP), np.zeros((4,) + AC.WF_ALLOC, np.int8))[0]
    flags, hit, grids, costs = AC.wf_outcome(case, EXACT, base=base)
    flagged, beyond = AC.WF_CASES[case][-1]
    assert flags.any() == flagged, (case, flags)
    if beyond is not None:
        assert hit.any() == beyond, case
    if case == "old-samples":
        old = np.zeros(hit.shape, bool)
        old[:, :AC.WF_MAP[0] + 10, :AC.WF_MAP[1] + 10] = True              # the large padded map
        assert (hit & old & (base != 0)).any()
        _, _, _, zeroed = AC.wf_outcome(case, EXACT, base=np.zeros_like(base))
        assert (zeroed != costs).any()
