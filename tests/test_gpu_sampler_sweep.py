"""The map sampler (csrc/sample.cu) against the oracle's restatement of sample_grids_numba, on the GPU, across every
variant of its launch plan (tests/sampler_sweep_cases.py): the staged kernel at NW = 1, 0, 3 and 8, alone and fused
for a lin/ang pair, the generic kernel on well-formed and ill-formed PMFs, forced row segments, ragged and empty tile
columns, partial map groups, wide thread tiles, tight and refused threshold tables, and boxed solves.  Plus the PMF
preprocessing of the one-map modes (collapse_pad_kernel) against the oracle's collapse.  Every comparison is an
equality: maps byte for byte (the pitch padding included), generator states word for word."""
import ctypes as C
import re
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import terrain_ref as TR                     # noqa: E402
from oracle import xoroshiro as X                        # noqa: E402
from tests import sampler_sweep_cases as S               # noqa: E402
from tests.gpu_harness import eng, planner_launches, quiet   # noqa: E402,F401
from tests.scenarios import make_scenario, random_pmf   # noqa: E402


class _Raw:
    """A device pointer as a flat int8 __cuda_array_interface__ (torch views it without a copy)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = dict(shape=(n,), typestr="|i1", data=(int(ptr), False), version=3,
                                             strides=None)


def pitched_view(E, handle, maps, rows):
    """The TDM's whole sample-grid allocation, (maps, max rows, pitch) int8, as a torch view of device memory.  Reading
    it does not complete a boxed sampling (only the C entry points do)."""
    import torch
    L = E._lib
    base, pitch = C.c_void_p(), C.c_int32()
    L.check(L.lib.b200mppi_tdm_sample_grid_view(handle, C.byref(base), C.byref(pitch)))
    n = maps * rows * pitch.value
    return torch.as_tensor(_Raw(base.value, n), device="cuda").view(maps, rows, pitch.value)


def fill(view, value):
    import torch
    view.fill_(value)
    torch.cuda.synchronize()                       # the library's streams do not wait for torch's


class RawTDM:
    """One TDM through the C-ABI: set_pmf / set_pmf_collapsed, sample_grids, the raw grid and the generator states."""

    def __init__(self, E, mode, M, maxdim, tile, seed):
        L = E._lib
        self.E, self.L = E, L
        self.M = M if mode == 0 else 1
        self.tile, self.maxdim = tile, maxdim
        pod = L.ConfigPOD(num_steps=8, num_control_rollouts=32, num_grid_samples=M, max_map_rows=maxdim[0],
                          max_map_cols=maxdim[1], tdm_thread_x=tile[0], tdm_thread_y=tile[1], num_vis_state_rollouts=1,
                          mode=mode, device=0, rank=0, world_size=1, seed=seed)
        self.h = C.c_void_p()
        L.check(L.lib.b200mppi_tdm_create(C.byref(pod), C.byref(self.h)))
        ng = C.c_int64()
        L.check(L.lib.b200mppi_tdm_num_generators(self.h, C.byref(ng)))
        self.ngen = ng.value

    def close(self):
        self.L.lib.b200mppi_tdm_destroy(self.h)

    def set_pmf(self, pmf, bv, bounds=S.BOUNDS, res=0.5):
        L = self.L
        pmf = np.ascontiguousarray(pmf, np.int8)
        bv, bb = np.ascontiguousarray(bv, np.float32), np.ascontiguousarray(bounds, np.float32)
        lim = np.array([0.0, 1.0], np.float32)
        L.check(L.lib.b200mppi_tdm_set_pmf(self.h, L.ptr(pmf), pmf.shape[0], pmf.shape[1], pmf.shape[2], L.ptr(bv),
                                           L.ptr(bb), np.float32(res), L.ptr(lim), L.ptr(lim)))

    def sample(self, alpha):
        self.L.check(self.L.lib.b200mppi_tdm_sample_grids(self.h, float(alpha)))

    def view(self):
        return pitched_view(self.E, self.h, self.M, self.maxdim[0])

    def states(self):
        out = np.empty((self.ngen, 2), np.uint64)
        self.L.check(self.L.lib.b200mppi_tdm_get_rng_states(self.h, self.L.ptr(out), out.nbytes))
        return out


def same(got, want, what):
    """Equal dtype, shape and bytes; a mismatch reports its count and the first indices."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, "%s: %d of %d differ; first %s" % (
        what, len(bad), got.size, [(tuple(int(i) for i in ix), got[tuple(ix)], want[tuple(ix)]) for ix in bad[:5]])


def set_segs(monkeypatch, segs):
    if segs is None:
        monkeypatch.delenv("B200MPPI_SAMPLE_SEGS", raising=False)
    else:
        monkeypatch.setenv("B200MPPI_SAMPLE_SEGS", str(segs))


# ----------------------------------------------------------------------------- 1. whole maps, one TDM
@pytest.mark.parametrize("row", S.CASES, ids=[r[0] for r in S.CASES])
def test_whole_map_sampling_vs_oracle(eng, monkeypatch, row):
    """Every call of the case: the whole pitched allocation (sentinel outside the map rectangle of every map, and in
    cells no bin reaches) and every generator state equal the oracle run on the same sequence of alphas."""
    c = S.case_dict(row)
    set_segs(monkeypatch, S.forced_segs(c))
    pmf, bv = S.case_pmf(c), S.bin_values(c["B"])
    t = RawTDM(eng, 0, c["M"], c["maxdim"], c["tile"], c["seed"])
    try:
        t.set_pmf(pmf, bv)
        full = t.view()
        fill(full, S.SENTINEL)
        want = np.full(tuple(full.shape), S.SENTINEL, np.int8)
        st = X.create_states(t.ngen, c["seed"])
        oracle_s = 0.0
        for k, a in enumerate(c["alphas"]):
            t.sample(a)
            t0 = time.perf_counter()
            TR.sample_grids(want, pmf, st, bv, S.BOUNDS, a, c["tile"], c["M"])
            oracle_s += time.perf_counter() - t0
            what = "%s call %d (alpha %g)" % (c["name"], k, a)
            same(full.cpu().numpy(), want, what + ": maps")
            same(t.states(), st, what + ": states")
        print("\n[%s] oracle %.3f s" % (c["name"], oracle_s))
    finally:
        t.close()


_KERNEL = re.compile(r"sample_grids_v2_kernel(?:<(\d), ?(\d)>|ILi(\d)ELi(\d)E)")


def launched_samplers(fn):
    """The sampler kernels fn() launches, as ("staged", NT, NW) or ("generic",), from the CUDA activity trace."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    out = []
    for e in prof.events():
        m = _KERNEL.search(e.name)
        if m:
            g = [v for v in m.groups() if v is not None]
            out.append(("staged", int(g[0]), int(g[1])))
        elif "sample_grids_kernel" in e.name:
            out.append(("generic",))
    return out


def test_whole_map_plan_is_the_predicted_kernel(eng, monkeypatch):
    """The restated plan (tests/sampler_sweep_cases.plan) names the kernel the library launches for every call of
    every case, so the CPU coverage test's variant list is what the GPU runs."""
    for row in S.CASES:
        c = S.case_dict(row)
        set_segs(monkeypatch, S.forced_segs(c))
        pmf = S.case_pmf(c)
        t = RawTDM(eng, 0, c["M"], c["maxdim"], c["tile"], c["seed"])
        try:
            t.set_pmf(pmf, S.bin_values(c["B"]))
            for a, p in zip(c["alphas"], S.case_plans(c, eng._lib)):
                want = [("staged", 1, p["NW"])] if p["kernel"] == "staged" else [("generic",)]
                assert launched_samplers(lambda: t.sample(a)) == want, (c["name"], a, p)
        finally:
            t.close()


# ----------------------------------------------------------------------------- 2. lin/ang pairs through solve()
def pair_planner(E, p, seed):
    """A planner over lin / ang TDMs with p's bin counts and shape, the reach box off (whole maps)."""
    sc = make_scenario("tdm", N=128, M=p["M"], T=8, H=p["H"], W=p["H"], res=p["res"], B=p["B0"], seed=seed,
                       thread_dim=p["tile"])
    sc["params"]["alpha_dyn"] = p["alpha"]
    rng = np.random.default_rng(seed + 7)
    pmfs = (random_pmf(rng, p["B0"], p["H"], p["H"]), random_pmf(rng, p["B1"], p["H"], p["H"]))
    cfg = E.Config(**sc["cfg"])
    tdms = []
    for B, pmf in zip((p["B0"], p["B1"]), pmfs):
        d = dict(sc["tdm_dict"], bin_values=np.linspace(0.0, 1.0, B) ** 1.5)
        t = E.TDM_Numba(cfg)
        t.set_TDM_from_PMF_grid(pmf, d, sc["obstacle"], sc["unknown"])
        tdms.append(t)
    if p["diverged"]:
        tdms[0].sample_grids()
    pl = E.MPPI_Numba(cfg)
    pl.setup(sc["params"], tdms[0], tdms[1])
    return pl, sc, cfg


@pytest.mark.parametrize("row", S.PAIRS, ids=[r[0] for r in S.PAIRS])
def test_pair_sampling_in_solve_vs_oracle(eng, monkeypatch, row):
    """Two solves of a planner with the reach box off: both TDMs' maps and generator states equal the oracle for each
    TDM's own history; the solve issues one sampler launch when the plan fuses the pair and two otherwise."""
    p = S.pair_dict(row)
    monkeypatch.setenv("B200MPPI_SAMPLE_BOX", "off")
    set_segs(monkeypatch, -(-p["shape"][0] // p["tile"][0]) if p["segs"] == "nrow" else p["segs"])
    pred = S.pair_plan(p)
    seed = 40 + sum(map(ord, p["name"]))
    with quiet():
        pl, sc, cfg = pair_planner(eng, p, seed)
    tdms = (pl.lin_tdm, pl.ang_tdm)
    tx, ty = p["tile"]
    wants, sts = [], []
    for k, t in enumerate(tdms):
        wants.append(np.zeros(t.sample_grid_batch_d.shape, np.int8))
        sts.append(X.create_states(tx * ty * p["M"], cfg.seed))
        if p["diverged"] and k == 0:
            TR.sample_grids(wants[0], t.pmf_grid_d.copy_to_host(), sts[0], t.bin_values, t.bin_values_bounds, 1.0,
                            p["tile"], p["M"])
    x0 = np.asarray(sc["params"]["x0"], np.float64)
    oracle_s = 0.0
    for call in range(2):
        n0 = planner_launches(pl)
        with quiet():
            u = pl.solve()
        assert planner_launches(pl) - n0 == 4 + (1 if pred["nt"] == 2 else 2), (p["name"], pred)
        for k, t in enumerate(tdms):
            t0 = time.perf_counter()
            TR.sample_grids(wants[k], t.pmf_grid_d.copy_to_host(), sts[k], t.bin_values, t.bin_values_bounds,
                            p["alpha"], p["tile"], p["M"])
            oracle_s += time.perf_counter() - t0
            what = "%s solve %d TDM %d" % (p["name"], call, k)
            same(t.sample_grid_batch_d.copy_to_host(), wants[k], what + ": maps")
            same(t.rng_states_d.copy_to_host(), sts[k], what + ": states")
        x0 = x0 + np.array([0.05, -0.03, 0.02])
        pl.shift_and_update(x0.copy(), u, 1)
    print("\n[%s] oracle %.3f s" % (p["name"], oracle_s))


# ----------------------------------------------------------------------------- 3. boxed solves
@pytest.mark.parametrize("row", S.BOXES, ids=[r[0] for r in S.BOXES])
def test_boxed_solve_vs_oracle(eng, monkeypatch, row):
    """A solve with the static reach box: its recorded box is the restated one; inside it (inside the disc, when on)
    the maps hold the oracle's whole-map values and nothing outside the box's rows and tile columns is written; the
    generator states are the oracle's after a whole walk; reading the maps completes them to the oracle's whole maps."""
    b = S.box_dict(row)
    pred, box, disc = S.box_plan(b)
    assert box is not None and pred["kernel"] == "staged" and pred["nt"] == 2, (b["name"], box, pred)
    monkeypatch.setenv("B200MPPI_SAMPLE_BOX", "static")
    monkeypatch.setenv("B200MPPI_SAMPLE_DISC", "1" if b["disc"] else "0")
    set_segs(monkeypatch, None)
    seed = 60 + sum(map(ord, b["name"]))
    sc = make_scenario("tdm", N=128, M=b["M"], T=b["T"], H=b["H"], W=b["H"], res=b["res"], B=b["B"], seed=seed,
                       thread_dim=b["tile"])
    sc["params"]["x0"] = S.box_x0(b)
    with quiet():
        cfg = eng.Config(**sc["cfg"])
        lin, ang = eng.TDM_Numba(cfg), eng.TDM_Numba(cfg)
        lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
        pl = eng.MPPI_Numba(cfg)
        pl.setup(sc["params"], lin, ang)
    views = [pitched_view(eng, t._handle, b["M"], cfg.max_map_dim[0]) for t in (lin, ang)]
    for v in views:
        fill(v, S.SENTINEL)
    with quiet():
        pl.solve()
    rec = pl.sample_box()
    rows, cols = b["shape"]
    r_lo, r_hi, c_lo, c_hi = rec[1:]
    ncol = pred["ncol"]
    tc_lo, tc_hi = (c_lo // ncol) * ncol, min(((c_hi - 1) // ncol + 1) * ncol, cols)
    region = np.zeros(tuple(views[0].shape[1:]), bool)
    region[r_lo:r_hi, tc_lo:tc_hi] = True
    need = region.copy()                                     # without the disc: every cell of the launch
    if b["disc"]:
        need[:] = False
        need[r_lo:r_hi, c_lo:c_hi] = True
        cx, cy, r = (float(v) for v in disc)
        yy, xx = np.mgrid[0:region.shape[0], 0:region.shape[1]]
        dy = np.maximum(np.maximum(yy - cy, cy - (yy + 1)), 0)
        dx = np.maximum(np.maximum(xx - cx, cx - (xx + 1)), 0)
        need &= dx ** 2 + dy ** 2 <= r ** 2
    tx, ty = b["tile"]
    for k, (t, v) in enumerate(zip((lin, ang), views)):
        got = v.cpu().numpy()                                  # the boxed launch's bytes, not completed
        states = t.rng_states_d.copy_to_host()                 # the advance_states_kernel jump
        want = np.full(got.shape, S.SENTINEL, np.int8)
        st = X.create_states(tx * ty * b["M"], cfg.seed)
        t0 = time.perf_counter()
        TR.sample_grids(want, t.pmf_grid_d.copy_to_host(), st, t.bin_values, t.bin_values_bounds, 1.0, b["tile"], b["M"])
        oracle_s = time.perf_counter() - t0
        what = "%s TDM %d" % (b["name"], k)
        same(got[:, ~region], np.full_like(want[:, ~region], S.SENTINEL), what + ": outside the box")
        same(got[:, need], want[:, need], what + ": inside the box")
        assert ((got == want) | (got == S.SENTINEL))[:, region].all(), what
        if b["disc"]:
            assert (got[:, region] == S.SENTINEL).any(), what + ": the disc parks no tile"
        same(states, st, what + ": states after the whole-tile jump")
        same(t.sample_grid_batch_d.copy_to_host(), want[:, :, :cfg.max_map_dim[1]], what + ": completed maps")
        same(v.cpu().numpy(), want, what + ": completed allocation")
        same(t.rng_states_d.copy_to_host(), st, what + ": states after completion")
        print("\n[%s] oracle %.3f s" % (what, oracle_s))
    assert rec[0] == 1 and tuple(rec[1:]) == box, (b["name"], rec, box)
    assert pred["cs0_unaligned"] == ((tc_lo & ~15) != tc_lo), (b["name"], pred)


# ----------------------------------------------------------------------------- 4. PMF preprocessing on the device
def collapse_pmf(seed, B, H, W, alpha):
    """Random columns summing to 100, plus: one-hot columns (the statistic equals a bin value exactly), columns whose
    running mass reaches 100 * alpha exactly or one either side (the float64 tie of 0.01 * isum against alpha), and
    columns that do not sum to 100."""
    rng = np.random.default_rng(seed)
    flat = S.sweep_pmf(seed, B, H, W).astype(np.int64).reshape(B, -1)
    n = flat.shape[1]
    for i in range(1, n, 11):
        flat[:, i] = 0
        flat[rng.integers(B), i] = 100
    if B >= 2:
        k = int(round(100 * alpha))
        for j, i in enumerate(range(3, n, 13)):
            m = min(max(k + j % 3 - 1, 0), 100)
            b = int(rng.integers(0, B - 1))
            flat[:, i] = 0
            flat[b, i] = m
            flat[int(rng.integers(b + 1, B)), i] += 100 - m
    for i in range(4, n, 17):
        flat[rng.integers(B), i] += int(rng.integers(-30, 28))
    return np.clip(flat, -128, 127).astype(np.int8).reshape(B, H, W)


COLLAPSE_SHAPES = [            # B, raw (H, W), kept (rows, cols), padding ring
    (1, (9, 11), (7, 10), 2),
    (5, (20, 17), (20, 13), 3),
    (127, (6, 8), (5, 8), 1),
]


@pytest.mark.parametrize("alpha", [1.0, 0.3, 0.7, 0.01])
@pytest.mark.parametrize("shape", COLLAPSE_SHAPES, ids=["B%d" % s[0] for s in COLLAPSE_SHAPES])
@pytest.mark.parametrize("mode", [1, 2], ids=["det", "spd"])
def test_collapsed_pmf_vs_oracle(eng, mode, shape, alpha):
    """b200mppi_tdm_set_pmf_collapsed (collapse_pad_kernel): the padded one-hot PMF, the risk map (speed-map mode; bin
    values outside the bounds, so the risk truncates below zero and wraps above 127) and the count of columns not
    summing to 100 equal the oracle's collapse; the map sampled from it equals the oracle's."""
    B, (H, W), (kr, kc), pad = shape
    L = eng._lib
    raw = collapse_pmf(500 + B + int(100 * alpha), B, H, W, alpha)
    bv = np.linspace(-0.3, 1.6, B).astype(np.float32) if B > 1 else np.array([1.45], np.float32)
    bounds = np.array([0.1, 0.9], np.float32)
    Hp, Wp = kr + 2 * pad, kc + 2 * pad
    t = RawTDM(eng, mode, 1, (Hp + 1, Wp + 3), (3, 2), 17)
    try:
        out = np.empty((B, Hp, Wp), np.int8)
        risk = np.empty((Hp, Wp), np.int8)
        bad = C.c_int32(-1)
        lim = np.array([0.0, 1.0], np.float32)
        L.check(L.lib.b200mppi_tdm_set_pmf_collapsed(t.h, L.ptr(raw), B, H, W, kr, kc, pad, L.ptr(bv), L.ptr(bounds),
                                                     np.float32(0.5), L.ptr(lim), L.ptr(lim), float(alpha), L.ptr(out),
                                                     L.ptr(risk) if mode == 2 else None, C.byref(bad)))
        inner = raw[:, :kr, :kc]
        want = np.zeros((B, Hp, Wp), np.int8)
        want[0] = 100
        if mode == 1:
            want[:, pad:pad + kr, pad:pad + kc] = TR.collapse_pmf_det_dynamics(inner, bv, alpha)
        else:
            onehot, r = TR.risk_traction_map(inner, bv, bounds, alpha)
            want[:, pad:pad + kr, pad:pad + kc] = onehot
            want_risk = np.zeros((Hp, Wp), np.int8)
            want_risk[pad:pad + kr, pad:pad + kc] = r[0]
            same(risk, want_risk, "risk map")
        same(out, want, "padded PMF")
        assert bad.value == int((inner.astype(np.int64).sum(0) != 100).sum()) > 0
        full = t.view()
        fill(full, S.SENTINEL)
        grid = np.full(tuple(full.shape), S.SENTINEL, np.int8)
        st = X.create_states(t.ngen, 17)
        t.sample(1.0)
        TR.sample_grids(grid, want, st, bv, bounds, 1.0, (3, 2), 1)
        same(full.cpu().numpy(), grid, "sampled map")
        same(t.states(), st, "states")
    finally:
        t.close()
