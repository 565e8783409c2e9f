"""CPU-only checks of the drop-in boundary: the C-ABI library loads and exports every symbol that
include/b200mppi.h declares, fails loudly without a GPU, and the host-side API mirrors behave like
the reference's Config / error conventions.  No compute calls (there is no GPU here)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def libmod():
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    return _lib


def test_every_declared_symbol_is_exported(libmod):
    hdr = open(os.path.join(ROOT, "include", "b200mppi.h")).read()
    declared = set(re.findall(r"\b(b200mppi_[a-z_0-9]+)\s*\(", hdr))
    assert len(declared) >= 35
    raw = C.CDLL(libmod.LIB_PATH)
    missing = [name for name in sorted(declared) if not hasattr(raw, name)]
    assert not missing, missing
    assert set(libmod.EXPORTS) == declared, set(libmod.EXPORTS) ^ declared


def test_library_has_sm90a_code(libmod):
    import subprocess
    from mppi_numba_b200 import build
    cuobjdump = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    out = subprocess.run([cuobjdump, "-lelf", libmod.LIB_PATH], capture_output=True, text=True)
    assert "sm_90a" in out.stdout


def test_pod_layouts_match_header(libmod, tmp_path):
    """sizeof/offsetof of the two PODs as gcc sees include/b200mppi.h == the ctypes mirrors."""
    import subprocess
    src = tmp_path / "layout.c"
    src.write_text("""
#include <stdio.h>
#include <stddef.h>
#include "b200mppi.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(b200mppi_config), offsetof(b200mppi_config, seed),
         offsetof(b200mppi_config, world_size), sizeof(b200mppi_params), offsetof(b200mppi_params, num_opt),
         offsetof(b200mppi_params, alpha_dyn), offsetof(b200mppi_params, wrange));
  return 0;
}
""")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    Cfg, Prm = libmod.ConfigPOD, libmod.ParamsPOD
    assert got == [C.sizeof(Cfg), Cfg.seed.offset, Cfg.world_size.offset, C.sizeof(Prm), Prm.num_opt.offset,
                   Prm.alpha_dyn.offset, Prm.wrange.offset]


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="GPU present")
def test_no_cpu_fallback(libmod):
    from mppi_numba_b200 import Config, MPPI_Numba, TDM_Numba, B200MPPIError
    assert libmod.device_count() == 0
    cfg = Config(T=1.0, dt=0.1, num_grid_samples=4, num_control_rollouts=100, use_tdm=True, max_map_dim=(20, 20))
    with pytest.raises(B200MPPIError, match="no CUDA device"):
        TDM_Numba(cfg)
    with pytest.raises(B200MPPIError, match="no CUDA device"):
        MPPI_Numba(cfg)


def test_product_never_imports_oracle():
    import ast
    pkg = os.path.join(ROOT, "mppi_numba_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            tree = ast.parse(open(os.path.join(pkg, fn)).read())
            for node in ast.walk(tree):
                names = []
                if isinstance(node, ast.Import):
                    names = [a.name for a in node.names]
                elif isinstance(node, ast.ImportFrom):
                    names = [node.module or ""]
                assert not any(n.split(".")[0] in ("oracle", "numba") for n in names), (fn, names)


def test_config_clamps_and_modes(capsys):
    from mppi_numba_b200 import Config
    c = Config(T=6.4, dt=0.1, use_det_dynamics=True, num_control_rollouts=64, num_grid_samples=0)
    assert c.num_steps == int(6.4 / 0.1) and c.num_control_rollouts == 100 and c.num_grid_samples == 1
    assert c.num_vis_state_rollouts == 1 and c.mode == 1 and c.det_dyn
    c = Config(use_tdm=True, num_control_rollouts=20000, num_grid_samples=20000, tdm_sample_thread_dim=(32, 32))
    assert c.num_control_rollouts == 15000 and c.num_grid_samples == 15000
    assert c.tdm_sample_thread_dim == (32, 32) and c.max_threads_per_block == 1024
    c = Config(use_tdm=True, tdm_sample_thread_dim=(64, 32))
    assert c.tdm_sample_thread_dim == (32, 32)
    assert Config(use_nom_dynamics_with_speed_map=True).mode == 2
    capsys.readouterr()
    for bad in (dict(), dict(use_tdm=True, use_det_dynamics=True), dict(use_costmap=True)):
        with pytest.raises(AssertionError):
            Config(**bad)
    with pytest.raises(AssertionError):
        Config(T=0.05, dt=0.1, use_tdm=True)


def test_combine_partials_host_matches_oracle_update(libmod):
    """The N>1 exchange math: per-rank (beta, S, V[2T]) partials merged by the library's host
    combine equal the oracle's single-process softmax update."""
    from oracle import mppi_ref as MR
    rng = np.random.default_rng(0)
    N, T, ws = 240, 7, 3
    costs = rng.uniform(50, 60, N).astype(np.float32)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(np.float32)
    u0 = rng.uniform(0, 1, (T, 2)).astype(np.float32)
    lam = np.float32(0.7)
    parts = []
    for r in range(ws):
        sl = slice(N * r // ws, N * (r + 1) // ws)
        beta = costs[sl].min()
        w = np.exp((-1.0 / float(lam)) * (costs[sl] - beta).astype(np.float64)).astype(np.float32)
        V = np.einsum("n,ntk->tk", w.astype(np.float64), noise[sl].astype(np.float64)).astype(np.float32)
        parts.append(np.concatenate([[beta, w.sum(dtype=np.float64)], V.ravel()]).astype(np.float32))
    g = np.ascontiguousarray(np.stack(parts))
    out = np.empty((T, 2), dtype=np.float32)
    vr = np.array([0, 3], np.float32)
    wr = np.array([-np.pi, np.pi], np.float32)
    libmod.check(libmod.lib.b200mppi_combine_partials_host(libmod.ptr(g), ws, T, lam, libmod.ptr(u0),
                                                          libmod.ptr(vr), libmod.ptr(wr), libmod.ptr(out)))
    want, _ = MR.update_useq(lam, costs, noise, vr, wr, u0)
    np.testing.assert_allclose(out, want, rtol=1e-5, atol=2e-6)


@pytest.mark.parametrize("alpha", [1.0, 0.9, 0.6, 0.3, 0.05, 1.27])
def test_sampler_threshold_tables_match_reference_arithmetic(libmod, alpha):
    """The sampler replaces q = int8(ceil(f64(f32((r >> 11) * 2^-53)) * 100 * alpha)) (terrain.py:682-684;
    numba's uint64_to_unit_float32, random.py:130-154) by a two-table lookup on the raw draw.  The very function
    the kernel inlines, evaluated on the host (b200mppi_debug_sample_threshold), against the oracle's float
    arithmetic: random draws, every bucket edge, and both sides of every breakpoint."""
    from oracle import terrain_ref as TR
    rng = np.random.default_rng(int(alpha * 1000))
    r = rng.integers(0, 2 ** 64, 400000, dtype=np.uint64)
    edges = (np.arange(256, dtype=np.uint64) << np.uint64(56))
    r = np.concatenate([r, edges, edges - np.uint64(1), edges + np.uint64(1), edges + np.uint64(2047), edges + np.uint64(2048),
                        np.array([0, 1, 2047, 2048, 2 ** 64 - 1, 2 ** 64 - 2048, 2 ** 64 - 2049], dtype=np.uint64)])

    def oracle_q(raw):
        u = ((raw >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)).astype(np.float32)
        return TR.sample_thresholds(u, alpha).astype(np.int64)

    def engine_q(raw):
        raw = np.ascontiguousarray(raw, dtype=np.uint64)
        out = np.empty(raw.shape, np.uint8)
        libmod.check(libmod.lib.b200mppi_debug_sample_threshold(alpha, 127, libmod.ptr(raw), raw.size, libmod.ptr(out)))
        return out.astype(np.int64)
    want = oracle_q(r)
    assert (engine_q(r) == want).all()
    # both sides of every breakpoint: bisect the oracle on the 53-bit draw v for each q level
    pts = []
    for k in range(1, int(want.max()) + 1):
        lo, hi = 0, 2 ** 53 - 1                       # q(lo) < k <= q(hi)
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if oracle_q(np.array([mid << 11], dtype=np.uint64))[0] >= k:
                hi = mid
            else:
                lo = mid
        pts += [(hi << 11) - 1, hi << 11, (hi << 11) + 2047, (lo << 11), (lo << 11) + 2047]
    pts = np.array(pts, dtype=np.uint64)
    assert (engine_q(pts) == oracle_q(pts)).all()


def test_sampler_threshold_tables_refuse_what_they_cannot_represent(libmod):
    r = np.zeros(4, np.uint64)
    out = np.empty(4, np.uint8)
    # q would exceed the smallest column total / alpha beyond the int8 range -> generic kernel
    assert libmod.lib.b200mppi_debug_sample_threshold(1.0, 50, libmod.ptr(r), 4, libmod.ptr(out)) != 0
    assert libmod.lib.b200mppi_debug_sample_threshold(1.5, 127, libmod.ptr(r), 4, libmod.ptr(out)) != 0
    assert "generic" in libmod.lib.b200mppi_last_error().decode()


def test_terrain_helper_mirrors_reference_constructor_and_statistics(libmod):
    """Terrain (terrain.py:24-66): positional order (name, rgb, lin_density, ang_density), saved samples, mean /
    var / std, CVaR = mean of the samples strictly below (front) or above the alpha-percentile, and
    update_cvar_alpha."""
    from mppi_numba_b200.terrain import Terrain

    class Dens:                                   # duck-typed: only sample()
        def __init__(self, seed, lo, hi):
            self.rng, self.lo, self.hi = np.random.default_rng(seed), lo, hi

        def sample(self, n):
            return self.rng.uniform(self.lo, self.hi, int(n))

    t = Terrain("grass", (0, 255, 0), Dens(1, 0.2, 0.9), Dens(2, 0.1, 0.5), cvar_alpha=0.2, cvar_front=True,
                num_saved_samples=2e3)
    assert t.name == "grass" and t.rgb == (0, 255, 0) and t.num_saved_samples == 2e3
    assert t.lin_saved_samples.shape == (2000,) and t.ang_saved_samples.shape == (2000,)
    for axis in ("lin", "ang"):
        smp = getattr(t, axis + "_saved_samples")
        assert getattr(t, axis + "_mean") == np.mean(smp) and getattr(t, axis + "_var") == np.var(smp)
        assert getattr(t, axis + "_std") == np.sqrt(np.var(smp))
        thres = np.percentile(smp, 20.0)
        assert getattr(t, axis + "_cvar_thres") == thres
        assert getattr(t, axis + "_cvar") == np.mean(smp[smp < thres])
    t.update_cvar_alpha(0.5)
    assert t.cvar_alpha == 0.5 and t.lin_cvar == np.mean(t.lin_saved_samples[t.lin_saved_samples < np.median(t.lin_saved_samples)])
    lin, ang = t.sample_traction(7)
    assert lin.shape == (7,) and ang.shape == (7,)
    assert "grass" in repr(t) and "2000" in repr(t).replace("2000.0", "2000")
    up = Terrain("rock", None, Dens(3, 0, 1), Dens(4, 0, 1), cvar_alpha=0.1, cvar_front=False)
    assert up.lin_cvar == np.mean(up.lin_saved_samples[up.lin_saved_samples > np.percentile(up.lin_saved_samples, 90.0)])

    class Full(Dens):                             # a density that brings its own statistics (density.py:25-56)
        def mean(self, samples=None):
            return 1.0

        def var(self, samples=None):
            return 4.0

        def cvar(self, alpha, front=True, samples=None):
            return 0.25, 0.5
    f = Terrain("x", None, Full(5, 0, 1), Full(6, 0, 1))
    assert (f.lin_mean, f.lin_var, f.lin_std, f.lin_cvar, f.lin_cvar_thres) == (1.0, 4.0, 2.0, 0.25, 0.5)


def test_sample_grids_true_dist_visits_classes_in_first_appearance_order(libmod):
    """TDM_Numba.sample_grids_true_dist (terrain.py:586-608) is host-only: semantic classes draw from their
    densities in the order they first appear in the grid (row-major), each cell of a class gets one draw."""
    import types
    from mppi_numba_b200.terrain import TDM_Numba, TractionGrid
    calls = []

    class Terr:
        def __init__(self, sid):
            self.sid = sid

        def sample_traction(self, n):
            calls.append((self.sid, n))
            return np.full(n, self.sid / 10.0) + np.arange(n) * 1e-3, np.full(n, self.sid / 20.0)
    sg = np.array([[5, 5, 2], [7, 2, 5], [7, 7, 7]])
    fake = types.SimpleNamespace(semantic_grid=sg, id2terrain_fn=lambda i: Terr(int(i)))
    g = TDM_Numba.sample_grids_true_dist(fake)
    assert isinstance(g, TractionGrid)
    assert calls == [(5, 3), (2, 2), (7, 4)]
    lin = g.lin_traction
    assert np.allclose(lin[sg == 5], 0.5 + np.arange(3) * 1e-3) and np.allclose(lin[sg == 7], 0.7 + np.arange(4) * 1e-3)
    assert np.allclose(g.ang_traction[sg == 2], 0.1)
    assert g.get(0.5, 0.5)[0] == lin[0, 0]
