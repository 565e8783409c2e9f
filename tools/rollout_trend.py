import io, contextlib, numpy as np, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mppi_numba_b200 as E
from bench import build_scenario
sc = build_scenario("c5")
with contextlib.redirect_stdout(io.StringIO()):
    cfg = E.Config(**sc["cfg"]); lin, ang = E.TDM_Numba(cfg), E.TDM_Numba(cfg)
    lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    pl = E.MPPI_Numba(cfg); pl.setup(sc["params"], lin, ang)
pl.set_profiling(True)
rows = []
for k in range(60):
    u = pl.solve()
    t = pl.last_timings()
    if k % 5 == 0 or k < 4:
        print(k, "rollout %.3f ms  sample %.3f  | mean v %.2f  mean |w| %.2f" % (t["rollout"], t["sample_grids"], float(u[:, 0].mean()), float(np.abs(u[:, 1]).mean())))
