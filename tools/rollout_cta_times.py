"""Per-CTA wall times of the persistent rollout kernel (CAUTION: the hook itself slows the kernel by ~16 %, and its
slow-path counters are global atomics per slow lane-step -- they stretch exactly the CTAs whose rollouts take the rare
paths; use it for which-CTA-does-what questions, not for how much the production kernel's CTAs differ) for one rank of a G-rank solve (run alone on one GPU).
Needs a library built with the hook:  B200MPPI_NVCC_FLAGS=-DB200MPPI_WIN_DEBUG_HOOK python mppi_numba_b200/build.py --force
(the default build leaves it out: the dead branches cost the hot loop 16 %).
    python tools/rollout_cta_times.py c5 8"""
import contextlib, ctypes as C, io, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import mppi_numba_b200 as E
from mppi_numba_b200._lib import lib, check
from bench import build_scenario
name, G = sys.argv[1], int(sys.argv[2])
sc = build_scenario(name)
with contextlib.redirect_stdout(io.StringIO()):
    cfg = E.Config(**sc["cfg"])
    lin, ang = E.TDM_Numba(cfg, rank=0, world_size=G), E.TDM_Numba(cfg, rank=0, world_size=G)
    lin.set_TDM_from_PMF_grid(sc["pmf_lin"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    ang.set_TDM_from_PMF_grid(sc["pmf_ang"], sc["tdm_dict"], sc["obstacle"], sc["unknown"])
    pl = E.MPPI_Numba(cfg, rank=0, world_size=G)
    pl.setup(sc["params"], lin, ang)
pl.move_mppi_task_vars_to_device()
def solve():
    if G == 1: pl.solve()
    else:
        check(lib.b200mppi_planner_solve_local(pl._handle, 1)); check(lib.b200mppi_planner_synchronize(pl._handle))
for _ in range(6): solve()
import torch
SMS = torch.cuda.get_device_properties(0).multi_processor_count
raw = np.zeros((256 + 99, 6), np.int64)        # SMS x 6 per-CTA slots, then (from word 1536) SMS x 4 extra counters
check(lib.b200mppi_debug_rollout_cta_times(1, None, 0))
solve()
check(lib.b200mppi_debug_rollout_cta_times(0, raw.ctypes.data_as(C.c_void_p), 256 + 99))
out = raw[:SMS].copy()
extra = raw.reshape(-1)[1536:1536 + SMS * 4].reshape(SMS, 4)
if not out[:, 1].any():
    sys.exit("no data: build the library with -DB200MPPI_WIN_DEBUG_HOOK (see the docstring)")
ran = out[:, 1] > 0
extra = extra[ran]
out = out[ran]                                # the CTAs that ran (B200MPPI_WIN_GRID < SMS)
smid = out[:, 2] >> 40
out[:, 2] &= (1 << 40) - 1
wsteps = out[:, 5] >> 40
out[:, 5] &= (1 << 40) - 1
t0 = out[:, 0].min()
dur = (out[:, 1] - out[:, 0]) / 1e3
start = (out[:, 0] - t0) / 1e3
end = (out[:, 1] - t0) / 1e3
M = sc["M"] // G
cpm = (sc["N"] + 31) // 32
print("kernel span %.1f us; CTA duration min/median/max %.1f / %.1f / %.1f us; latest start %.1f us" % (end.max(), dur.min(), np.median(dur), dur.max(), start.max()))
order = np.argsort(-dur)
for b in list(order[:12]) + list(order[-4:]):
    lo, hi = out[b, 2], out[b, 3]
    segs = []
    w = lo
    while w < hi:
        m = w // cpm
        e = min(hi, (m + 1) * cpm)
        segs.append(int(e - w)); w = e
    steps = (hi - lo) * 32 * sc["T"]
    print("cta %3d dur %6.1f us chunks %3d segments %s slow %.3f of lane-steps, outside window %.3f" % (
        b, dur[b], hi - lo, segs, out[b, 4] / steps, out[b, 5] / steps), flush=True)
tot = ((out[:, 3] - out[:, 2]) * 32 * sc["T"]).sum()
print("all CTAs: slow path %.4f of lane-steps, outside the window %.4f; corr(duration, outside) = %.2f" % (
    out[:, 4].sum() / tot, out[:, 5].sum() / tot, np.corrcoef(dur, out[:, 5] / ((out[:, 3] - out[:, 2]) * 32 * sc["T"]))[0, 1]))

print("warp-steps per CTA min/median/max %d / %d / %d; corr(duration, warp-steps) = %.3f; ns per warp-step min/median/max %.1f / %.1f / %.1f" % (
    wsteps.min(), np.median(wsteps), wsteps.max(), np.corrcoef(dur, wsteps)[0, 1], (dur * 1e3 / wsteps).min(), np.median(dur * 1e3 / wsteps), (dur * 1e3 / wsteps).max()))
print("by block (duration us / warp-steps):")
print(" ".join("%d:%.0f/%d" % (b, dur[b], wsteps[b]) for b in range(len(dur))))
print("by SM id (duration us):")
o = np.argsort(smid)
line = []
for b in o:
    line.append("%d:%.0f" % (smid[b], dur[b]))
print(" ".join(line))
pair = {}
for b in range(len(dur)):
    pair.setdefault(int(smid[b]) // 2, []).append(dur[b])
both = [v for v in pair.values() if len(v) == 2]
print("SM pairs (smid // 2) with both SMs busy: %d; mean |difference| within a pair %.1f us; mean of pair minima %.1f, maxima %.1f" % (
    len(both), np.mean([abs(v[0] - v[1]) for v in both]), np.mean([min(v) for v in both]), np.mean([max(v) for v in both])))
