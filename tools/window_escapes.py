"""Window-first map sampling at bench.py's workload (config 5 by default): the bench's timed loop of solve() calls
with B200MPPI_SAMPLE_BOX=dynamic (reach box, host wait) and unset (window-first), alternated `--runs` times in one
process.  Prints one JSON line: per run the device-timed ms per solve, the per-stage CUDA-event times, launches per
solve, and for window-first the maps flagged per solve (rollouts that read outside the sampled rectangle).
--warm-v V starts every solve from the warm start u = (V, 0) heading +x (the robot's heading set to 0): at V = 3 the
rollouts leave the window, so the gated completion and redo launches have work (their cost is the difference of the
rollout stages, which include them).

    python tools/window_escapes.py [--workload c5] [--steps 50] [--runs 3] [--warm-v 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run_mode(E, torch, sc, mode, steps, warmup, warm_v=None):
    import ctypes as C
    import bench
    from mppi_numba_b200._lib import lib, check
    if mode is None:
        os.environ.pop("B200MPPI_SAMPLE_BOX", None)
    else:
        os.environ["B200MPPI_SAMPLE_BOX"] = mode
    if warm_v is not None:
        sc = dict(sc, params=dict(sc["params"], x0=np.array([sc["params"]["x0"][0], sc["params"]["x0"][1], 0.0])))
    cfg, lin, ang, pl = bench.make_planner(E, sc, 0)
    if warm_v is not None:
        pl.u_cur_d.copy_to_device(np.stack([np.full(sc["T"], warm_v), np.zeros(sc["T"])], 1).astype(np.float32))
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    check(lib.b200mppi_planner_set_stream(pl._handle, C.c_void_p(stream.cuda_stream)))
    st0 = pl.get_state()
    for _ in range(warmup):
        pl.solve()
    pl.set_state(st0)
    torch.cuda.synchronize(dev)
    l0 = pl.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        e0.record(stream)
        for _ in range(steps):
            pl.solve()
        e1.record(stream)
    torch.cuda.synchronize(dev)
    ms = e0.elapsed_time(e1) / steps
    launches = (pl.launch_count() - l0) / steps
    pl.set_state(st0)                                  # the same solves again, untimed: the escapes of each
    flagged = []
    for _ in range(steps):
        pl.solve()
        flagged.append(pl.sample_window()[5])
    pl.set_profiling(True)
    acc = {}
    for _ in range(10):
        pl.solve()
        for k, v in pl.last_timings().items():
            acc.setdefault(k, []).append(v)
    pl.set_profiling(False)
    out = dict(mode=mode or "window", ms_per_solve=ms, launches_per_solve=launches,
               stage_ms={k: float(np.mean(v)) for k, v in acc.items()}, sample_box=list(pl.sample_box()),
               sample_window=list(pl.sample_window()), flagged_per_solve=flagged)
    del pl, lin, ang
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c5")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warm-v", type=float, default=None)
    args = ap.parse_args()
    import torch
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    import bench
    sc = bench.build_scenario(args.workload)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    runs = []
    for _ in range(args.runs):
        for mode in ("dynamic", None):
            runs.append(run_mode(E, torch, sc, mode, args.steps, args.warmup, args.warm_v))
    med = {m: float(np.median([r["ms_per_solve"] for r in runs if r["mode"] == m])) for m in ("dynamic", "window")}
    print(json.dumps(dict(workload=args.workload, warm_v=args.warm_v, gpu=gpu, median_ms=med, speedup=med["dynamic"] / med["window"],
                          runs=runs)))


if __name__ == "__main__":
    main()
