#!/usr/bin/env python
"""Summarise an `ncu --set full` report (CPU-side: `ncu -i <rep> --page raw --csv`) into

  * profiles/kernel_metrics.json -- the per-launch figures bench.py's `roofline` object quotes (DRAM bytes, warp
    instructions, the saturated resource) for the dominant kernels of one workload, and
  * a markdown table of the metrics that decide what bounds a kernel (pipes, issue, stalls, occupancy, memory).

    python tools/ncu_summary.py runs/prof_<tag>.ncu-rep --workload c5 --capture <tag> [--json profiles/kernel_metrics.json] [--md runs/<tag>_ncu_summary.md]

The averages are over the captured launches of each kernel name (warm launches: the capture skips the first solves).
"""
import argparse
import csv
import io
import json
import os
import re
import subprocess
import sys

KEYS = [
    ("duration_ms", "gpu__time_duration.sum", 1.0),
    ("dram_read_MB", "dram__bytes_read.sum", 1.0),
    ("dram_write_MB", "dram__bytes_write.sum", 1.0),
    ("dram_pct_of_peak", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", 1.0),
    ("warp_inst", "smsp__inst_executed.sum", 1.0),
    ("issue_active_pct", "smsp__issue_active.avg.pct_of_peak_sustained_active", 1.0),
    ("inst_per_cycle_active", "sm__inst_executed.avg.per_cycle_active", 1.0),
    ("pipe_alu_pct", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", 1.0),
    ("pipe_fma_pct", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", 1.0),
    ("pipe_fmaheavy_pct", "sm__inst_executed_pipe_fmaheavy.avg.pct_of_peak_sustained_active", 1.0),
    ("pipe_xu_pct", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", 1.0),
    ("pipe_fp64_pct", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active", 1.0),
    ("pipe_lsu_pct", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", 1.0),
    ("pipe_uniform_pct", "sm__inst_executed_pipe_uniform.avg.pct_of_peak_sustained_active", 1.0),
    ("lsu_wavefronts_pct", "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", 1.0),
    ("smem_ld_wavefronts", "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_ld.sum", 1.0),
    ("smem_ld_bank_conflicts", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_ld.sum", 1.0),
    ("warps_active_pct", "sm__warps_active.avg.pct_of_peak_sustained_active", 1.0),
    ("registers", "launch__registers_per_thread", 1.0),
    ("smem_per_block_KB", "launch__shared_mem_per_block_dynamic", 1.0),
    ("grid", "launch__grid_size", 1.0),
    ("block", "launch__block_size", 1.0),
    ("sm_clock_mhz", "sm__cycles_elapsed.avg.per_second", 1.0),
]
STALLS = "smsp__average_warps_issue_stalled_"      # + reason + "_per_issue_active.ratio"


def load(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True)
    if out.returncode != 0:
        sys.exit("ncu failed: " + out.stderr[-500:])
    rows = list(csv.reader(io.StringIO(out.stdout)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    return hdr, units, data


def num(x):
    try:
        return float(x.replace(",", ""))
    except ValueError:
        return None


def scale(value, unit):
    u = unit.strip().lower()
    f = {"kbyte": 1e-3, "mbyte": 1.0, "gbyte": 1e3, "byte": 1e-6, "usecond": 1e-3, "msecond": 1.0, "second": 1e3,
         "nsecond": 1e-6, "us": 1e-3, "ms": 1.0, "ns": 1e-6, "s": 1e3}.get(u)
    return value * f if f is not None else value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("report")
    ap.add_argument("--workload", default="c5")
    ap.add_argument("--capture", default="")
    ap.add_argument("--json", default=None)
    ap.add_argument("--md", default=None)
    args = ap.parse_args()
    hdr, units, data = load(args.report)
    col = {h: i for i, h in enumerate(hdr)}
    kn = col["Kernel Name"]
    kernels = {}
    for row in data:
        name = re.sub(r"^void ", "", row[kn])
        name = re.sub(r"\(.*$", "", name)
        k = kernels.setdefault(name, {"launches": 0})
        k["launches"] += 1
        for key, metric, _ in KEYS:
            if metric in col:
                v = num(row[col[metric]])
                if v is None:
                    continue
                if key.endswith("_MB") or key.endswith("_ms"):
                    v = scale(v, units[col[metric]])
                if key == "smem_per_block_KB":
                    v = scale(v, units[col[metric]]) * 1e3 if units[col[metric]].lower().endswith("byte") else v
                if key == "sm_clock_mhz":
                    u = units[col[metric]].lower()
                    v = v * {"ghz": 1e3, "mhz": 1.0, "hz": 1e-6}.get(u, 1.0) if "hz" in u else v / 1e6
                k.setdefault(key, []).append(v)
        for h, i in col.items():
            if h.startswith(STALLS) and h.endswith("_per_issue_active.ratio"):
                v = num(row[i])
                if v is not None:
                    k.setdefault("stall", {}).setdefault(h[len(STALLS):-len("_per_issue_active.ratio")], []).append(v)
    summ = {}
    for name, k in kernels.items():
        s = {"launches": k["launches"]}
        for key, _, _ in KEYS:
            if key in k:
                s[key] = sum(k[key]) / len(k[key])
        if "stall" in k:
            st = {r: sum(v) / len(v) for r, v in k["stall"].items()}
            s["stalled_warps_per_issue"] = dict(sorted(st.items(), key=lambda kv: -kv[1])[:6])
        summ[name] = s
    md = ["| kernel | ms | DRAM R+W MB | warp inst | issue % | ALU % | FMA % | XU % | FP64 % | LSU wavefronts % | warps act. % | regs | top stall reasons (warps stalled per issue) |",
          "|---|---|---|---|---|---|---|---|---|---|---|---|---|"]
    for name, s in summ.items():
        g = lambda k, f="%.1f": (f % s[k]) if k in s else "-"
        stalls = ", ".join("%s %.1f" % kv for kv in list(s.get("stalled_warps_per_issue", {}).items())[:4])
        md.append("| `%s` | %s | %.1f | %s | %s | %s | %s | %s | %s | %s | %s | %s | %s |" % (
            name, g("duration_ms", "%.3f"), s.get("dram_read_MB", 0) + s.get("dram_write_MB", 0), g("warp_inst", "%.3g"),
            g("issue_active_pct"), g("pipe_alu_pct"), g("pipe_fma_pct"), g("pipe_xu_pct"), g("pipe_fp64_pct"),
            g("lsu_wavefronts_pct"), g("warps_active_pct"), g("registers", "%d"), stalls))
    text = "\n".join(md)
    print(text)
    if args.md:
        with open(args.md, "w") as f:
            f.write("# ncu --set full, capture %s, workload %s (%s)\n\n%s\n\nFull per-kernel figures:\n\n```json\n%s\n```\n" % (
                args.capture, args.workload, os.path.basename(args.report), text, json.dumps(summ, indent=1)))
    if args.json:
        stage_of = {"rollout": "rollout_win_kernel", "sample_grids": "sample_grids_v2_kernel"}
        out = {"workload": args.workload, "capture": "%s (%s)" % (args.capture, os.path.basename(args.report)), "kernels": {}}
        for stage, prefix in stage_of.items():
            for name, s in summ.items():
                if name.startswith(prefix):
                    pipes = {p: s.get("pipe_%s_pct" % p, 0.0) for p in ("alu", "fma", "xu", "fp64", "lsu")}
                    top = max(pipes, key=pipes.get)
                    out["kernels"][stage] = {
                        "kernel": name, "ms_under_ncu": s.get("duration_ms"),
                        "dram_bytes": (s.get("dram_read_MB", 0) + s.get("dram_write_MB", 0)) * 1e6,
                        "warp_inst": s.get("warp_inst"), "issue_active_pct": s.get("issue_active_pct"),
                        "dram_pct_of_peak": s.get("dram_pct_of_peak"), "busiest_pipe": "%s %.0f %%" % (top, pipes[top]),
                        "bound": "issue" if (s.get("issue_active_pct", 0) > 2 * s.get("dram_pct_of_peak", 0)) else "hbm"}
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
