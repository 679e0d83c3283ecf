#!/usr/bin/env python
"""Condense an .ncu-rep (read with `ncu -i`) into the numbers the roofline needs.

    ncu_report.py rep.ncu-rep [copy_GBps]             last captured launch -> one JSON object
    ncu_report.py rep.ncu-rep --all [copy_GBps]       slowest launch of every distinct kernel -> JSON list

copy_GBps: measured device-to-device copy bandwidth (default: the H100 value of dfno_b200.models.fused).
"""
import csv, io, json, os, re, subprocess, sys
args = [a for a in sys.argv[1:] if a != "--all"]
every = "--all" in sys.argv
rep = args[0]
if len(args) > 1:
    copy_gbs = float(args[1])
else:
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from dfno_b200.models.fused import H100_COPY_GBS as copy_gbs
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
u = dict(zip(hdr, units))
MULT = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-9, "us": 1e-6, "ms": 1e-3, "s": 1,
        "nsecond": 1e-9, "usecond": 1e-6, "msecond": 1e-3, "second": 1}


def condense(vals):
    m = dict(zip(hdr, vals))

    def f(k):
        try:
            return float(m[k].replace(",", ""))
        except Exception:
            return float("nan")

    def scaled(k):
        return f(k) * MULT.get(u.get(k, ""), 1)

    t = scaled("gpu__time_duration.sum")
    rd, wr = scaled("dram__bytes_read.sum"), scaled("dram__bytes_write.sum")
    stalls = sorted(((f(k), re.sub(r".*issue_stalled_(.*)_per_issue_active\.ratio$", r"\1", k)) for k in hdr
                     if k.startswith("smsp__average_warps_issue_stalled") and k.endswith("per_issue_active.ratio")
                     and "selected" not in k and f(k) == f(k)), reverse=True)[:4]
    pipes = {re.sub(r"^sm__inst_executed_pipe_(.*)\.avg.*", r"\1", k): round(f(k), 1) for k in hdr
             if k.startswith("sm__inst_executed_pipe_") and k.endswith(".avg.pct_of_peak_sustained_active") and f(k) > 5}
    return {
        "kernel": re.sub(r"\(.*", "", m.get("Kernel Name", ""))[:80], "duration_ms": t * 1e3,
        "dram_read_GB": rd / 1e9, "dram_write_GB": wr / 1e9, "dram_TBps": (rd + wr) / t / 1e12,
        "frac_of_measured_copy_bw": (rd + wr) / t / 1e9 / copy_gbs,
        "dram_throughput_pct_of_peak": f("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
        "l2_throughput_pct_of_peak": f("lts__throughput.avg.pct_of_peak_sustained_elapsed"),
        "tensor_pipe_active_pct": f("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"),
        "issue_active_pct": f("smsp__issue_active.avg.pct_of_peak_sustained_active"),
        "warps_active_pct": f("sm__warps_active.avg.pct_of_peak_sustained_active"),
        "registers_per_thread": f("launch__registers_per_thread"), "grid": f("launch__grid_size"),
        "block": f("launch__block_size"),
        "top_stalls_warps_per_issue": [[name, round(v, 2)] for v, name in stalls],
        "busy_pipes_pct": pipes,
    }


if not every:
    print(json.dumps(condense(rows[-1]), indent=1))
else:
    best = {}
    for r in rows[2:]:
        c = condense(r)
        if c["kernel"] and (c["kernel"] not in best or c["duration_ms"] > best[c["kernel"]]["duration_ms"]):
            best[c["kernel"]] = c
    print(json.dumps(sorted(best.values(), key=lambda c: -c["duration_ms"]), indent=1))
