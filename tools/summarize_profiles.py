#!/usr/bin/env python
"""Turns the raw ncu outputs in gpurun_out/ into the small tracked summaries under profiles/.

  python tools/summarize_profiles.py launches gpurun_out/launches.csv profiles/r01_launches_summary.txt
  python tools/summarize_profiles.py full gpurun_out/ncu_r01_fwd_conv2c.ncu-rep [...] > profiles/r01_ncu_full_summary.json
"""
import csv
import json
import subprocess
import sys
from collections import defaultdict


def launches(src, dst):
    rows = []
    with open(src, newline="") as f:
        lines = [ln for ln in f if not ln.startswith("==")]
    rd = csv.DictReader(lines)
    tot = defaultdict(lambda: [0, 0.0])
    n = 0
    for r in rd:
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(r["Metric Value"].replace(",", ""))
        unit = r["Metric Unit"]
        us = v / 1e3 if unit in ("ns", "nsecond") else (v * 1e3 if unit in ("ms", "msecond") else v)
        name = r["Kernel Name"].split("(")[0][:70]
        tot[name][0] += 1
        tot[name][1] += us
        n += 1
    total = sum(v[1] for v in tot.values())
    with open(dst, "w") as f:
        f.write("# ncu launch list of `python bench.py --steps 1 --warmup 1 --no-cpu-baseline --no-e2e`\n"
                "# (1 warm-up + 1 timed + 1 per-launch-profiled training step), `ncu --metrics gpu__time_duration.sum\n"
                "# --clock-control none`; per-launch times are cold-cache and serialised: compare SHARES, not absolutes.\n"
                "# %d launches, %.1f ms total\n# kernel | launches | total us | share\n" % (n, total / 1e3))
        for k, (c, us) in sorted(tot.items(), key=lambda kv: -kv[1][1]):
            f.write("%-72s %6d %12.1f %6.2f%%\n" % (k, c, us, 100 * us / total))


WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_bytes.sum",
        "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "sm__cycles_elapsed.max", "smsp__inst_executed.sum",
        "launch__shared_mem_per_block_dynamic", "l1tex__m_xbar2l1tex_read_bytes.sum",
        "l1tex__m_xbar2l1tex_read_bytes.sum.per_second", "sm__inst_executed.avg.per_cycle_elapsed",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "lts__t_sector_hit_rate.pct",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum.per_second",
        "dram__bytes_write.sum.per_second", "sm__inst_executed_pipe_tensor.sum"]


def full(reps):
    out = {}
    for rep in reps:
        txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        rows = list(csv.reader(txt.splitlines()))
        hdr, units = rows[0], rows[1]
        for n_launch, vals in enumerate(rows[2:]):
            d = {}
            for h, u, v in zip(hdr, units, vals):
                if h in WANT or h == "Kernel Name":
                    d[h] = v if h == "Kernel Name" else {"value": float(v.replace(",", "")) if v else None, "unit": u}
            key = rep.split("/")[-1]
            out[key if n_launch == 0 else "%s#%d" % (key, n_launch)] = d
    json.dump(out, sys.stdout, indent=1)


if __name__ == "__main__":
    if sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3])
    else:
        full(sys.argv[2:])
