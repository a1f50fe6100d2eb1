#!/usr/bin/env python
"""Summarise ncu outputs into small text files under profiles/.

  python tools/ncu_summarize.py launches launches_X.csv profiles/rNN_launches.txt
  python tools/ncu_summarize.py full     prof_X.ncu-rep profiles/rNN_kernel.txt
"""
import collections
import csv
import re
import subprocess
import sys

KEYS = ["Kernel Name", "Grid Size", "Block Size", "gpu__time_duration.sum", "dram__bytes_read.sum",
        "dram__bytes_write.sum", "dram__bytes_read.sum.per_second",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor.sum", "lts__t_bytes.sum", "l1tex__t_bytes_pipe_lsu_mem_global_op_ld.sum",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio"]


def launches(src, dst):
    lines = [l for l in open(src) if not l.startswith("==")]
    agg, total, n = collections.OrderedDict(), 0.0, 0
    for row in csv.DictReader(lines):
        v = float(row["Metric Value"].replace(",", ""))
        v = {"ns": v / 1e3, "us": v, "ms": v * 1e3, "s": v * 1e6}.get(row["Metric Unit"], v)
        key = (re.sub(r"\(.*", "", row["Kernel Name"])[:90], row.get("Grid Size", ""), row.get("Block Size", ""))
        a = agg.setdefault(key, [0, 0.0]); a[0] += 1; a[1] += v
        total += v; n += 1
    with open(dst, "w") as f:
        f.write(f"# source: {src}  (ncu --metrics gpu__time_duration.sum --clock-control none; cold-cache, serialised:\n"
                f"# compare SHARES, not absolutes)\n# launches {n}  total {total:.1f} us\n")
        f.write(f"{'share':>7} {'total_us':>10} {'count':>6} {'avg_us':>9}  kernel grid block\n")
        for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"{100 * t / total:6.2f}% {t:10.1f} {c:6d} {t / c:9.2f}  {k[0]} {k[1]} {k[2]}\n")
    print(open(dst).read())


def full(src, dst):
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = [(k, hdr.index(k)) for k in KEYS if k in hdr]
    with open(dst, "w") as f:
        f.write(f"# source: {src}  (ncu --set full --clock-control none --import-source on)\n")
        for r in rows[2:]:
            f.write("-" * 100 + "\n")
            for k, i in idx:
                f.write(f"{k:85s} {r[i]} {units[i]}\n")
    print(open(dst).read())


def traffic(src, dst, workload, key, units_per_launch, note=""):
    """Append/replace profiles/dominant_kernel_traffic.json[workload][key] from an ncu --set full
    capture: dram__bytes_read.sum + dram__bytes_write.sum of the FIRST kernel in the report,
    divided by the units (tokens) that launch processed."""
    import json
    import os
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units, r = rows[0], rows[1], rows[2]

    def val(name):
        i = hdr.index(name)
        v = float(r[i].replace(",", ""))
        return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}.get(units[i], 1)
    rd, wr = val("dram__bytes_read.sum"), val("dram__bytes_write.sum")
    n = float(units_per_launch)
    db = json.load(open(dst)) if os.path.exists(dst) else {}
    db.setdefault(workload, {})[key] = {
        "dram_bytes_per_token": (rd + wr) / n, "dram_read_bytes_per_launch": rd, "dram_write_bytes_per_launch": wr,
        "tokens_per_launch": n, "kernel": r[hdr.index("Kernel Name")][:60], "source": os.path.basename(src),
        "note": note}
    json.dump(db, open(dst, "w"), indent=1)
    print(json.dumps(db[workload][key], indent=1))


if __name__ == "__main__":
    {"launches": launches, "full": full, "traffic": traffic}[sys.argv[1]](*sys.argv[2:])
