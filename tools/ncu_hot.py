#!/usr/bin/env python
"""Hot-loop view of an `ncu --set full --import-source on` capture: per SASS instruction the executed
count and the warp-stall samples by reason, for the N most-sampled instructions plus kernel totals.

    python tools/ncu_hot.py x.ncu-rep [N] > profiles/rNN_x_hot.txt
"""
import collections
import csv
import subprocess
import sys


def main():
    rep = sys.argv[1]
    top = int(sys.argv[2]) if len(sys.argv) > 2 else 40
    out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    h = rows[1]
    col = {c: i for i, c in enumerate(h)}
    reasons = [c for c in h if c.startswith("stall_") and "Not Issued" not in c]
    data = []
    for r in rows[2:]:
        try:
            data.append((int(r[col["# Samples"]]), int(r[col["Instructions Executed"]]), r[col["Address"]],
                         r[col["Source"]], {k: int(r[col[k]] or 0) for k in reasons}))
        except (ValueError, IndexError):
            pass
    tot_s = sum(d[0] for d in data)
    tot_i = sum(d[1] for d in data)
    agg = collections.Counter()
    for d in data:
        agg.update(d[4])
    print(f"# {rep}: {rows[0][1] if len(rows[0]) > 1 else ''}")
    print(f"# warp-instructions executed {tot_i}, stall samples {tot_s}")
    print("# stall samples by reason: " + ", ".join(f"{k[6:]} {100 * v / max(1, tot_s):.1f}%" for k, v in agg.most_common(10)))
    ops = collections.Counter()
    for d in data:
        s = d[3].split()
        if s:
            ops[(s[1] if s[0].startswith("@") and len(s) > 1 else s[0]).split(".")[0]] += d[1]
    print("# executed by opcode: " + ", ".join(f"{k} {100 * v / max(1, tot_i):.1f}%" for k, v in ops.most_common(16)))
    print(f"{'samples':>8} {'%':>5} {'executed':>11}  top stall reasons                      instruction")
    for smp, ex, addr, src, st in sorted(data, key=lambda d: -d[0])[:top]:
        rs = ", ".join(f"{k[6:]}:{v}" for k, v in sorted(st.items(), key=lambda kv: -kv[1])[:3] if v)
        print(f"{smp:8d} {100 * smp / max(1, tot_s):5.2f} {ex:11d}  {rs:38s} {src[:70]}")


if __name__ == "__main__":
    main()
