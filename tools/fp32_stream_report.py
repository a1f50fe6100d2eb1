#!/usr/bin/env python
"""Where the fp32 decode step's time goes, set against what the card can read.

    python tools/fp32_stream_report.py [--workload tinyllama-1.1b] [--pos 1 512]

Prints the card (name, power limit, clocks.max.sm), the measured read ceiling (a read-only fp32
reduction over 4.3 GB, device events, median of 5) and the phase timelines of tools/phase_timeline.py
in the fast numerics at the given positions.  The timelines' "prod_blk" column is the time the ring
producer waited for a free slot, i.e. the ring was full: of copies still in flight, or of stages the consumers
had not read yet.  Set against the consumers' own wait for a stage ("ringwait"), it shows which side holds the
ring.
"""
import argparse
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power, mhz = (f.strip() for f in out.split(","))
    return name, power, float(mhz.split()[0])


def read_ceiling(gbytes=4.3, reps=5):
    import torch
    n = int(gbytes * 1e9) // 4
    x = torch.ones(n, dtype=torch.float32, device="cuda")
    for _ in range(2):
        x.sum()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        x.sum()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
    times.sort()
    t = times[len(times) // 2]
    del x
    torch.cuda.empty_cache()
    return n * 4 / t / 1e12, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="tinyllama-1.1b")
    ap.add_argument("--pos", type=int, nargs="+", default=[1, 512])
    a = ap.parse_args()
    name, power, mhz = card()
    print(f"# card: {name}, power limit {power}, clocks.max.sm {mhz:.0f} MHz")
    tbs, t = read_ceiling()
    print(f"# read ceiling: torch sum over 4.3 GB fp32, median of 5: {tbs:.3f} TB/s ({t * 1e3:.2f} ms), "
          f"{tbs / 3.35:.3f} of the 3.35 TB/s data sheet", flush=True)
    env = dict(os.environ, KLLM_MODE="fast")
    for pos in a.pos:
        print(f"\n## {a.workload}, numerics fast, pos {pos}", flush=True)
        subprocess.run([sys.executable, str(ROOT / "tools" / "phase_timeline.py"), "--workload", a.workload,
                        "--pos", str(pos), "--ghz", str(mhz / 1e3)], env=env, check=True)


if __name__ == "__main__":
    main()
