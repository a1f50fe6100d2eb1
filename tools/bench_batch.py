"""Batched decoding on one GPU (DESIGN.md 5.14): B sequences stepped in one pass over the weights per step.

For each workload, batch size B and start position pos, B exact-numerics decoders on the default engine are built over
one synth_weights set with bench.py's seeds, and each is brought to pos by its own seeded prompt (the batched
prefill).  Then, host clock around synchronised calls, the arms alternated within each repetition, median of --reps:
  (a) kllm_batch_generate of --steps ids per member;
  (b) the same members, each running its own kllm_decoder_generate of --steps ids in turn (what a caller does
      without a batch);
  (c) one fast-numerics decoder's generate of --steps ids: the single-sequence headline rate.
(a)'s ids must equal (b)'s, or the run aborts.  batch_create_ms is kllm_batch_create's time, the capture of the
step's graph included.  Prints one JSON object per (workload, B, pos) and writes them all to --out.

    python tools/bench_batch.py [--workload tinyllama-1.1b,...] [--batch 1,2,4,8] [--pos 1,512,1024]
                                [--steps 64] [--reps 5] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

SEEDS = {"tinyllama-1.1b": 1235, "llama2-7b-int8": 1236, "qwen2.5-0.5b": 1237, "llama2-7b": 1238}  # bench.py's
WORKLOADS = ["tinyllama-1.1b", "qwen2.5-0.5b", "llama2-7b-int8", "llama2-7b:bf16"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.stdout.strip() else ""


def timed(fn):
    t0 = time.perf_counter()
    out = fn()  # every call below ends in a stream synchronise
    return (time.perf_counter() - t0) * 1e3, out


def bring_to(d, shape, pos, seed):
    """Feed d a seeded prompt of pos ids (batched prefill) and return the id it continues with."""
    import numpy as np
    prompt = [int(t) for t in np.random.default_rng(seed).integers(1, shape.vocab_size, pos)]
    return d.prefill_w8(prompt, 0) if shape.group_size else d.prefill_tf32(prompt, 0)


def run_workload(name, args, info):
    import torch
    from kuiperllama_b200 import SHAPES, Batch, Decoder, synth_weights
    from kuiperllama_b200.decoder import bf16_weights
    base, _, fmt = name.partition(":")
    fmt = fmt or "fp32"
    shape = SHAPES[base]
    w = synth_weights(shape, "cuda", SEEDS[base])
    if fmt == "bf16":
        w = bf16_weights(w)
        torch.cuda.empty_cache()
    os.environ.pop("KLLM_ENGINE", None)
    B_max = max(args.batch)
    members = [Decoder(shape, w, weight_format=fmt) for _ in range(B_max)]
    fast = Decoder(shape, w, weight_format=fmt, numerics="fast")
    rows = []
    for pos in args.pos:
        if pos + args.steps > shape.seq_len:
            raise SystemExit(f"{name}: pos {pos} + steps {args.steps} > seq_len {shape.seq_len}")
        firsts = [bring_to(d, shape, pos, 1000 * pos + b) for b, d in enumerate(members)]
        fast_first = bring_to(fast, shape, pos, 1000 * pos)
        for B in args.batch:
            ms = members[:B]
            create_ms, batch = timed(lambda: Batch(ms))
            starts = [pos] * B
            # warm-up: one pass of each arm
            batch.generate(firsts[:B], starts, args.steps)
            for b in range(B):
                ms[b].generate(firsts[b], pos, args.steps)
            fast.generate(fast_first, pos, args.steps)
            arms = {
                "a": lambda: batch.generate(firsts[:B], starts, args.steps),
                "b": lambda: [ms[b].generate(firsts[b], pos, args.steps) for b in range(B)],
                "c": lambda: fast.generate(fast_first, pos, args.steps),
            }
            times = {k: [] for k in arms}
            order = list(arms)
            for r in range(args.reps):
                outs = {}
                for k in order[r % 3:] + order[:r % 3]:
                    t, outs[k] = timed(arms[k])
                    times[k].append(t)
                if outs["a"] != outs["b"]:
                    raise SystemExit(f"{name} B={B} pos={pos}: the batch's ids differ from the members' own")
            batch.close()
            med = {k: statistics.median(v) for k, v in times.items()}
            tok = {k: (B if k != "c" else 1) * args.steps / (med[k] / 1e3) for k in med}
            row = {
                "workload": name, "engine": members[0].engine, "B": B, "pos": pos, "steps": args.steps,
                "reps": args.reps,
                "tok_s_batch": round(tok["a"], 1), "tok_s_members_in_turn": round(tok["b"], 1),
                "tok_s_fast_single": round(tok["c"], 1),
                "speedup_vs_in_turn": round(tok["a"] / tok["b"], 3), "speedup_vs_fast_single": round(tok["a"] / tok["c"], 3),
                "ms_per_batch_step": round(med["a"] / args.steps, 4),
                "batch_create_ms": round(create_ms, 2), "parity": "ids equal", **info,
            }
            print(json.dumps(row), flush=True)
            rows.append(row)
    for d in members + [fast]:
        d.close()
    del w
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default=",".join(WORKLOADS))
    ap.add_argument("--batch", default="1,2,4,8")
    ap.add_argument("--pos", default="1,512,1024")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    args.batch = [int(x) for x in args.batch.split(",")]
    args.pos = [int(x) for x in args.pos.split(",")]
    from kuiperllama_b200 import build
    build.build()
    name, power, clock = (card().split(", ") + ["", "", ""])[:3]
    info = {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    rows = []
    for wl in args.workload.split(","):
        rows += run_workload(wl, args, info)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
