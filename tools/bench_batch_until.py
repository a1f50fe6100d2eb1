"""Ragged requests in one batch (DESIGN.md 5.15): kllm_batch_generate_until, whose passes shrink to the members still
running, against what a caller does without it.

For each workload, batch size B and start position pos, B exact-numerics decoders on the default engine are built over
one synth_weights set with bench.py's seeds, and each is brought to pos by its own seeded prompt (the batched prefill),
as tools/bench_batch.py does.  Member b may produce up to max_steps[b] = RAGGED[b] ids.  Two variants:
  ragged: no stop ids, so member b ends at max_steps[b];
  stops:  member b's stop id is the id of its own greedy continuation at the first occurrence at or after step
          max_steps[b] / 2, so members end on a stop.
Host clock around synchronised calls, the arms alternated within each repetition, median of --reps:
  (a) kllm_batch_generate_until with the ragged lengths and the variant's stops;
  (b) kllm_batch_generate to the longest length, each member's ids cut after its end (what a caller does without (a));
  (c) each member's own kllm_decoder_generate_until in turn;
  (d) the loop's own cost: (a)'s call with --loop-steps ids for every member and no stops, over kllm_batch_generate of
      the same length; loop_ratio = t(until) / t(generate).
Useful ids are sum_b n_out[b].  Also measured in the same run: t(k), the time of one batch step of k rows
(kllm_batch_generate of --loop-steps ids over members[:k]), and predicted_ms = sum_k passes_k * t(k), where
passes_k is the number of (a)'s passes that carried k rows.  (a)'s ids must equal (c)'s, or the run aborts.  Prints
one JSON object per (workload, B, pos, variant) and writes them all to --out.

    python tools/bench_batch_until.py [--workload tinyllama-1.1b,qwen2.5-0.5b,llama2-7b:bf16] [--batch 4,8]
                                      [--pos 1,512] [--reps 3] [--loop-steps 64] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from bench_batch import SEEDS, bring_to, card, timed  # noqa: E402

WORKLOADS = ["tinyllama-1.1b", "qwen2.5-0.5b", "llama2-7b:bf16"]  # llama2-7b-int8 on request (--workload)
RAGGED = [16, 24, 32, 48, 64, 96, 128, 256]


def median_ms(fn, reps):
    return statistics.median(timed(fn)[0] for _ in range(reps))


def rows_per_pass(n_out):
    """passes_k: how many passes carried k rows, for k = 1 .. B."""
    out = {}
    for p in range(max(n_out)):
        k = sum(1 for n in n_out if n > p)
        out[k] = out.get(k, 0) + 1
    return out


def cut(ids, stops):
    return next((ids[:j + 1] for j in range(len(ids)) if ids[j] in stops), ids)


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
    rows = []
    for pos in args.pos:
        if pos + max(RAGGED[:B_max] + [args.loop_steps]) > shape.seq_len:
            raise SystemExit(f"{name}: pos {pos} leaves too little of seq_len {shape.seq_len}")
        firsts = [bring_to(d, shape, pos, 1000 * pos + b) for b, d in enumerate(members)]
        for B in args.batch:
            ms, starts, steps, M = members[:B], [pos] * B, RAGGED[:B], max(RAGGED[:B])
            # t(k): one batch step of k rows, each batch warmed by one call
            step_ms = {}
            for k in range(1, B + 1):
                bk = Batch(ms[:k])
                bk.generate(firsts[:k], starts[:k], args.loop_steps)
                step_ms[k] = median_ms(lambda: bk.generate(firsts[:k], starts[:k], args.loop_steps), args.reps) / \
                    args.loop_steps
                bk.close()
            batch = Batch(ms)
            own = [ms[b].generate_until(firsts[b], pos, steps[b]) for b in range(B)]
            for variant in ("ragged", "stops"):
                if variant == "ragged":
                    stops = [[] for _ in range(B)]
                else:
                    stops = []
                    for b in range(B):
                        ids = own[b]
                        hits = [j for j in range(steps[b] // 2, steps[b]) if ids[j] not in ids[:j]]
                        stops.append([ids[hits[0] if hits else 0]])  # a first occurrence: the stop lands there
                L = args.loop_steps
                arms = {
                    "a": lambda: batch.generate_until(firsts[:B], starts, steps, stops),
                    "b": lambda: [cut(r[:steps[b]], stops[b]) for b, r in enumerate(batch.generate(firsts[:B], starts, M))],
                    "c": lambda: [ms[b].generate_until(firsts[b], pos, steps[b], stops[b]) for b in range(B)],
                    "d_until": lambda: batch.generate_until(firsts[:B], starts, [L] * B, [[]] * B),
                    "d_generate": lambda: batch.generate(firsts[:B], starts, L),
                }
                for f in arms.values():  # warm-up: every graph the arms launch, captured and loaded
                    f()
                times = {k: [] for k in arms}
                order = list(arms)
                outs = {}
                for r in range(args.reps):
                    for k in order[r % len(order):] + order[:r % len(order)]:
                        t, outs[k] = timed(arms[k])
                        times[k].append(t)
                    ids_a, stats = outs["a"]
                    if ids_a != outs["c"] or ids_a != outs["b"]:
                        raise SystemExit(f"{name} B={B} pos={pos} {variant}: the batch's ids differ from the members' own")
                    if outs["d_until"][0] != outs["d_generate"]:
                        raise SystemExit(f"{name} B={B} pos={pos}: generate_until differs from generate")
                med = {k: statistics.median(v) for k, v in times.items()}
                n_out = [len(x) for x in ids_a]
                useful = sum(n_out)
                per_k = rows_per_pass(n_out)
                predicted = sum(c * step_ms[k] for k, c in per_k.items())
                row = {
                    "workload": name, "engine": ms[0].engine, "B": B, "pos": pos, "variant": variant,
                    "max_steps": steps, "n_out": n_out, "passes": stats["passes"], "rows": stats["rows"],
                    "reps": args.reps,
                    "ids_s_until": round(useful / (med["a"] / 1e3), 1),
                    "ids_s_generate_cut": round(useful / (med["b"] / 1e3), 1),
                    "ids_s_members_in_turn": round(useful / (med["c"] / 1e3), 1),
                    "speedup_vs_generate_cut": round(med["b"] / med["a"], 3),
                    "speedup_vs_in_turn": round(med["c"] / med["a"], 3),
                    "ms_until": round(med["a"], 2), "ms_predicted": round(predicted, 2),
                    "step_ms_by_rows": {k: round(v, 4) for k, v in step_ms.items()},
                    "loop_steps": L, "ms_loop_until": round(med["d_until"], 2),
                    "ms_loop_generate": round(med["d_generate"], 2),
                    "loop_ratio": round(med["d_until"] / med["d_generate"], 4),
                    "parity": "ids equal", **info,
                }
                print(json.dumps(row), flush=True)
                rows.append(row)
            batch.close()
    for d in members:
        d.close()
    del w
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default=",".join(WORKLOADS))
    ap.add_argument("--batch", default="4,8")
    ap.add_argument("--pos", default="1,512")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loop-steps", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    args.batch = [int(x) for x in args.batch.split(",")]
    args.pos = [int(x) for x in args.pos.split(",")]
    if max(args.batch) > len(RAGGED):
        raise SystemExit(f"--batch at most {len(RAGGED)}")
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
