"""Speculative decoding on one GPU in the exact numerics (DESIGN.md 5.13).

(a) The cost of one verify pass of n = 1..8 positions against one exact-mode step of the persistent engine and of the
    graph engine, at positions 1, 512 and 2040 (2040 + 8 <= seq_len 2048): host clock around synchronised calls,
    median of --reps, the arms alternated within each repetition.  break_even = verify_ms(n) / persistent_step_ms is
    the tokens a round must yield to pay for itself.
(b) End to end: kllm_decoder_generate_speculative against kllm_decoder_generate_until in tok/s, on a repetitive prompt
    and on the model's own greedy continuation from token 1; the ids must be equal and the stats equal
    speculative.simulate_rounds.

Synthetic weights with bench.py's seeds.  Prints one JSON object per line and writes them all to --out.

    python tools/bench_speculative.py [--workloads tinyllama-1.1b,...] [--reps 20] [--out results.json]
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

SEEDS = {"tinyllama-1.1b": 1235, "llama2-7b-int8": 1236, "qwen2.5-0.5b": 1237, "llama2-7b": 1238}
WORKLOADS = ["tinyllama-1.1b", "qwen2.5-0.5b", "llama2-7b-int8", "llama2-7b:bf16"]
POSITIONS = [1, 512, 2040]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn):
    t0 = time.perf_counter()
    fn()  # every call below ends in a stream synchronise
    return (time.perf_counter() - t0) * 1e3


def decoders(name):
    import torch
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    from kuiperllama_b200.decoder import bf16_weights
    base, _, fmt = name.partition(":")
    shape = SHAPES[base]
    w = synth_weights(shape, "cuda", SEEDS[base])
    if fmt == "bf16":
        w = bf16_weights(w)
        torch.cuda.empty_cache()
    fmt = fmt or "fp32"
    os.environ.pop("KLLM_ENGINE", None)
    pers = Decoder(shape, w, weight_format=fmt)
    os.environ["KLLM_ENGINE"] = "graph"
    graph = Decoder(shape, w, weight_format=fmt)
    os.environ.pop("KLLM_ENGINE", None)
    return shape, pers, graph


def cost(name, pers, graph, reps):
    rows = []
    for p in POSITIONS:
        arms = [("persistent_step", lambda: pers.generate(1, p, 1)), ("graph_step", lambda: graph.generate(1, p, 1))]
        arms += [(f"verify_{n}", (lambda n=n: pers.verify([1] * n, p))) for n in range(1, 9)]
        for _, fn in arms:  # warm-up, and the capture of each verify length
            fn()
        t = {k: [] for k, _ in arms}
        for _ in range(reps):
            for k, fn in arms:
                t[k].append(timed(fn))
        med = {k: statistics.median(v) for k, v in t.items()}
        step = med["persistent_step"]
        row = {"workload": name, "pos": p, "persistent_step_ms": round(step, 4),
               "graph_step_ms": round(med["graph_step"], 4)}
        for n in range(1, 9):
            row[f"verify_{n}_ms"] = round(med[f"verify_{n}"], 4)
            row[f"break_even_{n}"] = round(med[f"verify_{n}"] / step, 3)
        rows.append(row)
    return rows


def end_to_end(name, shape, pers, draft_len, steps, reps):
    from kuiperllama_b200.speculative import simulate_rounds
    rows = []
    pattern = [(17 * i + 5) % shape.vocab_size for i in range(16)]
    cases = {"repetitive_prompt": pattern * 4, "own_continuation": [1]}
    for case, prompt in cases.items():
        def prep():
            if len(prompt) > 1:
                pers.prompt(prompt, 0)
            return prompt[-1], len(prompt) - 1
        first, p = prep()
        ctx = [int(t) for t in pers.history()[:p]] + [first]
        t_until, t_spec = [], []
        ref = spec = stats = None
        for _ in range(reps):
            prep()
            t0 = time.perf_counter()
            ref = pers.generate_until(first, p, steps)
            t_until.append(time.perf_counter() - t0)
            prep()
            t0 = time.perf_counter()
            spec, stats = pers.generate_speculative(first, p, steps, draft_len=draft_len)
            t_spec.append(time.perf_counter() - t0)
        assert spec == ref, f"{name} {case}: speculative ids differ"
        sim = simulate_rounds(ctx, spec, draft_len=draft_len, ngram_max=3, max_steps=steps, seq_len=shape.seq_len)
        assert sim == stats, (sim, stats)
        tu, ts = statistics.median(t_until), statistics.median(t_spec)
        rows.append({"workload": name, "case": case, "draft_len": draft_len, "steps": steps,
                     "until_tok_s": round(len(ref) / tu, 1), "speculative_tok_s": round(len(spec) / ts, 1),
                     "speedup": round(tu / ts, 3), "tokens_per_round": round(len(spec) / stats["rounds"], 3),
                     **stats, "stats_match_simulate_rounds": sim == stats})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--draft-lens", default="2,4,7")
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_speculative: no CUDA device")
    from kuiperllama_b200 import build
    build.build()
    results = [{"card": card()}]
    print(json.dumps(results[0]), flush=True)
    for name in args.workloads.split(","):
        try:
            shape, pers, graph = decoders(name)
            pers.verify([1], 1)
        except Exception as e:  # reported, and the next workload still runs
            print(json.dumps({"workload": name, "error": str(e)}), flush=True)
            continue
        out = cost(name, pers, graph, args.reps)
        graph.close()
        for d in (int(x) for x in args.draft_lens.split(",")):
            out += end_to_end(name, shape, pers, d, args.steps, max(3, args.reps // 5))
        pers.close()
        for r in out:
            print(json.dumps(r), flush=True)
        results += out
        torch.cuda.empty_cache()
    results.append({"card_after": card()})
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
