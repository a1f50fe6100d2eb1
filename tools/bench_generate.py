#!/usr/bin/env python
"""The stoppable, streaming generate loop (kllm_decoder_generate_until) against kllm_decoder_generate.

    python tools/bench_generate.py --workloads tinyllama-1.1b qwen2.5-0.5b

Per workload, one exact-numerics decoder (synthetic weights, bench.py's seed for the workload) on the persistent
engine and one on the graph engine.  Every call ends in a host synchronisation, so a host clock around it times
it.  Each variant is warmed up once, then the variants of a measurement alternate for --reps repetitions and
the medians are reported:

  (a) overhead:     generate(n) against generate_until(max_steps = n) with a stop id that never occurs and a
                    callback, n = --steps: the cost of the stop check and the stream;
  (b) stop:         generate_until(max_steps = 1024) stopping at step --stop-at (the first step >= --stop-at
                    whose greedy id has not occurred before), against generate(stop step + 1);
  (c) first_token:  time from the call's start to the first callback of the (a) run, and one token's time;
  (d) graph:        the graph engine's host-driven generate_until(n) against its generate(n).

Prints ONE JSON line with the card's name and power limit, read in the same run.  Needs a CUDA device; there is
nothing to time without one.
"""
import argparse
import json
import os
import statistics
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from bench_prefill import SEEDS, gpu_card  # noqa: E402


def make(shape, weights, engine):
    from kuiperllama_b200 import Decoder
    old = os.environ.get("KLLM_ENGINE")
    os.environ["KLLM_ENGINE"] = engine  # read when the decoder is created
    try:
        return Decoder(shape, weights, numerics="exact")
    finally:
        if old is None:
            os.environ.pop("KLLM_ENGINE")
        else:
            os.environ["KLLM_ENGINE"] = old


def alternate(variants, reps):
    """variants: name -> fn() returning seconds; one warm-up each, then reps alternating rounds; medians."""
    for fn in variants.values():
        fn()
    times = {name: [] for name in variants}
    for _ in range(reps):
        for name, fn in variants.items():
            times[name].append(fn())
    return {name: statistics.median(v) for name, v in times.items()}


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def run_workload(workload, steps, stop_at, max_steps, reps):
    from kuiperllama_b200 import SHAPES, synth_weights
    shape = SHAPES[workload]
    if max(steps, max_steps) > shape.seq_len:
        raise SystemExit(f"{max(steps, max_steps)} positions exceed the context of {shape.name} ({shape.seq_len})")
    w = synth_weights(shape, "cuda", SEEDS[workload])
    dec = make(shape, w, "persistent")
    out = {"shape": shape.name, "engine": dec.engine}
    probe = dec.generate(1, 0, max_steps)
    never = next(t for t in range(shape.vocab_size) if t not in probe)
    first_cb = []

    def until_stream():
        t0 = time.perf_counter()
        seen = []
        dec.generate_until(1, 0, steps, [never], on_tokens=lambda t: seen.append(time.perf_counter()))
        first_cb.append(seen[0] - t0)
        return time.perf_counter() - t0

    a = alternate({"generate": lambda: timed(lambda: dec.generate(1, 0, steps)), "generate_until": until_stream}, reps)
    token_s = a["generate"] / steps
    out["a"] = {"steps": steps, "generate_tok_s": steps / a["generate"], "until_tok_s": steps / a["generate_until"],
                "overhead": a["generate_until"] / a["generate"] - 1.0}
    out["c"] = {"first_callback_ms": 1e3 * statistics.median(first_cb[1:]), "token_ms": 1e3 * token_s}

    j = next((j for j in range(stop_at, max_steps) if probe[j] not in probe[:j]), None)
    if j is not None:
        assert dec.generate_until(1, 0, max_steps, [probe[j]]) == probe[:j + 1]
        b = alternate({"generate": lambda: timed(lambda: dec.generate(1, 0, j + 1)),
                       "until": lambda: timed(lambda: dec.generate_until(1, 0, max_steps, [probe[j]]))}, reps)
        out["b"] = {"stop_step": j, "max_steps": max_steps, "generate_ms": 1e3 * b["generate"],
                    "until_ms": 1e3 * b["until"], "extra_ms": 1e3 * (b["until"] - b["generate"]),
                    "extra_tokens": (b["until"] - b["generate"]) / token_s}
    dec.close()

    g = make(shape, w, "graph")
    d = alternate({"generate": lambda: timed(lambda: g.generate(1, 0, steps)),
                   "until": lambda: timed(lambda: g.generate_until(1, 0, steps, [never]))}, reps)
    out["d"] = {"engine": g.engine, "steps": steps, "generate_tok_s": steps / d["generate"],
                "until_tok_s": steps / d["until"], "overhead": d["until"] / d["generate"] - 1.0}
    g.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workloads", nargs="+", default=["tinyllama-1.1b", "qwen2.5-0.5b"], choices=sorted(SEEDS))
    ap.add_argument("--steps", type=int, default=256, help="n of (a), (c) and (d)")
    ap.add_argument("--stop-at", type=int, default=32, help="step of (b)'s stop")
    ap.add_argument("--max-steps", type=int, default=1024, help="max_steps of (b)")
    ap.add_argument("--reps", type=int, default=5, help="timed repetitions of each variant; medians are reported")
    a = ap.parse_args()
    if a.steps < 1 or a.stop_at < 0 or a.max_steps <= a.stop_at or a.reps < 2:
        raise SystemExit("need --steps >= 1, 0 <= --stop-at < --max-steps and --reps >= 2")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the decode paths run on the GPU only")
    res = {w: run_workload(w, a.steps, a.stop_at, a.max_steps, a.reps) for w in a.workloads}
    print(json.dumps({"reps": a.reps, "numerics": "exact", "workloads": res,
                      "card": gpu_card(torch.cuda.current_device())}))


if __name__ == "__main__":
    main()
