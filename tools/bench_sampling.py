#!/usr/bin/env python
"""Decode throughput with sampling against greedy, on one GPU and one decoder.

    python tools/bench_sampling.py --workload qwen2.5-0.5b --steps 256

One exact-numerics decoder of the workload's model (synthetic weights, bench.py's seed for the workload) runs
kllm_decoder_generate windows of --steps positions from position 0: greedy, then temperature --temperature with
top_k 0, then with top_k --top-k, switched by kllm_decoder_set_sampling between windows (the engine is not
rebuilt).  With --top-p P two more modes run: top_p P alone, and top_k --top-k with top_p P
(kllm_decoder_set_sampling_top_p).  With --repetition-penalty R every mode also runs with the penalty R over
the last --repeat-last-n positions (0: the whole sequence; kllm_decoder_set_repetition_penalty), alternating with
the same mode without it.  --start-pos P starts the windows at position P, after an untimed generate that fills
positions [0, P), so that the penalty scans a history of that length.  Each window ends in a host
synchronisation, so a host clock around it times it.  Every mode is warmed up once, then the modes alternate for
--reps repetitions and the medians are reported.  Prints ONE JSON line:

  greedy_tok_s, sampled_tok_s {mode: tok/s}, overhead {mode: 1 - sampled / greedy}, engine, card (the GPU's
  name and power limit, read in the same run); with --top-p also nucleus_size {mode: mean}, the mean number of
  tokens the rule keeps per position, from a step loop over the same positions after the timed windows (the
  numpy mirror on the run's own logits): a top-p rate means little without it.  With --repetition-penalty,
  the modes with the penalty are named "<mode>+rp", and penalty_overhead {mode: 1 - rate with / rate without}.

--frequency F, --presence P (kllm_decoder_set_frequency_presence, counting from --start-pos: the ids generated in
the window) and --logit-bias N (N random ids with biases in [-2, 2], kllm_decoder_set_logit_bias) join the settings
of the "+rp" modes in the same way; they run without a repetition penalty unless --repetition-penalty is given.

Needs a CUDA device; there is nothing to time without one.
"""
import argparse
import json
import math
import random
import statistics
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from bench_prefill import SEEDS, gpu_card  # noqa: E402


def run(workload, steps, reps, seed, temperature, top_k, top_p=None, penalty=None, last_n=0, start_pos=0,
        frequency=0.0, presence=0.0, n_bias=0):
    import torch
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    shape = SHAPES[workload]
    if start_pos + steps > shape.seq_len:
        raise SystemExit(f"--start-pos + --steps {start_pos + steps} exceeds the context of {shape.name} ({shape.seq_len})")
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the decode paths run on the GPU only")
    dec = Decoder(shape, synth_weights(shape, "cuda", seed), numerics="exact")
    modes = [("greedy", 0.0, 0, 1.0), ("top_k=0", temperature, 0, 1.0), (f"top_k={top_k}", temperature, top_k, 1.0)]
    if top_p is not None:
        modes += [(f"top_p={top_p}", temperature, 0, top_p), (f"top_k={top_k},top_p={top_p}", temperature, top_k, top_p)]
    runs = [(name, t, k, p, False) for name, t, k, p in modes]
    extras = frequency != 0 or presence != 0 or n_bias > 0
    rng = random.Random(seed)
    bias = {}
    while len(bias) < n_bias:
        bias[rng.randrange(shape.vocab_size)] = rng.uniform(-2, 2)
    if penalty is not None or extras:  # each mode with the settings right after the same mode without them
        runs = [r for name, t, k, p in modes for r in ((name, t, k, p, False), (name + "+rp", t, k, p, True))]
    times = {r[0]: [] for r in runs}
    if start_pos > 0:  # the cache and the history of the positions before the windows
        dec.generate(1, 0, start_pos)

    def window(t, k, p, on):
        dec.set_sampling(t, k, seed, top_p=p)
        dec.set_repetition_penalty(penalty if on and penalty is not None else 1.0, last_n)
        if extras:
            dec.set_frequency_presence(frequency if on else 0.0, presence if on else 0.0, start_pos)
            dec.set_logit_bias(bias if on else None)
        t0 = time.perf_counter()
        dec.generate(1, start_pos, steps)
        return time.perf_counter() - t0

    for _, t, k, p, on in runs:
        window(t, k, p, on)
    for _ in range(max(1, reps)):
        for name, t, k, p, on in runs:
            times[name].append(window(t, k, p, on))
    dec.set_repetition_penalty(1.0)
    dec.set_frequency_presence(0.0, 0.0)
    dec.set_logit_bias(None)
    nucleus = {}
    if top_p is not None:  # untimed: the same positions stepped one by one, the kept set from each step's logits
        from kuiperllama_b200 import sampling
        for name, t, k, p in modes[1:]:
            dec.set_sampling(t, k, seed, top_p=p)
            tok, sizes = 1, []
            for pos in range(start_pos, start_pos + steps):
                tok = dec.step(tok, pos)
                sizes.append(sampling.nucleus_size(dec.logits(), t, k, p))
            nucleus[name] = statistics.fmean(sizes)
    engine = dec.engine
    dec.close()
    rate = {name: steps / statistics.median(v) for name, v in times.items()}
    g = rate["greedy"]
    sampled = {name: r for name, r in rate.items() if name != "greedy"}
    out = {"workload": workload, "shape": shape.name, "steps": steps, "reps": max(1, reps),
           "temperature": temperature, "greedy_tok_s": g, "sampled_tok_s": sampled,
           "overhead": {name: 1.0 - r / g for name, r in sampled.items()},
           "engine": engine, "numerics": "exact", "seed": seed, "card": gpu_card(torch.cuda.current_device())}
    if penalty is not None or extras:
        out.update(repetition_penalty=penalty, repeat_last_n=last_n, start_pos=start_pos, frequency=frequency,
                   presence=presence, logit_bias_ids=n_bias,
                   penalty_overhead={name: 1.0 - rate[name + "+rp"] / rate[name] for name, _, _, _ in modes})
    if top_p is not None:
        out["nucleus_size"] = nucleus
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", default="tinyllama-1.1b", choices=sorted(SEEDS))
    ap.add_argument("--steps", type=int, default=256, help="positions per generate window")
    ap.add_argument("--reps", type=int, default=7, help="timed windows of each mode; medians are reported")
    ap.add_argument("--temperature", type=float, default=0.8)
    ap.add_argument("--top-k", type=int, default=40)
    ap.add_argument("--top-p", type=float, default=None, help="also time top-p alone and top-k with top-p")
    ap.add_argument("--repetition-penalty", type=float, default=None,
                    help="also time every mode with this repetition penalty")
    ap.add_argument("--repeat-last-n", type=int, default=0, help="the penalty's window (0: the whole sequence)")
    ap.add_argument("--frequency", type=float, default=0.0, help="frequency penalty of the +rp modes")
    ap.add_argument("--presence", type=float, default=0.0, help="presence penalty of the +rp modes")
    ap.add_argument("--logit-bias", type=int, default=0, help="number of biased ids in the +rp modes")
    ap.add_argument("--start-pos", type=int, default=0, help="first position of the timed windows")
    ap.add_argument("--seed", type=int, default=None, help="default: bench.py's seed for the workload")
    a = ap.parse_args()
    if a.steps < 1:
        raise SystemExit("--steps must be at least 1")
    if a.top_p is not None and not 0 < a.top_p <= 1:
        raise SystemExit("--top-p must be in (0, 1]")
    if a.repetition_penalty is not None and not (math.isfinite(a.repetition_penalty) and a.repetition_penalty > 0):
        raise SystemExit("--repetition-penalty must be finite and > 0")
    if a.repeat_last_n < 0 or a.start_pos < 0:
        raise SystemExit("--repeat-last-n and --start-pos must be >= 0")
    seed = SEEDS[a.workload] if a.seed is None else a.seed
    print(json.dumps(run(a.workload, a.steps, a.reps, seed, a.temperature, a.top_k, a.top_p, a.repetition_penalty,
                         a.repeat_last_n, a.start_pos, a.frequency, a.presence, a.logit_bias)))


if __name__ == "__main__":
    main()
