#!/usr/bin/env python
"""Cost of recording log-probabilities (kllm_decoder_set_logprobs), and of scoring, on one GPU.

    python tools/bench_logprobs.py --workload qwen2.5-0.5b --steps 256 --reps 5

One exact-numerics decoder of the workload's model (synthetic weights, bench.py's seed) per engine (--engines,
KLLM_ENGINE at create time) runs kllm_decoder_generate windows of --steps positions from position 0 with logprobs
off, then top_n 0, 5 and 20, alternating for --reps repetitions after one warm-up window each, greedy and with
Qwen2.5-Instruct's sampling settings (T 0.7, top_k 20, top_p 0.8, repetition penalty 1.05).  Then --score-tokens
tokens are scored (kllm_decoder_score), generated teacher-forced (kllm_decoder_generate with a teacher) and fed as a
prompt (kllm_decoder_prompt), alternating.  Each window ends in a host synchronisation, so a host clock around it
times it.  Prints ONE JSON line: per engine and settings, the median tok/s of each mode and its overhead against
logprobs off; the median seconds of the three scoring paths; the card's name and power limit, read in the same run.
Needs a CUDA device.
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

SETTINGS = {"greedy": (0.0, 0, 1.0, 1.0), "qwen": (0.7, 20, 0.8, 1.05)}


def run_engine(workload, engine, steps, reps, score_tokens):
    import numpy as np
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    os.environ["KLLM_ENGINE"] = engine
    shape = SHAPES[workload]
    dec = Decoder(shape, synth_weights(shape, "cuda", SEEDS.get(workload, 1234)), numerics="exact")
    out = {"engine": dec.engine}

    def window(top_n):
        dec.set_logprobs(top_n)
        t0 = time.perf_counter()
        dec.generate(1, 0, steps)
        return time.perf_counter() - t0

    modes = {"off": -1, "n0": 0, "n5": 5, "n20": 20}
    for sname, (T, k, p, rp) in SETTINGS.items():
        dec.set_sampling(T, k, 42, top_p=p)
        dec.set_repetition_penalty(rp, 0)
        times = {m: [] for m in modes}
        for top_n in modes.values():
            window(top_n)
        for _ in range(max(1, reps)):
            for m, top_n in modes.items():
                times[m].append(window(top_n))
        rate = {m: steps / statistics.median(t) for m, t in times.items()}
        out[sname] = {"tok_s": rate, "overhead": {m: 1 - rate[m] / rate["off"] for m in modes if m != "off"}}
    dec.set_sampling(0.0)
    dec.set_repetition_penalty(1.0)
    dec.set_logprobs(-1)
    tokens = [int(t) for t in np.random.default_rng(0).integers(0, shape.vocab_size, score_tokens)]
    paths = {"score": lambda: dec.score(tokens), "generate_teacher": lambda: dec.generate(tokens[0], 0, score_tokens - 1, teacher=tokens),
             "prompt": lambda: dec.prompt(tokens[:-1])}
    times = {m: [] for m in paths}
    for f in paths.values():
        f()
    for _ in range(max(1, reps)):
        for m, f in paths.items():
            t0 = time.perf_counter()
            f()
            times[m].append(time.perf_counter() - t0)
    out["score_s"] = {m: statistics.median(t) for m, t in times.items()}
    dec.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", default="tinyllama-1.1b")
    ap.add_argument("--engines", default="persistent,graph")
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--score-tokens", type=int, default=1025)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the decode paths run on the GPU only")
    res = {"workload": a.workload, "steps": a.steps, "reps": a.reps, "card": gpu_card()}
    for e in a.engines.split(","):
        res[e] = run_engine(a.workload, e, a.steps, a.reps, a.score_tokens)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
