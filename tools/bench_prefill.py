#!/usr/bin/env python
"""Prompt prefill on one GPU: the batched tensor-core prefill against the bit-exact prompt path.

    python tools/bench_prefill.py --workload llama2-7b-int8 --tokens 1024

One seeded N-token prompt of the workload's model (synthetic weights, the seed bench.py uses for that workload)
goes through the batched entry -- kllm_decoder_prefill_w8 for int8 checkpoints, kllm_decoder_prefill_tf32 for fp32
-- and through kllm_decoder_prompt (one forward per position) on one exact-numerics decoder.  Each call rewrites
positions 0 .. N-1 and ends in a host synchronisation, so a host clock around it times it; the two are warmed up
once each, then alternate for --reps repetitions, and the medians are reported.  Prints ONE JSON line:

  tokens, entry, batched_tok_s, stepping_tok_s, speedup, batched_ms, stepping_ms
  matmul_tflops      2 x layer matmul weights x N / batched wall time: a whole-prefill rate (attention, norms and
                     the last position's classifier are inside the time), not a kernel's share of peak
  max_logit_err_rel  last-position logits of the batched path vs the exact path, over max|logit|
  card               the GPU's name and power limit, read in the same run

Needs a CUDA device; there is nothing to time without one.
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

SEEDS = {"stories15m": 1234, "tinyllama-1.1b": 1235, "llama2-7b-int8": 1236, "qwen2.5-0.5b": 1237,
         "llama2-7b": 1238, "small": 1239}  # bench.py's per-workload seeds


def gpu_card(index=0):
    """The card's name and power limit (read-only queries), stated beside every absolute number taken on it."""
    import torch
    card = {"name": torch.cuda.get_device_name(index), "power_limit": None}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        if q.returncode == 0 and q.stdout.strip():
            card["power_limit"] = q.stdout.strip().splitlines()[0].strip()
    except (OSError, subprocess.TimeoutExpired):
        pass
    return card


def matmul_weights(shape):
    """Weights of the layer matmuls (wq wo, wk wv, w1 w2 w3), the classifier excluded."""
    d, h, kv, L = shape.dim, shape.hidden_dim, shape.kv_dim, shape.layer_num
    return L * (2 * d * d + 2 * kv * d + 3 * h * d)


def run(workload, n, reps, seed):
    import numpy as np
    import torch
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    shape = SHAPES[workload]
    if n > shape.seq_len:
        raise SystemExit(f"--tokens {n} exceeds the context of {shape.name} ({shape.seq_len})")
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the prefill paths run on the GPU only")
    w = synth_weights(shape, "cuda", seed)
    rng = np.random.default_rng(seed)
    toks = [1] + [int(t) for t in rng.integers(2, shape.vocab_size, n - 1)]
    dec = Decoder(shape, w, numerics="exact")
    entry = "kllm_decoder_prefill_w8" if shape.group_size else "kllm_decoder_prefill_tf32"
    batched = dec.prefill_w8 if shape.group_size else dec.prefill_tf32
    dec.prompt(toks)
    exact = dec.logits()
    batched(toks)
    got = dec.logits()
    t_batched, t_stepping = [], []
    for _ in range(max(1, reps)):
        t0 = time.perf_counter(); batched(toks); t_batched.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); dec.prompt(toks); t_stepping.append(time.perf_counter() - t0)
    engine = dec.engine
    dec.close()
    tb, ts = statistics.median(t_batched), statistics.median(t_stepping)
    return {"workload": workload, "shape": shape.name, "tokens": n, "entry": entry,
            "batched_tok_s": n / tb, "stepping_tok_s": n / ts, "speedup": ts / tb,
            "batched_ms": tb * 1e3, "stepping_ms": ts * 1e3, "reps": max(1, reps),
            "matmul_tflops": 2 * matmul_weights(shape) * n / tb / 1e12,
            "matmul_tflops_what": "2 x layer matmul weights x tokens / batched wall time: a whole-prefill rate "
                                  "(attention, norms and the last position's classifier included in the time)",
            "max_logit_err_rel": float(np.abs(got - exact).max() / np.abs(exact).max()),
            "stepping": "kllm_decoder_prompt (bit-exact, one forward per position)", "engine": engine,
            "numerics": "exact-numerics decoder; the batched entry is TF32 (include/kllm_b200.h states its tolerance)",
            "seed": seed, "card": gpu_card(torch.cuda.current_device())}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", default="llama2-7b-int8", choices=sorted(SEEDS))
    ap.add_argument("--tokens", type=int, default=1024, help="prompt length N")
    ap.add_argument("--reps", type=int, default=5, help="timed repetitions of each path; medians are reported")
    ap.add_argument("--seed", type=int, default=None, help="default: bench.py's seed for the workload")
    a = ap.parse_args()
    if a.tokens < 1:
        raise SystemExit("--tokens must be at least 1")
    seed = SEEDS[a.workload] if a.seed is None else a.seed
    print(json.dumps(run(a.workload, a.tokens, a.reps, seed)))


if __name__ == "__main__":
    main()
