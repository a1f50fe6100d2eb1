#!/usr/bin/env python
"""Decode speed of the fast mode with an fp32, a bf16 and an fp8 KV cache (kllm_decoder_desc::kv_cache), by position.

    python tools/bench_kv_cache.py --workloads llama2-7b-int8 qwen2.5-0.5b tinyllama-1.1b
    python tools/bench_kv_cache.py --caches fp32 bf16 fp8

Per workload, fast-numerics decoders on one GPU over the same synthetic weights (bench.py's seed for the workload),
one per cache type of --caches (fp32 and bf16 by default; the fp8 cache at unit scales: its speed does not depend on
them), each on its own stream.  Each cache is filled once by the batched prefill up to the last
window; a window at position p then runs --window consecutive decode steps from p (kllm_decoder_generate, one
launch), which reads the cache rows < p only, so one fill serves every window.  A window is timed by device events
on the decoder's stream; the decoders alternate in the same call for --reps rounds after a warm-up, and the
median is reported.

Output: ONE JSON line with, per workload and window, tok/s for each cache type, the bytes one token must read
(the weights once plus the K and V rows of every earlier position, ModelShape.weight_bytes_per_token and
kv_bytes_at) and the resulting fraction of the H100 SXM's 3.35 TB/s, with the card's name and power limit read in
the same run.  Needs a CUDA device; there is nothing to time without one.
"""
import argparse
import json
import statistics
import sys
from dataclasses import replace
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from bench_prefill import SEEDS, gpu_card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # NVIDIA's data sheet figure for the H100 SXM
# seq_len and window positions per workload: the issue's long contexts, each model up to its own length
PLANS = {"llama2-7b-int8": (4096, [1, 1024, 2048, 4095]),
         "qwen2.5-0.5b": (32768, [1, 1024, 2048, 4095, 8192, 16384, 32767]),
         "tinyllama-1.1b": (2048, [1, 1024, 2047])}


def progress(*parts):
    print("[bench_kv_cache]", *parts, file=sys.stderr, flush=True)


def kv_bytes(shape, pos, kv_cache):
    return shape.kv_bytes_at(pos, kv_cache)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", nargs="+", default=list(PLANS), choices=list(PLANS))
    ap.add_argument("--window", type=int, default=64, help="decode steps per timed window")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--caches", nargs="+", default=["fp32", "bf16"], choices=["fp32", "bf16", "fp8"])
    a = ap.parse_args()

    import torch
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    if not torch.cuda.is_available():
        sys.exit("bench_kv_cache: no CUDA device")
    results = {}
    for name in a.workloads:
        seq_len, positions = PLANS[name]
        shape = replace(SHAPES[name], seq_len=seq_len)
        w = synth_weights(shape, "cuda", SEEDS[name])
        W = a.window
        starts = {p: max(1, min(p, seq_len - W)) for p in positions}  # a window [s, s + W) near p, inside seq_len
        fill = max(starts.values())
        gen = torch.Generator().manual_seed(SEEDS[name])
        prompt = torch.randint(0, shape.vocab_size, (fill,), generator=gen).tolist()
        decs = {}
        for kv in a.caches:
            s = torch.cuda.Stream()
            d = Decoder(shape, w, stream=s.cuda_stream, numerics="fast", kv_cache=kv)
            (d.prefill_w8 if shape.group_size else d.prefill_tf32)(prompt)
            decs[kv] = (d, s)
            progress(name, kv, f"cache filled to position {fill}")

        def window(kv, start):
            d, s = decs[kv]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            d.generate(prompt[start - 1], start, W)
            e1.record(s)
            e1.synchronize()
            return e0.elapsed_time(e1) / 1e3

        per = {}
        for p, start in starts.items():
            for kv in decs:
                window(kv, start)  # warm-up
            t = {kv: [] for kv in decs}
            for _ in range(a.reps):
                for kv in decs:
                    t[kv].append(window(kv, start))
            row = {"window": [start, start + W - 1]}
            for kv in decs:
                tok_s = W / statistics.median(t[kv])
                # the window's middle position stands for its bytes per token
                b = shape.weight_bytes_per_token() + kv_bytes(shape, start + W // 2, kv)
                row[kv] = {"tok_s": round(tok_s, 1), "bytes_per_token": b,
                           "fraction_of_3.35TBps": round(b * tok_s / HBM_BYTES_PER_S, 3)}
            for x, y in (("bf16", "fp32"), ("fp8", "fp32"), ("fp8", "bf16")):
                if x in decs and y in decs:
                    row[f"{x}_over_{y}"] = round(row[x]["tok_s"] / row[y]["tok_s"], 3)
            per[str(p)] = row
            progress(name, json.dumps(row))
        results[name] = {"seq_len": seq_len, "engine": next(iter(decs.values()))[0].engine, "windows": per}
        for d, _ in decs.values():
            d.close()
        del w, decs
        torch.cuda.empty_cache()
    print(json.dumps({"numerics": "fast", "window_steps": a.window, "reps": a.reps, "statistic": "median",
                      "timing": "CUDA events on the decoder's stream", "card": gpu_card(torch.cuda.current_device()),
                      "workloads": results}))


if __name__ == "__main__":
    main()
