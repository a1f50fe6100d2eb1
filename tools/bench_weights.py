#!/usr/bin/env python
"""Decode speed with fp32 and bf16 weight matrices (kllm_decoder_desc::weights), by position, in both numerics modes.

    python tools/bench_weights.py --workloads tinyllama-1.1b qwen2.5-0.5b llama2-7b

Per workload and numerics mode, decoders on one GPU over the same synthetic fp32 weights (bench.py's seed for the
workload): one with the fp32 matrices, one with the same matrices rounded to bf16 (decoder.bf16_weights), each on its
own stream; --bf16-stages adds bf16 decoders pinned to other ring-stage sizes (KLLM_STAGE_BYTES at create time).
Each cache is filled once by the batched prefill up to the last window; a window at position p then runs --window
consecutive greedy decode steps from p (kllm_decoder_generate, device resident), timed by device events on the
decoder's stream.  The decoders alternate in the same call for --reps rounds after a warm-up, and the median is
reported.

Output: ONE JSON line with, per workload, mode and window, tok/s of each decoder, the bytes one token must read (the
weights once in that decoder's format plus the K and V rows of every earlier position,
ModelShape.weight_bytes_per_token and kv_bytes_at) and the resulting fraction of the H100 SXM's 3.35 TB/s, with the
card's name and power limit read in the same run.  Needs a CUDA device; there is nothing to time without one.
"""
import argparse
import json
import os
import statistics
import sys
from dataclasses import replace
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from bench_prefill import SEEDS, gpu_card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # NVIDIA's data sheet figure for the H100 SXM
SEQ_LEN = 2048
POSITIONS = [1, 512, 2047]


def progress(*parts):
    print("[bench_weights]", *parts, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", nargs="+", default=["tinyllama-1.1b", "qwen2.5-0.5b", "llama2-7b"],
                    choices=["tinyllama-1.1b", "qwen2.5-0.5b", "llama2-7b"])
    ap.add_argument("--modes", nargs="+", default=["exact", "fast"], choices=["exact", "fast"])
    ap.add_argument("--window", type=int, default=64, help="decode steps per timed window")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bf16-stages", nargs="*", type=int, default=[],
                    help="also time bf16 decoders with these ring-stage sizes (bytes)")
    a = ap.parse_args()

    import torch
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    from kuiperllama_b200.decoder import bf16_weights
    if not torch.cuda.is_available():
        sys.exit("bench_weights: no CUDA device")
    os.environ.pop("KLLM_STAGE_BYTES", None)
    results = {}
    for name in a.workloads:
        shape = replace(SHAPES[name], seq_len=SEQ_LEN)
        w32 = synth_weights(shape, "cuda", SEEDS[name])
        w16 = bf16_weights(w32)
        W = a.window
        starts = {p: max(1, min(p, SEQ_LEN - W)) for p in POSITIONS}  # a window [s, s + W) near p, inside seq_len
        fill = max(starts.values())
        gen = torch.Generator().manual_seed(SEEDS[name])
        prompt = torch.randint(0, shape.vocab_size, (fill,), generator=gen).tolist()
        results[name] = {"seq_len": SEQ_LEN}
        for mode in a.modes:
            variants = [("fp32", "fp32", None), ("bf16", "bf16", None)]
            variants += [(f"bf16@{b}", "bf16", b) for b in a.bf16_stages]
            decs = {}
            for label, fmt, stage in variants:
                if stage is not None:
                    os.environ["KLLM_STAGE_BYTES"] = str(stage)
                s = torch.cuda.Stream()
                d = Decoder(shape, w16 if fmt == "bf16" else w32, stream=s.cuda_stream, numerics=mode,
                            weight_format=fmt)
                os.environ.pop("KLLM_STAGE_BYTES", None)
                d.prefill_tf32(prompt)
                decs[label] = (d, s, fmt)
                progress(name, mode, label, d.engine, f"stage {d.attention_geometry[3]}", f"filled to {fill}")

            def window(label, start):
                d, s, _ = decs[label]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(s)
                d.generate(prompt[start - 1], start, W)
                e1.record(s)
                e1.synchronize()
                return e0.elapsed_time(e1) / 1e3

            per = {}
            for p, start in starts.items():
                for label in decs:
                    window(label, start)  # warm-up
                t = {label: [] for label in decs}
                for _ in range(a.reps):
                    for label in decs:
                        t[label].append(window(label, start))
                row = {"window": [start, start + W - 1]}
                for label, (d, _, fmt) in decs.items():
                    tok_s = W / statistics.median(t[label])
                    # the window's middle position stands for its bytes per token
                    b = shape.weight_bytes_per_token(fmt) + shape.kv_bytes_at(start + W // 2)
                    row[label] = {"tok_s": round(tok_s, 1), "stage_bytes": d.attention_geometry[3],
                                  "bytes_per_token": b, "fraction_of_3.35TBps": round(b * tok_s / HBM_BYTES_PER_S, 3)}
                row["bf16_over_fp32"] = round(row["bf16"]["tok_s"] / row["fp32"]["tok_s"], 3)
                per[str(p)] = row
                progress(name, mode, json.dumps(row))
            results[name][mode] = {"engine": decs["bf16"][0].engine, "windows": per}
            for d, _, _ in decs.values():
                d.close()
            del decs
        del w32, w16
        torch.cuda.empty_cache()
    print(json.dumps({"window_steps": a.window, "reps": a.reps, "statistic": "median",
                      "timing": "CUDA events on the decoder's stream", "card": gpu_card(torch.cuda.current_device()),
                      "workloads": results}))


if __name__ == "__main__":
    main()
