"""Beam search over a batch of decoders (DESIGN.md 5.16): kllm_batch_beam_search against the same search composed on
the host from the other public entries, and against not searching.

For each workload, beam count B and start position pos, B exact-numerics decoders on the default engine are built over
one synth_weights set with bench.py's seeds; member 0 is brought to pos by a seeded prompt (the batched prefill), as
tools/bench_batch_until.py does.  Every search runs --new ids with no eos, so it runs its full length.  Host clock
around synchronised calls, the arms alternated within each repetition, median of --reps:
  (a) Batch.beam_search (kllm_batch_beam_search);
  (b) the same rule (kuiperllama_b200/beam.py) driven from the host: Batch.step for each pass, kllm_logprobs_f32 once
      per beam, and one synchronised copy_prefix of the whole prefix per fork, by the same relabelling as (a);
  (c) member 0's greedy generate_until of --new ids, the cost of not searching.
(a)'s hypotheses must equal (b)'s, or the run aborts.  Also measured: t(B), one batch step of B rows
(Batch.generate of --new ids over the B members, per step), and, in a separate torch.profiler run of (a), the fork
kernel's and the candidates kernel's mean times.  fork_bytes_per_pass = fork_rows * 2 * layers * kv_dim * 4 / passes.
Prints one JSON object per (workload, B, pos) and writes them all to --out.

    python tools/bench_beam.py [--workload tinyllama-1.1b,qwen2.5-0.5b,llama2-7b:bf16] [--beams 2,4,8]
                               [--pos 1,512] [--new 64] [--reps 3] [--out results.json]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from bench_batch import SEEDS, bring_to, card, timed  # noqa: E402

WORKLOADS = ["tinyllama-1.1b", "qwen2.5-0.5b", "llama2-7b:bf16"]  # llama2-7b-int8 on request (--workload)


def host_search(members, one, full, first, pos, new, B):
    """Arm (b): beam.py's rule over candidates from Batch.step and kllm_logprobs_f32, forks by copy_prefix"""
    import torch
    from kuiperllama_b200 import beam, check
    lib, V = members[0].lib, members[0].shape.vocab_size
    ids_buf = torch.zeros(1, dtype=torch.int32, device="cuda")
    lp_buf = torch.empty(1, device="cuda")
    ti = torch.empty(B, dtype=torch.int32, device="cuda")
    tl = torch.empty(B, device="cuda")

    def cands(d):
        check(lib.kllm_logprobs_f32(ctypes.c_void_p(lib.kllm_decoder_logits_device(d.handle)), V,
                                    ctypes.c_void_p(ids_buf.data_ptr()), 1, B, ctypes.c_void_p(lp_buf.data_ptr()),
                                    ctypes.c_void_p(ti.data_ptr()), ctypes.c_void_p(tl.data_ptr()), None),
              "kllm_logprobs_f32")
        return [int(i) for i in ti.cpu().numpy()], tl.cpu().numpy()

    state = {"member": [0]}

    def candidates(beams):
        p = len(beams[0].ids)
        if p == 0:
            one.step([first], [pos])
            return [cands(members[0])]
        prev, mem, kept = state["member"], [-1] * B, set()
        for j, bm in enumerate(beams):
            if bm.parent not in kept:
                kept.add(bm.parent)
                mem[j] = prev[bm.parent]
        free = sorted(set(range(B)) - set(mem))
        for j, bm in enumerate(beams):
            if mem[j] < 0:
                mem[j] = free.pop(0)
                members[mem[j]].copy_prefix(members[prev[bm.parent]], pos + p)
        tokens, positions = [0] * B, [0] * B
        for j, bm in enumerate(beams):
            tokens[mem[j]], positions[mem[j]] = bm.ids[-1], pos + p
        full.step(tokens, positions)
        state["member"] = mem
        return [cands(members[mem[j]]) for j in range(B)]

    return beam.beam_search(candidates, B, new, (), 1.0, False, B, pos)


def kernel_times(fn):
    """Mean device time per launch (ms) of the fork and candidates kernels in one profiled call of fn"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    out = {}
    for e in prof.key_averages():
        for key in ("fork_rows_kernel", "beam_candidates_kernel"):
            if key in e.key and e.count:
                total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                out[key] = round(total / e.count / 1e3, 4)
    return out


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
    members = [Decoder(shape, w, weight_format=fmt) for _ in range(max(args.beams))]
    row_bytes = 2 * shape.layer_num * shape.kv_dim * 4  # one position's K and V rows of every layer, fp32
    rows = []
    for pos in args.pos:
        if pos + args.new > shape.seq_len:
            raise SystemExit(f"{name}: pos {pos} leaves too little of seq_len {shape.seq_len}")
        first = bring_to(members[0], shape, pos, 1000 * pos)
        for B in args.beams:
            ms = members[:B]
            full, one = Batch(ms), Batch(ms[:1])
            starts = [pos] * B
            firsts = [first] * B
            arms = {
                "a": lambda: full.beam_search(first, pos, args.new, (), 1.0, False, B),
                "b": lambda: host_search(ms, one, full, first, pos, args.new, B),
                "c": lambda: ms[0].generate_until(first, pos, args.new),
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
                if outs["a"] != outs["b"]:
                    raise SystemExit(f"{name} B={B} pos={pos}: kllm_batch_beam_search differs from the host search")
            # t(B): one batch step of B rows; the members' rows past pos are the searches' scratch
            full.generate(firsts, starts, args.new)
            step_ms = statistics.median(timed(lambda: full.generate(firsts, starts, args.new))[0]
                                        for _ in range(args.reps)) / args.new
            kt = kernel_times(arms["a"])
            med = {k: statistics.median(v) for k, v in times.items()}
            hyps, stats = outs["a"]
            passes = stats["passes"]
            row = {
                "workload": name, "engine": ms[0].engine, "B": B, "pos": pos, "new": args.new, "reps": args.reps,
                "passes": passes, "forks": stats["forks"], "fork_rows": stats["fork_rows"],
                "ms_beam": round(med["a"], 2), "ms_host_composed": round(med["b"], 2),
                "ms_greedy": round(med["c"], 2),
                "speedup_vs_host_composed": round(med["b"] / med["a"], 3),
                "cost_vs_greedy": round(med["a"] / med["c"], 3),
                "ms_per_pass": round(med["a"] / passes, 4), "t_B_ms": round(step_ms, 4),
                "pass_over_t_B": round(med["a"] / passes / step_ms, 4),
                "fork_kernel_ms": kt.get("fork_rows_kernel"), "candidates_kernel_ms": kt.get("beam_candidates_kernel"),
                "fork_bytes_per_pass": round(stats["fork_rows"] * row_bytes / passes),
                "best_score": hyps[0]["score"], "parity": "hypotheses equal", **info,
            }
            print(json.dumps(row), flush=True)
            rows.append(row)
            full.close(), one.close()
    for d in members:
        d.close()
    del w
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default=",".join(WORKLOADS))
    ap.add_argument("--beams", default="2,4,8")
    ap.add_argument("--pos", default="1,512")
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    args.beams = [int(x) for x in args.beams.split(",")]
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
