#!/usr/bin/env python
"""Phase timeline of one decode step of the persistent megakernel (kllm_decoder_profile).

    python tools/phase_timeline.py [--workload tinyllama-1.1b] [--pos 512] > profiles/rNN_phase_timeline.txt
"""
import argparse
import ctypes
import os
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="tinyllama-1.1b")
    ap.add_argument("--pos", type=int, default=256)
    ap.add_argument("--ghz", type=float, default=1.98, help="SM clock for cycles -> us (nvidia-smi clocks.max.sm)")
    a = ap.parse_args()
    from kuiperllama_b200 import SHAPES, Decoder, check, synth_weights
    shape = SHAPES[a.workload]
    dec = Decoder(shape, synth_weights(shape, "cuda", 1235))
    assert dec.engine == "persistent"
    dec.generate(1, 0, 8)
    NS = 16  # stamps per (CTA, phase): mega::kProfStamps
    cap = 200 * 2000 * NS
    buf = np.zeros(cap, np.uint64)
    g, p = ctypes.c_int32(), ctypes.c_int32()
    n = a.pos + 1
    check(dec.lib.kllm_decoder_profile(dec.handle, 1, 0, n, a.pos, buf.ctypes.data_as(ctypes.c_void_p), cap,
                                       ctypes.byref(g), ctypes.byref(p)), "profile")
    G, P = g.value, p.value
    raw = buf[: G * P * NS].reshape(G, P, NS).astype(np.int64)
    st = raw[:, :, :4]
    cyc = raw[:, :, 4:10]  # SM cycles of warp 0: addend prefetch, dots, reductions, epilogues, ring waits, stage rows
    polled = raw[:, :, 10]
    pblk = raw[:, :, 11]  # cycles the ring producer waited for a free slot (ring full: copies in flight or unread stages)
    pfills = raw[:, :, 12]
    t0 = st[:, 0, 0].min()
    st = (st - t0) / 1e3  # us
    polled = np.where(polled > 0, (polled - t0) / 1e3, st[:, :, 1])
    L = shape.layer_num
    print(f"# {shape.name}: phase timeline of the decode step at pos {a.pos} (us, globaltimer), grid {G}, {P} phases")
    print(f"# token time (first phase entered -> last barrier passed): {st[:, -1, 3].max():.1f} us")
    NPL = (P - 1) // L  # phases per layer: 5 with the fused attention, 6 with the split one
    names = ["qkv", "attn", "wo", "w1w3", "w2"] if NPL == 5 else ["qkv", "scores", "attn_pv", "wo", "w1w3", "w2"]
    stage = (st[:, :, 1] - st[:, :, 0])          # input staging (+norm)
    work = (st[:, :, 2] - st[:, :, 1])           # consuming ring stages (or attention)
    bar = (st[:, :, 3] - st[:, :, 2])            # waiting at the grid barrier
    dur = st[:, :, 3].max(axis=0) - st[:, :, 0].min(axis=0)
    poll = polled - st[:, :, 0]                  # of stage_x: until the input vector is complete
    ghz = a.ghz  # cycles -> us; the split is what matters
    print(f"{'phase':>10} {'count':>5} {'phase_us':>9} {'stage_x':>8} {'(poll)':>7} {'work_med':>9} {'work_max':>9} {'barrier_min':>11} "
          f"{'barrier_med':>11} {'prod_blk':>8} {'fills':>5} | warp 0 of the median CTA, us: {'ringwait':>8} {'dots':>6} {'reduce':>6} {'epilog':>6} {'addend':>6}")

    def row(nm, idx, ctas=slice(None)):
        c = np.median(cyc[ctas][:, idx], axis=0).mean(axis=0) / ghz / 1e3 if len(idx) > 1 else np.median(cyc[ctas][:, idx], axis=0)[0] / ghz / 1e3
        print(f"{nm:>10} {len(idx):5d} {dur[idx].mean():9.2f} {np.median(stage[:, idx]):8.2f} {np.median(poll[:, idx]):7.2f} {np.median(work[:, idx]):9.2f} "
              f"{work[:, idx].max(axis=0).mean():9.2f} {bar[:, idx].min(axis=0).mean():11.2f} {np.median(bar[:, idx]):11.2f} "
              f"{np.median(pblk[ctas][:, idx].mean(axis=1)) / ghz / 1e3:8.2f} {np.median(pfills[ctas][:, idx].mean(axis=1)):5.1f} | "
              f"{'':32s}{c[4]:8.2f} {c[1]:6.2f} {c[2]:6.2f} {c[3]:6.2f} {c[0]:6.2f}")
    fast = os.environ.get("KLLM_MODE") == "fast"
    sp = int(os.environ.get("KLLM_ATTN_SPLIT_SHOWN", "0")) or (4 if (NPL == 6 or fast) else 1)
    for k, nm in enumerate(names):
        attn_row = nm in ("attn", "scores", "attn_pv")
        row(nm, [l * NPL + k for l in range(L)], slice(0, shape.head_num * sp) if attn_row else slice(None))
    row("cls", [P - 1])
    print("# attention rows (thread 0 of the median ATTENTION CTA): ringwait = K/V tile waits, dots = scores, reduce = softmax, "
          "epilog = P.V, addend = input polls (+RoPE)")
    # with tagged hand-overs most phases have no barrier: `barrier_*` is then ~0 and the wait for the
    # previous phase's outputs shows up in `stage_x` of the consuming phase (the poll loop)
    heads = shape.head_num
    ai = [l * NPL + 1 for l in range(L)]
    pvi = [l * NPL + (2 if NPL == 6 else 1) for l in range(L)]
    attn = (st[:heads, pvi, 2] - st[:heads, ai, 0])
    print(f"# attention (scores + softmax + P.V) on the first {heads} attention CTAs: median {np.median(attn):.2f} us, slowest head per layer (mean) "
          f"{attn.max(axis=0).mean():.2f} us")
    print(f"# sum of phase durations: {dur.sum():.1f} us; barrier_min = time the LAST arriving CTA spends in the barrier")
    tok_us = st[:, -1, 3].max()
    blk_us = pblk.sum(axis=1) / ghz / 1e3
    ring_us = cyc[:, :, 4].sum(axis=1) / ghz / 1e3
    print(f"# ring producer waiting for a free slot (ring full): median CTA {np.median(blk_us):.1f} us = "
          f"{100 * np.median(blk_us) / tok_us:.1f} % of the token, max CTA {blk_us.max():.1f} us; "
          f"consumer warp 0 waiting on a stage (ringwait): median CTA {np.median(ring_us):.1f} us = "
          f"{100 * np.median(ring_us) / tok_us:.1f} %")
    # ---- critical path: absolute times of one layer's all-to-all points, averaged over the layers -----------
    # last_done(X) = when the slowest CTA finished producing X; polled(Y) = when the median CTA held all of
    # Y's input vector; hand-off latency = polled(next) - last_done(prev); the phase body = last_done - polled.
    n_attn = shape.head_num * sp
    if NPL == 5:
        k_qkv, k_attn, k_wo, k_w13, k_w2 = 0, 1, 2, 3, 4
        rows = []
        for l in range(1, L - 1):
            b = l * NPL
            q_pol = np.median(polled[:, b + k_qkv])
            q_done = st[:, b + k_qkv, 2].max()
            a_done = st[:n_attn, b + k_attn, 2].max()
            a_done_med = np.median(st[:n_attn, b + k_attn, 2])
            wo_pol = np.median(polled[:, b + k_wo])
            wo_done = st[:, b + k_wo, 2].max()
            w13_pol = np.median(polled[:, b + k_w13])
            w13_done = st[:, b + k_w13, 2].max()
            w2_pol = np.median(polled[:, b + k_w2])
            w2_done = st[:, b + k_w2, 2].max()
            nq_pol = np.median(polled[:, b + NPL + k_qkv])
            rows.append([q_done - q_pol, a_done_med - q_done, a_done - q_done, wo_pol - a_done, wo_done - wo_pol,
                         w13_pol - wo_done, w13_done - w13_pol, w2_pol - w13_done, w2_done - w2_pol, nq_pol - w2_done,
                         nq_pol - q_pol])
        m = np.array(rows).mean(axis=0)
        print("# critical path of a layer (us, mean over layers 1..L-2): qkv body %.2f | attention: median CTA done +%.2f, "
              "last CTA done +%.2f after the last qkv row | -> wo input complete %.2f | wo body %.2f | -> w1w3 input %.2f | "
              "w1w3 body %.2f | -> w2 input %.2f | w2 body %.2f | -> next qkv input %.2f | layer %.2f"
              % tuple(m))
        # which attention CTAs finish last, and how their time splits (thread 0 cycles)
        b = (L // 2) * NPL
        order = np.argsort(-st[:n_attn, b + k_attn, 2])[:6]
        q_done = st[:, b + k_qkv, 2].max()
        for c in order:
            cy = cyc[c, b + k_attn] / ghz / 1e3
            print(f"#   layer {L // 2}: attention CTA {c} (head {c // sp}, split {c % sp}) entered {st[c, b + k_attn, 0] - q_done:+.2f}, "
                  f"done {st[c, b + k_attn, 2] - q_done:+.2f} vs last qkv row; polls+rope {cy[0]:.2f} scores {cy[1]:.2f} merges {cy[2]:.2f} "
                  f"pv {cy[3]:.2f} ringwait {cy[4]:.2f}")
        # who finishes the qkv phase last (the rows every attention CTA waits for)
        order = np.argsort(-st[:, b + k_qkv, 2])[:4]
        print("#   layer %d: last qkv CTAs %s finish %s us after the median CTA" % (
            L // 2, list(order), np.round(st[order, b + k_qkv, 2] - np.median(st[:, b + k_qkv, 2]), 2)))


if __name__ == "__main__":
    main()
